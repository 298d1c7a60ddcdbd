// rank_select.cuh -- cFunctionalPercentiles of contours longer than the shared-memory sort takes (functionals.cu,
// pctl_select_kernel), written once for the device and for a host build (tests/native/rank_select_host.cpp, compared on the CPU
// with np.sort).  An order statistic is one value whatever sorts the contour, so instead of sorting, every rank the enabled
// quartiles and percentiles read (both neighbours of an interpolated one) is found by an MSB-first radix walk over the
// order-preserving unsigned key of the float: four 8-bit digits, each chosen from a histogram of the values that share the
// rank's prefix so far.
//
// +-0: the key orders -0 just below +0 (its sign bit decides).  std::sort, which the reference uses (functionals.cpp:296-299),
// compares them equal, so every interleaving of the zeros is a sorted sequence; the key picks the one with the negative zeros
// first, and an order statistic that lands on a zero is -0 exactly when the contour holds more -0 than the rank reaches into.
// Compile with FMA contraction off (-fmad=false / -ffp-contract=off): the interpolation keeps the reference's two roundings.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "../../include/osm_b200_functionals.h"

#ifdef __CUDACC__
#define OSM_RS_HD __host__ __device__ __forceinline__
#else
#define OSM_RS_HD inline
#endif

namespace osm {
namespace rsel {

constexpr int kMaxRanks = 2 * (3 + OSM_B200_F_MAX_PCTL);   // (i1, i2) of three quartiles and every percentile
constexpr int kDigits = 256;

OSM_RS_HD uint32_t key(float x)
{
  uint32_t u;
  memcpy(&u, &x, sizeof u);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
OSM_RS_HD float value(uint32_t k)
{
  const uint32_t u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  float x;
  memcpy(&x, &u, sizeof x);
  return x;
}
// the prefix a key shares with the rank being walked before the digit at `shift` (24, 16, 8, 0) is chosen
OSM_RS_HD uint32_t prefix(uint32_t k, int shift) { return (uint32_t)((uint64_t)k >> (shift + 8)); }
OSM_RS_HD int digit(uint32_t k, int shift) { return (int)((k >> shift) & 0xffu); }

// hist: how many values with the rank's prefix have each digit; r: the rank among them.  Returns the digit that holds rank r and
// leaves in r its rank among the values with that digit.
template <class Count>
OSM_RS_HD int digit_of_rank(const Count *hist, long long &r)
{
  int d = 0;
  while (r >= (long long)hist[d]) { r -= (long long)hist[d]; d++; }
  return d;
}

// getInterpPctl / getPctlIdx (functionalPercentiles.cpp:309-336): the ranks a percentile reads, i1 == i2 when it reads one
OSM_RS_HD void pctl_ranks(double p, long long N, int interp, long long &i1, long long &i2)
{
  if (interp) {
    const double idx = p * (double)(N - 1);
    i1 = (long long)floor(idx); i2 = (long long)ceil(idx);
    i1 = i1 < 0 ? 0 : (i1 >= N ? N - 1 : i1);
    i2 = i2 < 0 ? 0 : (i2 >= N ? N - 1 : i2);
  } else {
    long long r = (long long)round(p * (double)(N - 1));
    i1 = i2 = r < 0 ? 0 : (r >= N ? N - 1 : r);
  }
}
OSM_RS_HD float pctl_value(double p, long long N, long long i1, long long i2, float s1, float s2)
{
  if (i1 == i2) return s1;
  const double idx = p * (double)(N - 1);
  const double w1 = idx - (double)i1, w2 = (double)i2 - idx;
  return s1 * (float)w2 + s2 * (float)w1;
}

// the ranks of the percentile block: walker 2j / 2j + 1 are (i1, i2) of quartile j (j < 3) or of percentile j - 3
template <class Pctl>
OSM_RS_HD int pctl_walkers(const Pctl &P, long long N, long long *rank)
{
  const int nP = 3 + P.n_percentile;
  for (int j = 0; j < nP; j++) {
    const double p = j < 3 ? 0.25 * (double)(j + 1) : P.percentile[j - 3];
    pctl_ranks(p, N, P.interp, rank[2 * j], rank[2 * j + 1]);
  }
  return 2 * nP;
}

// the values of the percentile block in the reference's order (functionalPercentiles.cpp:219-262) from the values at the walkers'
// ranks; returns the number written
template <class Pctl>
OSM_RS_HD int pctl_block(const Pctl &P, long long N, const long long *rank, const float *sel, float *out)
{
  float q[3];
  for (int j = 0; j < 3; j++) q[j] = pctl_value(0.25 * (double)(j + 1), N, rank[2 * j], rank[2 * j + 1], sel[2 * j], sel[2 * j + 1]);
  int n = 0;
  if (P.quartile1) out[n++] = q[0];
  if (P.quartile2) out[n++] = q[1];
  if (P.quartile3) out[n++] = q[2];
  if (P.iqr12) out[n++] = q[1] - q[0];
  if (P.iqr23) out[n++] = q[2] - q[1];
  if (P.iqr13) out[n++] = q[2] - q[0];
  const int n0 = n;
  for (int i = 0; i < P.n_percentile; i++) {
    const int j = 2 * (3 + i);
    out[n++] = pctl_value(P.percentile[i], N, rank[j], rank[j + 1], sel[j], sel[j + 1]);
  }
  for (int i = 0; i < P.n_pctlrange; i++) out[n++] = fabsf(out[n0 + P.pctlrange[i][1]] - out[n0 + P.pctlrange[i][0]]);
  return n;
}

}  // namespace rsel
}  // namespace osm
