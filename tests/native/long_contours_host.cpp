// Host build of the long-contour path's host-visible pieces for the CPU tests (tests/test_long_contours_cpu.py): the order-preserving
// key and the radix digit walk of opensmile_b200/csrc/rank_select.cuh, with the percentile block assembled from the selected values
// as pctl_select_kernel does, and the work space chunk plan of opensmile_b200/csrc/long_contours.hpp.  Test infrastructure.
#include <vector>

#include "../../opensmile_b200/csrc/long_contours.hpp"
#include "../../opensmile_b200/csrc/rank_select.cuh"

using namespace osm;

extern "C" {

unsigned lch_key(float x) { return rsel::key(x); }
float lch_value(unsigned k) { return rsel::value(k); }

// the value of rank r of x[0 .. N) by the four-digit walk: one histogram per digit over the values sharing the prefix so far
float lch_select(const float *x, long long N, long long r)
{
  uint32_t pre = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    unsigned hist[rsel::kDigits] = {0};
    for (long long i = 0; i < N; i++) {
      const uint32_t k = rsel::key(x[i]);
      if (rsel::prefix(k, shift) == pre) hist[rsel::digit(k, shift)]++;
    }
    pre = (pre << 8) | (uint32_t)rsel::digit_of_rank(hist, r);
  }
  return rsel::value(pre);
}

// the percentile block of cFunctionalPercentiles for x[0 .. N) (spec: its percentile options); returns the number of values
int lch_pctl_block(const osm_b200_functionals_spec *s, const float *x, long long N, float *out)
{
  long long rank[rsel::kMaxRanks];
  float sel[rsel::kMaxRanks];
  const int nr = rsel::pctl_walkers(s->percentiles, N, rank);
  for (int w = 0; w < nr; w++) sel[w] = lch_select(x, N, rank[w]);
  return rsel::pctl_block(s->percentiles, N, rank, sel, out);
}

// chunk plan: contours [nC][3] = (u, e, chunk), chunks [nK][3] = (begin, end, cap); returns the work space floats, or -1 when the
// output arrays are too small
long long lch_plan(const int64_t *nRows, int nUtt, int nIn, int listMul, int lensFloats, long long capFloats, int *contours, int maxC,
                   int *chunks, int maxK, int *nC, int *nK)
{
  std::vector<LongContour> lc;
  std::vector<LongChunk> ch;
  const long long need = plan_long_contours(nRows, nUtt, nIn, listMul, lensFloats, capFloats, lc, ch);
  *nC = (int)lc.size(); *nK = (int)ch.size();
  if ((int)lc.size() > maxC || (int)ch.size() > maxK) return -1;
  for (size_t k = 0; k < ch.size(); k++) {
    chunks[3 * k] = ch[k].begin; chunks[3 * k + 1] = ch[k].end; chunks[3 * k + 2] = ch[k].cap;
    for (int c = ch[k].begin; c < ch[k].end; c++) { contours[3 * c] = lc[c].u; contours[3 * c + 1] = lc[c].e; contours[3 * c + 2] = (int)k; }
  }
  return need;
}

long long lch_slice_floats(long long cap, int listMul, int lensFloats) { return long_slice_floats(cap, listMul, lensFloats); }
int lch_max_short(void) { return kMaxShort; }
long long lch_ws_cap(void) { return kLongWsCapFloats; }

}  // extern "C"
