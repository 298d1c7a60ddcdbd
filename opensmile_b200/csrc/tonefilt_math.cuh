// tonefilt_math.cuh -- the block form of cTonefilt (lld/tonefilt.cpp:204-226) shared by tonefilt.cu and its host build
// (tests/native/tonefilt_host.cpp).
//
// Per note k (frequency f, decay d) the reference runs, for every sample m of the utterance (absolute index, T = 1 / fs),
//   s = d s + ((1 - d) sin(((2 pi) f) (m T))) x_m,   c = the same with cos,
// and writes y = (float) sqrt(c^2 + s^2), y *= 10.0 once per block of P samples.  With z = c + i s this is a first-order
// complex recurrence with a constant coefficient; over block b (samples bP .. bP + P - 1) it folds into
//   z_b = d^P z_{b-1} + e^{i theta_b} G_b,   theta_b = ((2 pi) f) ((double)(bP) T),   G_b = sum_j w_j x_{bP+j},
//   w_j = (1 - d) d^{P-1-j} e^{i ((2 pi) f) (j T)}.
// G is one product of the block matrix [blocks x P] with the table W [P x 2 nNotes] (re / im interleaved), in double; the
// block phase is evaluated from the reference's own argument once per block (no rotation carried across blocks, which would
// drift over a long file).  Everything here is double except the samples and the output values.
#pragma once
#include <cmath>
#include <vector>

#if defined(__CUDACC__)
#define OSM_TF_HD __host__ __device__ __forceinline__
#else
#define OSM_TF_HD inline
#endif

namespace osm {
namespace tf {

constexpr int kMaxNotes = 128;     // 2 nNotes columns = at most 32 column tiles of the product (4 per warp)

// columns of W and of the block sums: 2 per note, padded to whole 8-column MMA tiles
inline int padded_cols(int nNotes) { return (2 * nNotes + 7) / 8 * 8; }
// rows of W: the samples of a block, padded to whole k-steps of 4 (the padding rows are zero)
inline int padded_rows(int P) { return (P + 3) / 4 * 4; }

// W [padded_rows(P)][padded_cols(nNotes)] and the per-block decay a[k] = d^P, from the reference's tables freq / decayF
inline void block_tables(const std::vector<double> &freq, const std::vector<double> &decay, int P, double T,
                         std::vector<double> &W, std::vector<double> &a)
{
  const int n = (int)freq.size(), nc = padded_cols(n), kp = padded_rows(P);
  W.assign((size_t)kp * nc, 0.0);
  a.assign(n, 0.0);
  for (int k = 0; k < n; k++) {
    const double d = decay[k], w = 2.0 * M_PI * freq[k];
    a[k] = pow(d, (double)P);
    for (int j = 0; j < P; j++) {
      const double g = (1.0 - d) * pow(d, (double)(P - 1 - j));
      const double arg = w * ((double)j * T);
      W[(size_t)j * nc + 2 * k] = g * cos(arg);
      W[(size_t)j * nc + 2 * k + 1] = g * sin(arg);
    }
  }
}

// z <- a z + e^{i theta_b} G for block b (absolute block index) of note frequency f
OSM_TF_HD void block_step(double &zr, double &zi, double a, double gr, double gi, double f, long long b, int P, double T)
{
  const double arg = (2.0 * M_PI * f) * ((double)(b * (long long)P) * T);
  double sn, cs;
#if defined(__CUDA_ARCH__)
  sincos(arg, &sn, &cs);
#else
  sn = sin(arg); cs = cos(arg);
#endif
  const double hr = cs * gr - sn * gi, hi = cs * gi + sn * gr;
  zr = a * zr + hr;
  zi = a * zi + hi;
}

// the reference's output value: (float) sqrt(c * c + s * s), then y *= 10.0 (a multiply in double and another float rounding)
OSM_TF_HD float tone_value(double zr, double zi)
{
  const float y = (float)sqrt(zr * zr + zi * zi);
  return (float)((double)y * 10.0);
}

// cChroma on one row of nNotes tone values (lld/chroma.cpp:86-117): chroma i = float sum over the octaves in ascending order of
// note j * K + i; a value below silThresh or a zero double total gives a zero vector, otherwise every value is divided by (float)
// total.  Strided access: tone value n at t[n * ts], chroma value i to out[i * os].
OSM_TF_HD void chroma_row(const float *t, int ts, int nNotes, int K, float silThresh, float *out, int os)
{
  const int nOct = nNotes / K;
  double sum = 0.0;
  bool sil = false;
  for (int i = 0; i < K; i++) {
    float s = 0.f;
    for (int j = 0; j < nOct; j++) s = s + t[(j * K + i) * ts];
    if (s < silThresh) sil = true;
    sum += (double)s;
    out[i * os] = s;
  }
  if (sum == 0.0 || sil) {
    for (int i = 0; i < K; i++) out[i * os] = 0.f;
  } else {
    const float tot = (float)sum;
    for (int i = 0; i < K; i++) out[i * os] = out[i * os] / tot;
  }
}

}  // namespace tf
}  // namespace osm
