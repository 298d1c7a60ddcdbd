// formant_math.cuh -- per-frame arithmetic of the formant chain (cLpc -> cFormantLpc), written once for the
// device (formant.cu) and for a host build of the same statements (tests/native/formant_host.cpp, which the
// CPU tests compare with the reference's level taps: the lanes of a warp become a loop).
// Citations relative to /root/reference/src.  Compile with FMA contraction off (-fmad=false / -ffp-contract=off):
// the float recursions below follow the reference's statement order.
#pragma once
#include <math.h>
#include <stddef.h>
#include "fft_ref_order.cuh"

#ifdef __CUDACC__
#define OSM_FM_HD __host__ __device__ __forceinline__
#else
#define OSM_FM_HD inline
#endif

namespace osm {
namespace fm {

constexpr int kMaxLpcOrder = 16;     // predictor order p (GeMAPS: 11)
constexpr int kAberthMaxIter = 64;

// CTA shape and per-warp scratch of formant_kernel (formant.cu).  They live here so that the graph pass can size the
// kernel's shared memory on the host (tables.cpp build_formant) and refuse a geometry before a plan touches a device.
constexpr int kFmtWarps = 8;               // warps per CTA = frames per transform / resampling batch
constexpr int kFmtFpw = 2;                 // frames per warp in the per-frame phase: a half warp each (one lane per lag / root, p <= 15)
constexpr int kFmtBatch = kFmtWarps * kFmtFpw;
constexpr size_t kFmtSmemLimit = 200 * 1024;

struct FmtWarpWs {                          // per-warp scratch of the per-frame phase
  double c[kMaxLpcOrder];                   // polynomial, ascending powers (monic)
  double zr[kMaxLpcOrder], zi[kMaxLpcOrder];
  double f[kMaxLpcOrder], b[kMaxLpcOrder];
  float r[kMaxLpcOrder + 1];
  float a[kMaxLpcOrder];
  int ok[kMaxLpcOrder];
  int n, z0;
};

// dynamic shared memory of formant_kernel: scratch | windowed frames or FFT planes of one batch | resampled frames of
// kFmtBatch frames
inline size_t formant_smem_bytes(bool refOrder, int frameSize, int nResPad)
{
  const size_t perFrame = refOrder ? (size_t)4 * ro::kPlane : (size_t)frameSize;
  return sizeof(FmtWarpWs) * kFmtBatch + ((size_t)kFmtWarps * perFrame + (size_t)kFmtBatch * nResPad) * sizeof(float);
}

// smileDsp_autoCorr (smileutil/smileUtil.c:1560-1569): one lag, float accumulation over i = lag .. n-1
OSM_FM_HD float acf_lag(const float *x, int n, int lag)
{
  float acc = 0.0f;
  for (int i = lag; i < n; i++) acc = acc + x[i] * x[i - lag];
  return acc;
}

// smileDsp_calcLpcAcf (smileutil/smileUtil.c:1572-1627): Levinson-Durbin in float on r[0..p].
// a[0..p-1] = predictor coefficients, returns the final error (lpc gain); all zero when r[0] == 0.
OSM_FM_HD float durbin(const float *r, int p, float *a)
{
  for (int i = 0; i < p; i++) a[i] = 0.0f;
  if (r[0] == 0.0f) return 0.0f;
  float e = r[0];
  for (int m = 1; m <= p; m++) {
    float s = 1.0f * r[m];
    for (int i = 1; i < m; i++) s = s + a[i - 1] * r[m - i];
    const float km = (-1.0f / e) * s;
    a[m - 1] = km;
    for (int i = 1; i <= m / 2; i++) {
      const float x = a[i - 1];
      a[i - 1] = a[i - 1] + km * a[m - i - 1];
      if (i < m / 2 || (m & 1) == 1) a[m - i - 1] = a[m - i - 1] + km * x;
    }
    e = e * (1.0f - km * km);
    if (e == 0.0f) { for (int i = m; i < p; i++) a[i] = 0.0f; break; }
  }
  return e;
}

// ------------------------------------------------------------------------------------------------------
// Roots of the monic polynomial  z^n + c[n-1] z^(n-1) + ... + c[0]  (double).  The reference balances the
// companion matrix and runs a shifted QR iteration on it (smileutil/zerosolve.cpp); here every root is refined
// simultaneously (Aberth-Ehrlich: Newton step of root k deflated by the other roots), one lane per root on the
// device.  Both deliver the roots of the same polynomial to a few ulps of its conditioning; cFormantLpc sorts the
// formants it derives from them, so the order in which a solver lists the roots is immaterial as long as no
// candidate is cut off (the graph compiler requires nFormants >= p / 2).
// ------------------------------------------------------------------------------------------------------

// starting points: a slightly irregular circle of radius |c0|^(1/n) (the geometric mean of the root moduli)
OSM_FM_HD void aberth_init(const double *c, int n, int k, double *zr, double *zi)
{
  double c0 = fabs(c[0]);
  double rad = c0 > 0.0 ? exp(log(c0) / (double)n) : 0.5;
  if (rad < 0.05) rad = 0.05;
  if (rad > 2.0) rad = 2.0;
  const double th = 6.283185307179586 * ((double)k + 0.25) / (double)n + 0.4;
  *zr = rad * cos(th) * (1.0 + 0.013 * (double)(k & 3));
  *zi = rad * sin(th) * (1.0 + 0.013 * (double)(k & 3));
}

// one simultaneous update of root k from the current set (zr, zi)[0..n-1]; returns |correction|^2
OSM_FM_HD double aberth_step(const double *c, int n, const double *zr, const double *zi, int k, double *outR, double *outI)
{
  const double x = zr[k], y = zi[k];
  // Horner for p and p' (explicit fused multiply-adds: this solver is not a restatement of reference arithmetic, any accurate
  // evaluation serves; the translation unit is otherwise compiled without contraction)
  double pr = 1.0, pi = 0.0, dr = 0.0, di = 0.0;
  for (int j = n - 1; j >= 0; j--) {
    const double ndr = fma(dr, x, fma(-di, y, pr)), ndi = fma(dr, y, fma(di, x, pi));
    dr = ndr; di = ndi;
    const double npr = fma(pr, x, fma(-pi, y, c[j])), npi = fma(pr, y, pi * x);
    pr = npr; pi = npi;
  }
  // w = p / p'
  double den = fma(dr, dr, di * di);
  if (den == 0.0) { *outR = x + 1e-3; *outI = y + 1e-3; return 1.0; }
  double inv = 1.0 / den;
  const double wr = fma(pr, dr, pi * di) * inv, wi = fma(pi, dr, -(pr * di)) * inv;
  // s = sum_{j != k} 1 / (z_k - z_j): one division per term
  double sr = 0.0, si = 0.0;
  for (int j = 0; j < n; j++) {
    if (j == k) continue;
    const double ar = x - zr[j], ai = y - zi[j];
    const double ad = fma(ar, ar, ai * ai);
    if (ad == 0.0) continue;
    const double ia = 1.0 / ad;
    sr = fma(ar, ia, sr); si = fma(-ai, ia, si);
  }
  // z_k -= w / (1 - w s)
  const double qr = 1.0 - fma(wr, sr, -(wi * si)), qi = -fma(wr, si, wi * sr);
  den = fma(qr, qr, qi * qi);
  double cr, ci;
  if (den == 0.0) { cr = wr; ci = wi; }
  else { inv = 1.0 / den; cr = fma(wr, qr, wi * qi) * inv; ci = fma(wi, qr, -(wr * qi)) * inv; }
  *outR = x - cr; *outI = y - ci;
  return cr * cr + ci * ci;
}

// convergence test of one root after a step: correction below 1e-14 of its modulus, or no longer shrinking while
// already below 1e-9 of it (the rounding floor of evaluating p at an ill-conditioned root).  The iteration converges
// cubically, so the step after the test passes sits at that floor; the callers run one more sweep.
OSM_FM_HD bool aberth_done(double corr2, double prev2, double zr, double zi)
{
  const double m2 = zr * zr + zi * zi;
  if (corr2 <= 1e-28 * m2 || corr2 < 1e-300) return true;
  return corr2 <= 1e-18 * m2 && corr2 >= 0.0625 * prev2;
}

// One root -> formant candidate.  smileMath_complexIntoUnitCircle (smileutil/smileUtil.c:992-1004) +
// the per-root part of smileDsp_lpcrootsToFormants (:2019-2054).  Returns true if the root yields a candidate.
// A root whose imaginary part is rounding noise of a real root is treated as real (the reference's QR iteration
// returns exactly 0 there): positive real roots map to 0 Hz, negative ones to the Nyquist frequency.
OSM_FM_HD bool root_to_formant(double re, double im, double T, double fLow, double fHigh, double *f, double *bw)
{
  if (fabs(im) <= 1e-13 * (fabs(re) + 1e-300)) im = 0.0;
  double ab = sqrt(re * re + im * im);
  if (ab > 1.0) {                       // 1 / conj(root)
    const double d2 = re * re + im * im;
    re = re / d2; im = im / d2;
    ab = sqrt(re * re + im * im);
  }
  if (im < 0.0) return false;
  const double spPi = T * 3.14159265358979323846;
  if (fHigh < fLow || fHigh > 1.0 / T) fHigh = 0.5 / T - fLow;
  const double fr = fabs(atan2(im, re)) / (spPi * 2.0);
  if (fr >= fLow && fr <= fHigh) { *f = fr; *bw = -log(ab) / spPi; return true; }
  return false;
}

}  // namespace fm
}  // namespace osm
