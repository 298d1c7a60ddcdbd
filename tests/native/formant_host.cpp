// formant_host.cpp -- host build of opensmile_b200/csrc/formant_math.cuh (test infrastructure).
// The CUDA kernel (opensmile_b200/csrc/formant.cu) runs these statements with one lane per lag / per root; here the
// lanes are loops, so the CPU tests can hold the arithmetic against the reference's level taps without a GPU.
//   g++ -O2 -ffp-contract=off -shared -fPIC -o formant_host.so formant_host.cpp
#include "../../opensmile_b200/csrc/formant_math.cuh"
#include "../../opensmile_b200/csrc/harmonics_math.cuh"
#include "../../opensmile_b200/csrc/fft_ref_order.cuh"
#include <vector>

using namespace osm::fm;

extern "C" {

// x[n] -> a[p] (predictor coefficients), returns the gain
float fmh_lpc(const float *x, int n, int p, float *a)
{
  float r[kMaxLpcOrder + 1];
  for (int l = 0; l <= p; l++) r[l] = acf_lag(x, n, l);
  return durbin(r, p, a);
}

// roots of z^n + c[n-1] z^(n-1) + .. + c[0]; returns the number of sweeps
int fmh_roots(const double *c, int n, double *zr, double *zi)
{
  double nr[kMaxLpcOrder], ni[kMaxLpcOrder], prev[kMaxLpcOrder];
  for (int k = 0; k < n; k++) prev[k] = 1e300;
  for (int k = 0; k < n; k++) aberth_init(c, n, k, &zr[k], &zi[k]);
  int it = 0;
  bool last = false;
  for (; it < kAberthMaxIter; it++) {
    bool all = true;
    for (int k = 0; k < n; k++) {
      const double c2 = aberth_step(c, n, zr, zi, k, &nr[k], &ni[k]);
      all = all && aberth_done(c2, prev[k], nr[k], ni[k]);
      prev[k] = c2;
    }
    for (int k = 0; k < n; k++) { zr[k] = nr[k]; zi[k] = ni[k]; }
    if (last) { it++; break; }          // the polishing sweep after every root met the test
    last = all;
  }
  return it;
}

// a[p] (cLpc level) -> freq[nF] | bw[nF] as cFormantLpc writes them (lld/formantLpc.cpp:255-301,379-392)
int fmh_formants(const float *a, int p, double T, int nF, double minF, double maxF, float *freq, float *bw)
{
  double c[kMaxLpcOrder], zr[kMaxLpcOrder], zi[kMaxLpcOrder], f[kMaxLpcOrder], b[kMaxLpcOrder];
  for (int i = 0; i < p; i++) c[i] = -(double)a[p - 1 - i];
  int n = p, z0 = 0;
  while (z0 < n && c[z0] == 0.0) z0++;               // roots at the origin: no candidates
  int nv = 0;
  if (z0 < n) {
    const int m = n - z0;
    fmh_roots(c + z0, m, zr, zi);
    for (int k = 0; k < m && nv < nF; k++)
      if (root_to_formant(zr[k], zi[k], T, minF, maxF, &f[nv], &b[nv])) nv++;
  }
  for (int i = nv; i < nF; i++) { f[i] = 0.0; b[i] = 0.0; }
  int nz = 0;
  while (nz < nF && f[nz] != 0.0) nz++;
  for (int i = 0; i < nz; i++)
    for (int j = i + 1; j < nz; j++)
      if (f[j] < f[i]) { double t = f[j]; f[j] = f[i]; f[i] = t; t = b[j]; b[j] = b[i]; b[i] = t; }
  for (int i = 0; i < nF; i++) { freq[i] = (float)f[i]; bw[i] = (float)b[i]; }
  return nv;
}

}

// ---- the product's table builder (opensmile_b200/csrc/tables.cpp, linked into this harness) + the kernel's
// resampling loop: xw[T][N] windowed frames -> res[T][I] (fmaf in sample order, as formant_kernel phase 2) ----
#include <cmath>
#include <cstdlib>
#include <string>
#include "../../opensmile_b200/csrc/plan.hpp"

namespace {
// the kernel's resampling of T windowed frames xw[T][N] -> res[T][nRes] with the op's table
void resample_frames(const osm::FormantOp &op, int N, const float *xw, int T, float *res)
{
  if (op.refOrder) {
    // the kernel's reference-order path (formant.cu): 512-point transform of the zero padded frame, then the float inverse sum
    using namespace osm::ro;
    const float *wc = op.D.data(), *cosT = wc + kNw + kNc, *sinT = cosT + (size_t)op.kHalf * op.nResPad;
    std::vector<float> buf(4 * kPlane);
    Planes a{buf.data(), buf.data() + kPlane}, b{buf.data() + 2 * kPlane, buf.data() + 3 * kPlane};
    for (int t = 0; t < T; t++) {
      for (int n = 0; n < kN; n++) {
        const int m = n - op.padLeft;
        const float v = (m >= 0 && m < N) ? xw[(size_t)t * N + m] : 0.0f;
        ((n & 1) ? a.im : a.re)[phys(n >> 1)] = v;
      }
      for (int i = 0; i < kItemsA; i++) phase_a(a, wc, i);
      for (int i = 0; i < kItemsB; i++) phase_b(a, wc, i);
      for (int i = 0; i < kItemsC; i++) phase_c(a, wc, i);
      for (int i = 0; i < kItemsD; i++) phase_d(a, b, wc + kNw, i);
      for (int i = 0; i < op.nRes; i++) {
        float acc = b.re[0];
        for (int k2 = 1; k2 < op.kHalf; k2++) {
          acc = acc + b.re[phys(k2)] * cosT[(size_t)k2 * op.nResPad + i];
          acc = acc + b.im[phys(k2)] * sinT[(size_t)k2 * op.nResPad + i];
        }
        res[(size_t)t * op.nRes + i] = acc / op.halfK;
      }
    }
  } else
    for (int t = 0; t < T; t++)
      for (int i = 0; i < op.nRes; i++) {
        float acc = 0.0f;
        for (int m = 0; m < N; m++) acc = fmaf(xw[(size_t)t * N + m], op.D[(size_t)m * op.nResPad + i], acc);
        res[(size_t)t * op.nRes + i] = acc;
      }
}

// the formant op the graph pass builds for these options (tables.cpp build_formant); false where it refuses them
bool formant_op(double sampleRate, int N, int nfft, double frameSizeSec, int zeroPadSymmetric, double targetFs, int p, int nFormants,
                double minF, double maxF, int saveNValid, int saveFormants, int saveBandwidths, osm::FormantOp &op)
{
  osm::FrontEnd fe;
  fe.sampleRate = sampleRate; fe.frameSize = N; fe.nfft = nfft; fe.frameSizeSec = frameSizeSec;
  fe.fftFrameSizeSec = nfft != N ? frameSizeSec * (double)nfft / (double)N : frameSizeSec;     // graph.cpp, cTransformFFT
  osm_b200_specresample rs{targetFs, -1.0};
  osm_b200_lpc lp{}; lp.p = p; lp.saveLPCoeff = 1;
  osm_b200_formantlpc fl{}; fl.nFormants = nFormants; fl.saveFormants = saveFormants; fl.saveBandwidths = saveBandwidths;
  fl.saveNumberOfValidFormants = saveNValid; fl.minF = minF; fl.maxF = maxF;
  // the composed table of a long frame takes seconds to build: the last op is kept for the calls of one case
  static std::vector<double> lastKey;
  static osm::FormantOp lastOp;
  static bool lastOk = false;
  const std::vector<double> key{sampleRate, (double)N, (double)nfft, frameSizeSec, (double)zeroPadSymmetric, targetFs, (double)p,
                                (double)nFormants, minF, maxF, (double)saveNValid, (double)saveFormants, (double)saveBandwidths,
                                getenv("OSM_B200_FORMANT_COMPOSED") ? 1.0 : 0.0};
  if (key != lastKey) {
    std::string err;
    lastOp = osm::FormantOp();                     // build_formant sets the reference-order fields only on that path
    lastOk = osm::build_formant(rs, lp, fl, fe, zeroPadSymmetric != 0, lastOp, err);
    lastKey = key;
  }
  op = lastOp;
  return lastOk;
}
}  // namespace

extern "C" {

// returns I (resampled samples per frame) or -1; *Tper = base period of the cLpc level; res may be null (query)
int fmh_resample(double sampleRate, int N, int nfft, double frameSizeSec, int zeroPadSymmetric, double targetFs,
                 int p, int nFormants, const float *xw, int T, float *res, double *Tper)
{
  osm::FormantOp op;
  if (!formant_op(sampleRate, N, nfft, frameSizeSec, zeroPadSymmetric, targetFs, p, nFormants, 50.0, 5450.0, 0, 1, 1, op)) return -1;
  if (Tper) *Tper = op.T;
  if (res) resample_frames(op, N, xw, T, res);
  return op.nRes;
}

// the path formant_kernel takes for these options: info = {refOrder, gathered (reference order: the inverse sum reads the
// bins gathered per frame batch), kHalf, padLeft, nRes, nResPad, frames per warp, shared memory bytes}; -1 = refused
int fmh_formant_path(double sampleRate, int N, int nfft, double frameSizeSec, int zeroPadSymmetric, double targetFs, int p,
                     int nFormants, int *info)
{
  osm::FormantOp op;
  if (!formant_op(sampleRate, N, nfft, frameSizeSec, zeroPadSymmetric, targetFs, p, nFormants, 50.0, 5450.0, 0, 1, 1, op)) return -1;
  info[0] = op.refOrder; info[1] = op.refOrder && op.kHalf <= 4 * ((2 * osm::ro::kPlane) / 16);    // formant.cu `gathered`
  info[2] = op.kHalf; info[3] = op.padLeft; info[4] = op.nRes; info[5] = op.nResPad;
  info[6] = (op.p + 1 <= 16) ? osm::fm::kFmtFpw : 1;                                               // formant.cu `fpw`
  info[7] = (int)osm::fm::formant_smem_bytes(op.refOrder, N, op.nResPad);
  return 0;
}

// formant_kernel's shared memory (formant_math.cuh) and the limit above which the graph pass refuses an op
long fmh_formant_smem(int refOrder, int N, int nResPad) { return (long)osm::fm::formant_smem_bytes(refOrder != 0, N, nResPad); }
long fmh_formant_smem_limit() { return (long)osm::fm::kFmtSmemLimit; }

}

// ---- cHarmonics (harmonics_math.cuh): one frame.  The kernel evaluates the autocorrelation lags it needs with the lanes of
// a warp over the bins; here the same cosine sum runs sequentially. ----
namespace {
struct AcfHost {
  const float *mag; int nb, N; const double *cosTab;
  float operator()(int j) const
  {
    auto p = [&](int k) { return (double)(mag[k] * mag[k]); };
    double s = 0.5 * p(0) + 0.5 * p(N / 2) * ((j & 1) ? -1.0 : 1.0);
    for (int k = 1; k < N / 2; k++) s += p(k) * cosTab[(j * k) & (N - 1)];
    return (float)fabs(s) / (float)nb;
  }
};
struct MagHost { const float *m; float operator()(int b) const { return m[b]; } };
}

extern "C" {

// out = [HNRdB if doHnr] | nDiffs differences | formant amplitudes faStart..faEnd (log rel. F0); returns the count
int fmh_harmonics(float F0, const float *formants, int nFmt, const float *mag, int nb, double binHz, int nHarm, int nDiffs,
                  const int *diffs, int faStart, int faEnd, float floorUnvoiced, int doHnr, float *out)
{
  using namespace osm::hm;
  int o = 0;
  const int N = (nb - 1) * 2;
  if (doHnr) {
    std::vector<double> cosTab(N);
    for (int m = 0; m < N; m++) cosTab[m] = cos(2.0 * M_PI * (double)m / (double)N);
    AcfHost A{mag, nb, N, cosTab.data()};
    const double fs = (double)(nb - 1) * binHz * 2.0;
    const int f0bin = F0 > 0.0f ? (int)floor(fs / (double)F0) : 0;                 // freqToAcfBinLin (:393-401)
    int ref = 0;
    if (f0bin > 0) ref = closest_peak(A, nb, f0bin);
    out[o++] = ref <= 0 ? 0.0f : hnr_db(A(0), A(ref));
  }
  if (F0 > 0.0f) {
    std::vector<Harm> H(nHarm);
    MagHost M{mag};
    find_harmonics(F0, M, nb, binHz, nHarm, H.data());
    int fa[kMaxFormants];
    for (int k = 0; k < nFmt; k++) fa[k] = formant_harmonic(H.data(), nHarm, formants[k]);
    for (int i = 0; i < nDiffs; i++)
      out[o++] = harmonic_difference(H.data(), nHarm, fa, nFmt, Diff{diffs[4 * i], diffs[4 * i + 1], diffs[4 * i + 2], diffs[4 * i + 3]});
    for (int k = faStart; k <= faEnd; k++) out[o++] = (k >= 1 && k <= nFmt && fa[k - 1] >= 0) ? H[fa[k - 1]].lr : 0.0f;
  } else {
    for (int i = 0; i < nDiffs; i++) out[o++] = 0.0f;
    for (int k = faStart; k <= faEnd; k++) out[o++] = floorUnvoiced;
  }
  return o;
}

// fmh_harmonics over T rows: F0[T], formants[T][nFmt], mag[T][nb] -> out[T][nOut]; returns nOut
int fmh_harmonics_rows(int T, const float *F0, const float *formants, int nFmt, const float *mag, int nb, double binHz, int nHarm,
                       int nDiffs, const int *diffs, int faStart, int faEnd, float floorUnvoiced, int doHnr, float *out)
{
  const int nOut = (doHnr ? 1 : 0) + nDiffs + (faEnd >= faStart ? faEnd - faStart + 1 : 0);
  for (int t = 0; t < T; t++)
    fmh_harmonics(F0[t], formants + (size_t)t * nFmt, nFmt, mag + (size_t)t * nb, nb, binHz, nHarm, nDiffs, diffs, faStart, faEnd,
                  floorUnvoiced, doHnr, out + (size_t)t * nOut);
  return nOut;
}

// harmonics_kernel's per-lane shortcut: lane i takes its predecessor's candidate bin from the closed form freq_to_bin(i F0, 0)
// and checks that its own candidate equals freq_to_bin((i + 1) F0, 0).  Returns the first harmonic whose check fails (the
// kernel then falls back to the sequential search), -1 if every check holds.  The candidates depend on F0 and the axis only.
int fmh_harmonic_shortcut_fails(float F0, int nb, double binHz, int nHarm)
{
  using namespace osm::hm;
  const int last0 = freq_to_bin(binHz, nb, 0.5f * F0, 1);
  for (int i = 0; i < nHarm; i++) {
    const int prev = i == 0 ? last0 : freq_to_bin(binHz, nb, (float)i * F0, 0);
    if (freq_to_bin(binHz, nb, (float)(i + 1) * F0, prev) != freq_to_bin(binHz, nb, (float)(i + 1) * F0, 0)) return i;
  }
  return -1;
}

// the product's window table (tables.cpp build_window), as the plan's windower level applies it
void fmh_window(int winFunc, int N, double sigma, double gain, float *w)
{
  const double al[4] = {0.16, 0.0, 0.0, 0.0};
  std::vector<float> v;
  osm::build_window(winFunc, N, sigma, gain, v, al, 0, 0.0);
  for (int n = 0; n < N; n++) w[n] = v[n];
}

// PCM -> cFormantLpc rows of T frames through formant_kernel's statements.  x = the mono float samples of the wave level (the
// caller converts and mixes down as td_pcm does), frames of N samples every S, windowed as FrameReader::at (x w + offset);
// then fmh_resample's transform / inverse sum, the autocorrelation, Durbin, the roots and emit().  out[T][nOut] with
// nOut = [nValid] | formants[nF] | bandwidths[nF] (nF = the clamped nFormants); res[T][I] and lpc[T][p] when not null.
// Returns nOut, or -1 where the graph pass refuses the geometry.
int fmh_formant_rows(const float *x, int N, int S, int T, const float *win, float winOffset, double sampleRate, int nfft,
                     double frameSizeSec, int zeroPadSymmetric, double targetFs, int p, int nFormants, double minF, double maxF,
                     int saveNValid, int saveFormants, int saveBandwidths, float *out, float *resOut, float *lpcOut)
{
  osm::FormantOp op;
  if (!formant_op(sampleRate, N, nfft, frameSizeSec, zeroPadSymmetric, targetFs, p, nFormants, minF, maxF, saveNValid, saveFormants,
                  saveBandwidths, op)) return -1;
  const int I = op.nRes, nF = op.nFormants;
  std::vector<float> xw((size_t)N), res((size_t)I), a(p), fq(nF), bw(nF);
  for (int t = 0; t < T; t++) {
    for (int m = 0; m < N; m++) xw[m] = x[(size_t)t * S + m] * win[m] + winOffset;
    resample_frames(op, N, xw.data(), 1, res.data());
    fmh_lpc(res.data(), I, p, a.data());
    const int nv = fmh_formants(a.data(), p, op.T, nF, minF, maxF, fq.data(), bw.data());
    float *dst = out + (size_t)t * op.nOut;
    int o = 0;
    if (op.saveNValid) dst[o++] = (float)nv;
    if (op.saveFormants) for (int i = 0; i < nF; i++) dst[o++] = fq[i];
    if (op.saveBandwidths) for (int i = 0; i < nF; i++) dst[o++] = bw[i];
    if (resOut) for (int i = 0; i < I; i++) resOut[(size_t)t * I + i] = res[i];
    if (lpcOut) for (int i = 0; i < p; i++) lpcOut[(size_t)t * p + i] = a[i];
  }
  return op.nOut;
}

}
