// pitch.cu -- the sub-harmonic-summation pitch chain of the ComParE / GeMAPS graphs (SURVEY.md 8f-1), sm_90a:
//   shs_kernel       cSpecScale + cPitchShs (+ cPitchBase output logic), one WARP per frame
//   viterbi_kernel   cPitchSmootherViterbi [+ cValbasedSelector], one THREAD per utterance (sequential in time)
//   jitter_kernel    cPitchJitter, one WARP per utterance (sequential over frames and pitch periods, lanes =
//                    candidate period lengths of the waveform matching; -DOSM_JITTER_EXACT_CC selects the reference's
//                    two-pass cross correlation instead of the one-pass form)
//   seq_post_kernel  cContourSmoother / cDeltaRegression(onlyInSegments) of the levels behind them, one thread
//                    per utterance (the delta's norm is a running sum over the whole level)
// Citations are relative to /root/reference/src.  Compiled with -fmad=false: the reference's x86-64 build has
// no FMA contraction, and the discrete decisions below (peak picking, path costs, period matching) should see
// the same roundings.
#include <cfloat>
#include <climits>
#include <cmath>

#include "kernels.cuh"

namespace osm {

namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kShsWarps = 8;      // warps per CTA (fewer when a long spectrum needs more workspace per warp)

// smileutil/smileUtil.c:1009-1034: vertex of the parabola through three points
__device__ double quad3(double x1, double y1, double x2, double y2, double x3, double y3, double *y, double *aOut)
{
  const double den = x1 * x1 * x2 + x2 * x2 * x3 + x3 * x3 * x1 - x3 * x3 * x2 - x2 * x2 * x1 - x1 * x1 * x3;
  if (den != 0.0) {
    const double a = (y1 * x2 + y2 * x3 + y3 * x1 - y3 * x2 - y2 * x1 - y1 * x3) / den;
    const double b = (x1 * x1 * y2 + x2 * x2 * y3 + x3 * x3 * y1 - x3 * x3 * y2 - x2 * x2 * y1 - x1 * x1 * y3) / den;
    const double c = (x1 * x1 * x2 * y3 + x2 * x2 * x3 * y1 + x3 * x3 * x1 * y2 - x3 * x3 * x2 * y1 - x2 * x2 * x1 * y3 - x1 * x1 * x3 * y2) / den;
    if (a != 0.0) {
      if (aOut) *aOut = a;
      const double x = -b / (2.0 * a);
      if (y) *y = c - a * x * x;
      return x;
    }
  }
  if (aOut) *aOut = 0.0;
  if (y1 > y2 && y1 > y3) { if (y) *y = y1; return x1; }
  else if (y2 > y1 && y2 > y3) { if (y) *y = y2; return x2; }
  else if (y3 > y1 && y3 > y2) { if (y) *y = y3; return x3; }
  if (y) *y = y1;
  return x1;
}

// ------------------------------------------------------------------------------------------ shs_kernel

// warp-wide (value, index) maximum; ties keep the lower index; idx < 0 = no entry
__device__ __forceinline__ void warp_argmax(float &v, int &idx)
{
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    const float ov = __shfl_xor_sync(kFull, v, d);
    const int oi = __shfl_xor_sync(kFull, idx, d);
    if (oi >= 0 && (idx < 0 || ov > v || (ov == v && oi < idx))) { v = ov; idx = oi; }
  }
}

__global__ void __launch_bounds__(kShsWarps * 32) shs_kernel(const ShsParams p)
{
  extern __shared__ __align__(16) unsigned char smemRaw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int N = p.nMag, M = p.nPts;
  // per warp: spectrum yS | second derivatives uS (doubles), scaled spectrum hps (float), 24 candidate floats; the
  // summed spectrum SS reuses the second-derivative buffer, which is dead once the interpolation has run
  const size_t perWarp = ((size_t)2 * (N + 2) * sizeof(double) + (size_t)M * sizeof(float) + 128 + 15) & ~(size_t)15;   // keeps the doubles aligned
  unsigned char *ws = smemRaw + warp * perWarp;
  double *yS = reinterpret_cast<double *>(ws);
  double *uS = yS + (N + 2);
  float *hps = reinterpret_cast<float *>(yS + 2 * (N + 2));
  float *cand = hps + M;                      // [3][8]: f0 | voicing | score
  const OpTile tl = p.tiles[blockIdx.x];
  const long long rowBase = p.statOff[tl.utt] + tl.f0;
  const int lo = lane * p.blk, hi = min(N, lo + p.blk);

  const int nWarps = blockDim.x >> 5;
  for (int f = warp; f < tl.nf; f += nWarps) {
    const float *mg = p.mag + ((size_t)blockIdx.x * N) * p.F + f;
#pragma unroll 4
    for (int j = lane; j < N; j += 32) yS[j] = (double)mg[(size_t)j * p.F];      // dsp/specScale.cpp:329-331
    __syncwarp();
    if (p.enhance) {                                                             // smileUtil.c:1965-2003
      // local maxima as bits: position j = 32 k + lane -> bit `lane` of the k-th ballot word (kept in shared memory,
      // 65 words at most); "a maximum within two bins" is a 5-bit window of the concatenated words
      unsigned int *mw = reinterpret_cast<unsigned int *>(uS);
      const int nWords = (N + 31) >> 5;
      int cnt = 0, fmin = INT_MAX, fmax = -1;
      for (int k = 0; k < nWords; k++) {
        const int j = (k << 5) + lane;
        bool m = false;
        if (j < N) {
          if (j == 0) m = yS[0] > yS[1];
          else if (j == N - 1) m = yS[N - 1] > yS[N - 2];
          else m = yS[j] > yS[j - 1] && yS[j] >= yS[j + 1];
        }
        const unsigned int w = __ballot_sync(kFull, m);
        if (lane == 0) mw[k + 1] = w;
        if (w) {
          cnt += __popc(w);
          if (fmin == INT_MAX) fmin = (k << 5) + __ffs(w) - 1;
          fmax = (k << 5) + 31 - __clz(w);
        }
      }
      if (lane == 0) { mw[0] = 0; mw[nWords + 1] = 0; }
      __syncwarp();
      for (int k = 0; k < nWords; k++) {
        const int j = (k << 5) + lane;
        if (j >= N) break;
        bool zero;
        if (cnt == 1) zero = j >= 3;            // the reference reads posmax[1] == 0 here
        else {
          // bits of positions 32k-32 .. 32k+63 ; position j sits at bit 32 + lane
          const unsigned long long lo64 = ((unsigned long long)mw[k + 1] << 32) | mw[k];
          const unsigned int hiw = mw[k + 2];
          const int b = 32 + lane;                                       // window bits b-2 .. b+2
          unsigned long long win = lo64 >> (b - 2);
          if (b + 2 >= 64) win |= (unsigned long long)hiw << (64 - (b - 2));
          zero = j > fmin && j < fmax && (win & 0x1full) == 0;
        }
        if (zero) yS[j] = 0.0;
      }
      __syncwarp();
    }
    if (p.smooth) {                                                              // smileUtil.c:2006-2016
      for (int j = lane; j < N; j += 32)
        uS[j] = j < N - 1 ? ((j > 0 ? yS[j - 1] : 0.0) + 2.0 * yS[j] + yS[j + 1]) / 4.0 : yS[j];
      __syncwarp();
      double *t = yS; yS = uS; uS = t;
    }
    // natural cubic spline: second derivatives by two first-order recurrences (smileUtilSpline.c:142-190);
    // lane l owns points [lo, hi), the carries cross the lanes through a scan of affine maps
    {
      double A = 1.0, B = 0.0;
      // (coefficient tables are stored lane-interleaved: entry of (lane, step k) at [k * 32 + lane] -> coalesced)
#pragma unroll 4                                // the table loads (L2) of four steps in flight; only A, B carry a dependency
      for (int i = lo; i < hi; i++) {
        double a = 0.0, b = 0.0;
        const int q = (i - lo) * 32 + lane;
        if (i >= 1 && i <= N - 2) { a = p.fwdA[q]; b = p.fwdP6[q] * ((yS[i + 1] - yS[i]) * p.r1[q] - (yS[i] - yS[i - 1]) * p.r2[q]); }
        B = a * B + b; A = a * A;
        uS[i] = b;                              // the second pass of the scan reads it back instead of rebuilding it from four tables
      }
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const double A2 = __shfl_up_sync(kFull, A, d), B2 = __shfl_up_sync(kFull, B, d);
        if (lane >= d) { B = A * B2 + B; A = A * A2; }
      }
      double u = __shfl_up_sync(kFull, B, 1);
      if (lane == 0) u = 0.0;
      for (int i = lo; i < hi; i++) {
        const double a = (i >= 1 && i <= N - 2) ? p.fwdA[(i - lo) * 32 + lane] : 0.0;
        u = a * u + uS[i];
        uS[i] = u;
      }
      __syncwarp();
      A = 1.0; B = 0.0;
      for (int j = hi - 1; j >= lo; j--) {
        const double a = j <= N - 2 ? p.bwdD[(j - lo) * 32 + lane] : 0.0, b = j <= N - 2 ? uS[j] : 0.0;
        B = a * B + b; A = a * A;
      }
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const double A2 = __shfl_down_sync(kFull, A, d), B2 = __shfl_down_sync(kFull, B, d);
        if (lane + d < 32) { B = A * B2 + B; A = A * A2; }
      }
      double v = __shfl_down_sync(kFull, B, 1);
      if (lane == 31) v = 0.0;
      for (int j = hi - 1; j >= lo; j--) {
        const double a = j <= N - 2 ? p.bwdD[(j - lo) * 32 + lane] : 0.0, b = j <= N - 2 ? uS[j] : 0.0;
        v = a * v + b;
        uS[j] = v;
      }
      __syncwarp();
    }
#pragma unroll 4                                 // independent points: four iterations' table loads (5 per point, from L2) in flight
    for (int i = lane; i < M; i += 32) {                                         // smileUtilSpline.c:355-368, specScale.cpp:343-368
      const int k = p.ik[i];
      const double a = p.ia[i], b = 1.0 - a;
      const double o = a * yS[k] + b * yS[k + 1] + p.ic[i] * uS[k] + p.id[i] * uS[k + 1];
      float of = (float)o;
      if (p.hasAudW) of = of > 0.0f ? (float)((double)of * p.audW[i]) : 0.0f;
      if (i <= p.lfCutBin) of = 0.0f;                                            // lld/pitchShs.cpp:230-236
      hps[i] = of;
    }
    __syncwarp();
    // sub-harmonic summation (lld/pitchShs.cpp:238-258)
    float *SS = reinterpret_cast<float *>(uS);
    double part = 0.0;
    // two points per lane and iteration: the 15-fold shift-add of a point is one dependent float chain (the reference's order),
    // two independent chains hide its latency; the lane's running sum still takes its points in ascending order
    for (int j = lane; j < M; j += 64) {
      const int j2 = j + 32;
      const bool two = j2 < M;
      float s = hps[j], s2 = two ? hps[j2] : 0.0f;
      for (int h = 0; h < p.nHarm - 1; h++) {
        const int sh = p.shift[h];
        const float hs = p.hscale[h];
        const int q = j + sh, q2 = j2 + sh;
        if (q < M) s = s + hps[q] * hs;
        if (q2 < M) s2 = s2 + hps[q2] * hs;
      }
      s = s / (float)p.nHarm;
      if (s < 0) s = 0.0f;
      SS[j] = s;
      part += (double)s;
      if (two) {
        s2 = s2 / (float)p.nHarm;
        if (s2 < 0) s2 = 0.0f;
        SS[j2] = s2;
        part += (double)s2;
      }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) part += __shfl_xor_sync(kFull, part, d);
    const double ssMean = part / (double)M;                                      // :271,320
    __syncwarp();
    // peak candidates (:271-318)
    const int nC = p.nCand;
    if (lane < 8) { cand[lane] = 0.0f; cand[8 + lane] = 0.0f; cand[16 + lane] = 0.0f; }
    __syncwarp();
    int nCand = 0;
    if (p.greedy) {
      // the lane's local maxima (positions 1 + lane + 32 k) as a bit mask, found once: word 0 holds k < 64 (positions up to
      // 2048), word 1 the rest (nPts <= 4096 puts the last candidate position, nPts - 2, at k <= 127)
      unsigned long long pk0 = 0, pk1 = 0;
      for (int i = 1 + lane, k = 0; i < M - 1; i += 32, k++) {
        const float s = SS[i];
        if (SS[i - 1] < s && s > SS[i + 1]) {
          if (k < 64) pk0 |= 1ull << k;
          else pk1 |= 1ull << (k - 64);
        }
      }
      float lastS = FLT_MAX; int lastI = -1;
      for (int r = 0; r < nC; r++) {
        float bs = -1.0f; int bi = -1;
        for (unsigned long long m = pk0; m; m &= m - 1) {
          const int i = 1 + lane + 32 * (__ffsll((long long)m) - 1);
          const float s = SS[i];
          if ((s < lastS || (s == lastS && i > lastI)) && s > bs) { bs = s; bi = i; }
        }
        for (unsigned long long m = pk1; m; m &= m - 1) {
          const int i = 1 + lane + 32 * (63 + __ffsll((long long)m));
          const float s = SS[i];
          if ((s < lastS || (s == lastS && i > lastI)) && s > bs) { bs = s; bi = i; }
        }
        warp_argmax(bs, bi);
        if (bi < 0) break;
        if (lane == 0) { cand[r] = (float)bi; cand[16 + r] = bs; }
        lastS = bs; lastI = bi; nCand++;
      }
    } else {
      if (lane == 0) {
        for (int i = 1; i < M - 1; i++) {
          if (SS[i - 1] < SS[i] && SS[i] > SS[i + 1] && (SS[i] > cand[16] || cand[16] == 0.0f)) {
            for (int j = nC - 1; j > 0; j--) { cand[16 + j] = cand[16 + j - 1]; cand[j] = cand[j - 1]; }
            cand[0] = (float)i; cand[16] = SS[i];
            if (nCand < nC) nCand++;
          }
        }
      }
      nCand = __shfl_sync(kFull, nCand, 0);
    }
    __syncwarp();
    if (lane < nCand) {                                                          // :323-343
      const float fc = cand[lane];
      const int jx = (int)fc;
      const float f1 = fc * p.Fstept + p.Fmint;
      const float f2 = (fc + 1.0f) * p.Fstept + p.Fmint;
      const float f0 = (fc - 1.0f) * p.Fstept + p.Fmint;
      double sc = 0;
      const double fx = quad3((double)f0, (double)SS[jx - 1], (double)f1, (double)SS[jx], (double)f2, (double)SS[jx + 1], &sc, nullptr);
      cand[lane] = (float)exp(fx * p.logBase);
      cand[16 + lane] = (float)sc;
      cand[8 + lane] = (sc > 0.0 && sc > ssMean) ? (float)(1.0 - ssMean / sc) : 0.0f;
    }
    __syncwarp();
    if (lane == 0) {
      float *cf = cand, *cv = cand + 8, *cs = cand + 16;
      if (p.octaveCorr) {                                                        // :346-358
        for (int i = 1; i < nCand; i++) {
          if (cf[i] < cf[0] && cf[i] > 0 && (cv[i] > p.voicingCutoff || cv[i] >= 0.9 * p.voicingCutoff) &&
              cs[i] > ((1.0 / (float)(p.nHarm - 1) * p.hscale[0])) * cs[0]) {
            float t;
            t = cf[0]; cf[0] = cf[i]; cf[i] = t;
            t = cv[0]; cv[0] = cv[i]; cv[i] = t;
            t = cs[0]; cs[0] = cs[i]; cs[i] = t;
          }
        }
      }
      // cPitchBase::processVector (lldcore/pitchBase.cpp:196-290)
      int nc = nCand;
      if (nc > 0) {
        for (int i = 0; i < nC && nc > 0; i++) {
          if ((double)cf[i] > p.maxPitch || (double)cf[i] < p.minPitch) {
            const float origF = cf[i];
            int j;
            for (j = i + 1; j < nC; j++) { cf[j - 1] = cf[j]; cv[j - 1] = cv[j]; cs[j - 1] = cs[j]; }
            cf[j - 1] = 0; cv[j - 1] = 0; cs[j - 1] = 0;
            if (origF > 0.0f) { nc--; i--; }
          }
        }
      }
      float *dst = p.shs + (size_t)(rowBase + f) * p.nShsCols;
      int n = 0;
      dst[n++] = (float)nc;
      int maxI = 0;
      if (!p.octaveCorr) {
        float mx = cs[0];
        for (int i = 1; i < nC; i++) if (cs[i] > mx) { mx = cs[i]; maxI = i; }
      }
      if (maxI > 0) {
        float t;
        t = cf[0]; cf[0] = cf[maxI]; cf[maxI] = t;
        t = cv[0]; cv[0] = cv[maxI]; cv[maxI] = t;
        t = cs[0]; cs[0] = cs[maxI]; cs[maxI] = t;
      }
      for (int i = 0; i < nC; i++) dst[n++] = cf[i];
      if (p.voicing) for (int i = 0; i < nC; i++) dst[n++] = cv[i];
      if (p.scores) for (int i = 0; i < nC; i++) dst[n++] = cs[i];
      if (p.F0C1) dst[n++] = cf[0];
      if (p.voicingC1) dst[n++] = cv[0];
      if (p.F0raw) dst[n++] = cv[0] <= p.voicingCutoff ? 0.0f : cf[0];
      if (p.voicingClip) dst[n++] = cv[0] <= p.voicingCutoff ? 0.0f : cv[0];
    }
    __syncwarp();
    if (p.smooth) { double *t = yS; yS = uS; uS = t; }      // undo the swap: same buffers for the next frame
  }
}

// ------------------------------------------------------------------------------------------ viterbi_kernel

constexpr int kVitStates = 9, kVitBuf = 64;

// include/lld/pitchSmootherViterbi.hpp:167-197
__device__ __forceinline__ double vit_fweight(float f)
{
  if (f > 0.0 && f < 100.0) return -(1.0 / 100.0) * f + 1.0;
  else if (f >= 100.0 && f < 350.0) return 0.0;
  else if (f >= 350.0 && f < 600.0) return ((f - 350.0) / 250.0);
  else if (f >= 600.0) return 1.2;
  else if (f <= 0) return 2.0;
  return 0.0;
}

__global__ void __launch_bounds__(64) viterbi_kernel(const ViterbiParams p, int u0, int u1)
{
  const int u = u0 + blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= u1) return;
  const int T = (int)frame_count(p.uttOff[u + 1] - p.uttOff[u], p.frameSize, p.frameStep, p.frameCenter);
  if (T <= 0) { p.lag[u] = 0; return; }
  const long long row0 = p.statOff[u];
  const int nC = p.nCand, nS = nC + 1, last = nC, bl = p.bufLen;
  double costA[kVitStates], costB[kVitStates];
  // best path per state as packed bytes (entry k = byte k%4 of word k/4): copying a path moves bufLen/4 words
  unsigned int paths[2][kVitStates][kVitBuf / 4];
  unsigned char bestPath[kVitBuf];
  const int nW = (bl + 3) >> 2;
  auto path_get = [&](int b, int s, int k) -> int { return (paths[b][s][k >> 2] >> ((k & 3) * 8)) & 0xff; };
  auto path_set = [&](int b, int s, int k, int v) {
    const unsigned int sh = (k & 3) * 8;
    paths[b][s][k >> 2] = (paths[b][s][k >> 2] & ~(0xffu << sh)) | ((unsigned int)v << sh);
  };
  double rr[kVitStates][kVitStates];          // log(f1_i / f0_j) of the current frame pair (NaN = empty candidate)
  double *pathCosts = costA, *pathCostsNew = costB;
  double lastChange = 1.0;
  int pathBuf = 0, pathIdx = 0, convIdx = -1, rdIdx = 0;
  float lastValidf0 = 0.0f;
  const double thrD = (double)p.voiceThresh;

  auto local_cost = [&](int i, const float *fr) -> double {              // hpp:202-221; fr[1+k] = F0, fr[1+nC+k] = voicing
    if (i < last) {
      double pv = (double)fr[1 + nC + i];
      double thr = 0.0;
      if (pv < 0.01) pv = 0.01;
      if (pv > 1.00) pv = 1.00;
      if (pv < thrD) thr = p.wThr;
      return (-log(pv) + thr) * p.wLocal + vit_fweight(fr[1 + i]) * p.wRange;
    }
    double flag = 0.0;
    for (int j = 0; j < nC; j++) if (fr[1 + nC + j] >= p.voiceThresh) { flag = p.wThr; break; }
    return p.wLocal * flag;
  };
  auto drain = [&]() {                                                       // lld/pitchSmootherViterbi.cpp:470-545
    while (rdIdx <= convIdx) {
      const int state = bestPath[rdIdx % bl];
      const float *b = p.shs + (size_t)(row0 + rdIdx) * p.nShsCols;
      float f0 = state < last ? b[1 + state] : 0.0f;
      const float vp = state < nC ? b[1 + nC + state] : b[1 + nC];
      float *o = p.stat + (size_t)(row0 + rdIdx) * p.statStride + p.outCol;
      bool copy = true;
      if (p.hasSel) {                                                         // other/valbasedSelector.cpp:153-233
        const float val = p.stat[(size_t)(row0 + rdIdx) * p.statStride + p.selCol];
        copy = (!p.selInvert && val > p.selThreshold) || (p.selInvert && val < p.selThreshold) || (p.selAllowEqual && val == p.selThreshold);
      }
      int n = 0;
      // semitones above 27.5 Hz, float arithmetic like the reference's log(float) overload (:490-500,512-522).  CUDA's logf
      // is 1 ulp off the host's (glibc) logf on ~5 % of F0 values; the rounded double logarithm differs from it on ~0.1 %
      auto semitone = [](float f) -> float {
        return f > 29.136 ? 12.0f * (float)log((double)(f / 27.5f)) / (float)log(2.0) : (f > 0.0 ? 1.0f : 0.0f);
      };
      if (p.oF0final) o[n++] = copy ? f0 : p.selOutputVal;
      if (p.oF0finalLog) o[n++] = copy ? semitone(f0) : p.selOutputVal;
      if (p.oF0finalEnv || p.oF0finalEnvLog) {
        if (f0 <= 0.0) f0 = lastValidf0; else lastValidf0 = f0;
        if (p.oF0finalEnv) o[n++] = copy ? f0 : p.selOutputVal;
        if (p.oF0finalEnvLog) o[n++] = copy ? semitone(f0) : p.selOutputVal;
      }
      if (p.oVClipped) o[n++] = copy ? (vp >= p.voiceThresh ? vp : 0.0f) : p.selOutputVal;
      if (p.oVUnclipped) o[n++] = copy ? vp : p.selOutputVal;
      rdIdx++;
    }
  };

  for (int t = 0; t < T; t++) {                                               // lld/pitchSmootherViterbi.cpp:79-183
    const float *cur = p.shs + (size_t)(row0 + t) * p.nShsCols;
    const float *prv = cur - p.nShsCols;
    if (pathIdx == 0) {
      convIdx = -1;
      for (int i = 0; i < nS; i++) {
        pathCosts[i] = local_cost(i, cur);
        for (int w = 0; w < nW; w++) paths[pathBuf][i][w] = 0;
        path_set(pathBuf, i, 0, i);
      }
    } else {
      const int nb = pathBuf ^ 1;
      // the logarithms do not depend on the running `lastChange`: evaluate them up front (independent, pipelined),
      // then walk the (i, j) pairs in the reference's order
      for (int i = 0; i < nC; i++)
        for (int j = 0; j < nC; j++) {
          const float f0 = prv[1 + j], f1 = cur[1 + i];
          rr[i][j] = (f0 == 0 || f1 == 0) ? nan("") : log((double)(f1 / f0));
        }
      double lc[kVitStates];
      for (int i = 0; i < nS; i++) lc[i] = local_cost(i, cur);
      for (int i = 0; i < nS; i++) {
        int minState = 0;
        double minCost = 0.0;
        for (int j = 0; j < nS; j++) {
          double tc;                                                          // hpp:224-252 (i = current state, j = previous state)
          if ((int)(i == j) == last) tc = p.wTuu;                             // the reference's `i == j == nStates-1`
          else if (i < last && j < last) {
            const double r = rr[i][j];
            if (r != r) tc = 999.0;
            else {
              tc = p.wTvv * fabs(r) + p.wTvvd * fabs(r - lastChange);
              lastChange = r;
            }
          } else if ((i == last && j < last) || (i < last && j == last)) { lastChange = 0.0; tc = p.wTvuv; }
          else tc = 1.0;
          const double c = tc + pathCosts[j];
          if (j == 0 || c < minCost) { minState = j; minCost = c; }
        }
        pathCostsNew[i] = minCost + lc[i];
        for (int w = 0; w < nW; w++) paths[nb][i][w] = paths[pathBuf][minState][w];
        path_set(nb, i, pathIdx % bl, i);
      }
      double *tmp = pathCosts; pathCosts = pathCostsNew; pathCostsNew = tmp;
      pathBuf = nb;
    }
    pathIdx++;
    if (pathIdx - convIdx > bl) {
      int minState = 0;
      for (int i = 1; i < nS; i++) if (pathCosts[i] < pathCosts[minState]) minState = i;
      convIdx++;
      bestPath[convIdx % bl] = (unsigned char)path_get(pathBuf, minState, convIdx % bl);
    } else {
      for (int n = convIdx + 1; n < pathIdx; n++) {
        const int x = path_get(pathBuf, 0, n % bl);
        bool match = true;
        for (int i = 1; i < nS; i++) if (x != path_get(pathBuf, i, n % bl)) { match = false; break; }
        if (!match) break;
        convIdx++;
        bestPath[convIdx % bl] = (unsigned char)x;
      }
    }
    drain();
  }
  p.lag[u] = rdIdx;                       // frames written before the end of input is signalled
  {                                       // flushTrellis (hpp:105-125)
    int minState = 0;
    for (int i = 1; i < nS; i++) if (pathCosts[i] < pathCosts[minState]) minState = i;
    // at most bufLen entries are pending (forced decisions keep pathIdx - convIdx <= bufLen), so the ring is intact
    while (convIdx + 1 < pathIdx) {
      convIdx++;
      bestPath[convIdx % bl] = (unsigned char)path_get(pathBuf, minState, convIdx % bl);
      drain();
    }
  }
}

// ------------------------------------------------------------------------------------------ jitter_kernel

constexpr int kJitWarps = 4;

template <bool F32>
__device__ __forceinline__ float jit_pcm(const int16_t *s, int nChan)       // smileutil/smileUtil.c:2520-2534
{
  if constexpr (F32) return *reinterpret_cast<const float *>(s);      // pre-converted mono float sample (JitterParams::pcmF32)
  float tmp = (float)s[0];
  for (int c = 1; c < nChan; c++) tmp = tmp + (float)s[c];
  if (nChan > 1) tmp = tmp / (float)nChan;
  return tmp / 32767.0f;
}

#ifdef OSM_JITTER_EXACT_CC
// lld/pitchJitter.cpp:339-413, one lag per lane
__device__ double jit_cross_corr(const float *x, const float *y, int N)
{
  double cc = 0.0, mx = 0.0, my = 0.0, nx = 0.0, ny = 0.0;
#pragma unroll 4
  for (int i = 0; i < N; i++) { mx += x[i]; my += y[i]; }
  mx /= (double)N; my /= (double)N;
#pragma unroll 4
  for (int i = 0; i < N; i++) {
    const double dx = x[i] - mx, dy = y[i] - my;
    cc += dx * dy;
    nx += dx * dx;
    ny += dy * dy;
  }
  cc /= sqrt(nx) * sqrt(ny);
  return cc;
}
#endif

// first maximum / minimum of x[1 .. N-2] (lld/pitchJitter.cpp:424-431), all lanes get the result
__device__ void jit_extrema(const float *x, int N, int lane, float &mx, int &mI, float &mn)
{
  float bv = -FLT_MAX, lo = FLT_MAX; int bi = -1;
  for (int i = 1 + lane; i < N - 1; i += 32) {
    const float v = x[i];
    if (bi < 0 || v > bv) { bv = v; bi = i; }
    lo = fminf(lo, v);
  }
  warp_argmax(bv, bi);
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) lo = fminf(lo, __shfl_xor_sync(kFull, lo, d));
  if (bi < 0) { mx = x[1]; mI = 1; mn = x[1]; }
  else { mx = bv; mI = bi; mn = lo; }
}

// 80 registers: six CTAs (24 warps) per SM; faster than five on the ComParE workload (10 k utterances)
template <bool F32>
__global__ void __launch_bounds__(kJitWarps * 32, 6) jitter_kernel(const JitterParams p, int u0, int u1)
{
  extern __shared__ __align__(16) unsigned char smemRaw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int u = u0 + blockIdx.x * kJitWarps + warp;
  if (u >= u1) return;
  // workspace per warp, sized by the host from the frame geometry and the pitch range (launch_jitter)
  const int kJitCC = p.capCC, kJitWav = p.capWav, kJitAvg = p.capAvg, kJitPb = p.capPb;
  const size_t perWarp = (size_t)kJitCC * sizeof(double) + (size_t)(kJitWav + kJitAvg) * sizeof(float) + (size_t)kJitPb * sizeof(int);
  unsigned char *ws = smemRaw + warp * perWarp;
  double *cc = reinterpret_cast<double *>(ws);
  float *wav = reinterpret_cast<float *>(cc + kJitCC);
  float *avgWf = wav + kJitWav;
  int *pb = reinterpret_cast<int *>(avgWf + kJitAvg);

  const long long L = p.uttOff[u + 1] - p.uttOff[u];
  const int T = (int)frame_count(L, p.frameSize, p.frameStep, p.frameCenter);
  const int16_t *pcm = p.pcm + p.uttOff[u] * p.nChan;
  const long long row0 = p.statOff[u];
  const double Ts = p.Ts;
  // state (lld/pitchJitter.cpp:88-93), identical in every lane
  long long lastIdx = 0, lastMis = 0;
  float lastT0 = 0.0f, lastDiff = 0.0f, lastJitterLocal = 0.0f, lastJitterDDP = 0.0f, lastShimmerLocal = 0.0f;
  float lastJitterLocal_b = 0.0f, lastJitterDDP_b = 0.0f, lastShimmerLocal_b = 0.0f;
  float threshCC = p.threshCC;
  const int nOutCols = p.jitterLocal + p.jitterDDP + p.jitterLocalEnv + p.jitterDDPEnv + p.shimmerLocal + p.shimmerLocalDB +
                       p.shimmerLocalEnv + p.shimmerLocalDBEnv + p.harmonicERMS + p.noiseERMS + p.linearHNR + p.logHNR +
                       p.refinedF0 + p.srcQualMean + p.srcQualRange;

  for (int t = 0; t < T; t++) {
    float *o = p.stat + (size_t)(row0 + t) * p.statStride + p.outCol;
    const float F0 = p.stat[(size_t)(row0 + t) * p.statStride + p.f0Col];
    // time meta of frame t (core/dataMemoryLevel.cpp:617-625: lengthSec spans the source samples)
    const long long s0 = (long long)t * p.frameStep;
    const double time = (double)s0 * Ts;
    const double lengthSec = (double)(s0 + p.frameSize - 1) * Ts - (double)s0 * Ts + Ts;
    long long lenF = (long long)ceil(lengthSec / Ts);                         // :609
    const long long startVidx = (long long)round(time / Ts);                   // :612
    const long long ppLen = (long long)ceil(p.pitchT / Ts);                    // :616
    const long long toRead0 = ppLen + lastMis;
    long long toRead = toRead0;
    double Tf = 0.0;
    long long T0f = 0, T0minF = 0, T0maxF = 0;
    if (F0 > 0.0) {                                                            // :635-648
      const double T0 = 1.0 / F0;
      Tf = T0 / Ts;
      T0f = (long long)round(Tf);
      T0minF = (long long)floor((1.0 - p.searchRangeRel) * Tf);
      T0maxF = (long long)ceil((1.0 + p.searchRangeRel) * Tf);
      const long long two_pp = p.minNumPeriods * T0maxF + p.minNumPeriods;
      if (toRead < two_pp) toRead = two_pp;
    }
    long long maxRead = lastMis + lenF;
    if (toRead > maxRead) toRead = maxRead;
    if (startVidx - lastMis != lastIdx) {                                      // :658-663
      lastIdx = startVidx;
      if (toRead > lenF) toRead = lenF;
      if (maxRead > lenF) maxRead = lenF;
    }
    // a read window past the end of the input: the reference's getMatrix fails and the frame is dropped from its level
    // (:668-673).  That happens only in the last frames (lengthSec can round up to frameSize + 1 samples); the plan keeps one
    // row per frame, so the row is written as zeros and the state moves on as the reference's does
    const bool pastEnd = lastIdx + toRead > L;
    bool bad = toRead > kJitWav || toRead < 1;
    if (F0 > 0.0 && (T0maxF - T0minF + 1 > kJitCC || T0f + 1 > kJitAvg || T0minF < 1 || toRead / T0minF + 4 > kJitPb)) bad = true;
    if (bad || pastEnd) {    // outside the supported geometry: flagged
      if (lane == 0) { if (!pastEnd) atomicOr(p.errFlag, 1); for (int k = 0; k < nOutCols; k++) o[k] = 0.0f; }
      lastIdx += toRead0;
      continue;
    }
    const int nT = (int)toRead;
    __syncwarp();
    for (int i = lane; i < nT; i += 32) wav[i] = jit_pcm<F32>(pcm + (lastIdx + i) * p.nChan, p.nChan);
    __syncwarp();

    float nPeriodsLocal = 0, nPeriodsDDP = 0, nPeriods = 0, avgPeriod = 0.0f, JitterDDP = 0.0f, JitterLocal = 0.0f;
    float avgAmp = 0.0f, avgAmpDiff = 0.0f, eH = 0.0f, eN = 0.0f, HNR = 0.0f, lgHNR = 0.0f, sumCC = 0.0f, maxCC = -2.0f, minCC = -2.0f;
    long long lastPeriod = 0;
    if (F0 > 0.0) {
      const int t0f = (int)T0f, tmin = (int)T0minF, tmax = (int)T0maxF, nLag = tmax - tmin + 1;
      int numPeriods = 0, start = 0, pp = 0;
      for (int i = lane; i <= t0f; i += 32) avgWf[i] = 0.0f;
      for (int i = lane; i < kJitPb; i += 32) pb[i] = 0;
      __syncwarp();
      while (start < nT - 2 * tmax - 1) {                                      // :728
#ifdef OSM_JITTER_EXACT_CC
        // the reference's two-pass form, bit-identical cc (lld/pitchJitter.cpp:339-413); ~3.7x the instructions
        for (int k = lane; k < nLag; k += 32) cc[k] = jit_cross_corr(wav + start, wav + start + tmin + k, tmin + k);
#else
        // One-pass form of the same normalised cross correlation:
        //   cc = (Sxy - Sx Sy / N) / (sqrt(Sxx - Sx^2 / N) sqrt(Syy - Sy^2 / N)),
        // x = w[start .. start+tf), y = w[start+tf .. start+2tf).  The window sums of all candidate lengths are prefix
        // sums P(t) = sum_{i<t} w[start+i] (and of squares): Sx = P(tf), Sy = P(2 tf) - P(tf).  Per round of 32
        // consecutive tf they come from two warp scans; only Sxy needs a loop per lane.  Products of floats are
        // exact in double, so the result differs from the two-pass value by a few 1e-16 (relative to the sums).
        {
          const float *w = wav + start;
          double PA1 = 0.0, PA2 = 0.0, PB1 = 0.0, PB2 = 0.0;            // P(t0), P(2 t0) -- uniform over the warp
          for (int i = lane; i < 2 * tmin; i += 32) {
            const double v = (double)w[i], v2 = v * v;
            PB1 += v; PB2 += v2;
            if (i < tmin) { PA1 += v; PA2 += v2; }
          }
#pragma unroll
          for (int d = 16; d > 0; d >>= 1) {
            PA1 += __shfl_xor_sync(kFull, PA1, d); PA2 += __shfl_xor_sync(kFull, PA2, d);
            PB1 += __shfl_xor_sync(kFull, PB1, d); PB2 += __shfl_xor_sync(kFull, PB2, d);
          }
          for (int t0 = tmin; t0 <= tmax; t0 += 32) {
            const int tf = t0 + lane;
            // elements entering the prefixes between this lane's tf and the next one
            double e1 = 0.0, e2 = 0.0, g1 = 0.0, g2 = 0.0;
            if (start + tf < nT) { const double v = (double)w[tf]; e1 = v; e2 = v * v; }
            if (start + 2 * tf + 1 < nT) {
              const double a = (double)w[2 * tf], b = (double)w[2 * tf + 1];
              g1 = a + b; g2 = a * a + b * b;
            }
            double s1 = e1, s2 = e2, q1 = g1, q2 = g2;                  // inclusive scans
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
              const double a1 = __shfl_up_sync(kFull, s1, d), a2 = __shfl_up_sync(kFull, s2, d);
              const double b1 = __shfl_up_sync(kFull, q1, d), b2 = __shfl_up_sync(kFull, q2, d);
              if (lane >= d) { s1 += a1; s2 += a2; q1 += b1; q2 += b2; }
            }
            const double Sx = PA1 + (s1 - e1), Sxx = PA2 + (s2 - e2);   // P(tf)
            const double P2a = PB1 + (q1 - g1), P2b = PB2 + (q2 - g2);  // P(2 tf)
            if (tf <= tmax) {
              const float *x = w, *y = w + tf;
              // (measured alternatives, both slower at the kernel's 96-register budget: four independent partial sums 54.1 -> 59.5 ms;
              // an explicit double FMA -- exact here, float products are exact in double -- with the PCM loads unrolled 55.0 -> 58.8 ms)
              double Sxy = 0.0;
#pragma unroll 4
              for (int i = 0; i < tf; i++) Sxy += (double)x[i] * (double)y[i];
              const double N = (double)tf, Sy = P2a - Sx, Syy = P2b - Sxx;
              cc[tf - tmin] = (Sxy - Sx * Sy / N) / (sqrt(Sxx - Sx * Sx / N) * sqrt(Syy - Sy * Sy / N));
            }
            PA1 += __shfl_sync(kFull, s1, 31); PA2 += __shfl_sync(kFull, s2, 31);
            PB1 += __shfl_sync(kFull, q1, 31); PB2 += __shfl_sync(kFull, q2, 31);
          }
        }
#endif
        __syncwarp();
        int maxI = -1;                                                         // :743-754 (first of the highest peaks)
        {
          double bd = 0.0;
          for (int i = 1 + lane; i < nLag - 2; i += 32)
            if (cc[i - 1] < cc[i] && cc[i] > cc[i + 1] && (maxI < 0 || cc[i] > bd)) { bd = cc[i]; maxI = i; }
          // reduce on the double value: ties keep the lower index
#pragma unroll
          for (int d = 16; d > 0; d >>= 1) {
            const double od = __shfl_xor_sync(kFull, bd, d);
            const int oi = __shfl_xor_sync(kFull, maxI, d);
            if (oi >= 0 && (maxI < 0 || od > bd || (od == bd && oi < maxI))) { bd = od; maxI = oi; }
          }
        }
        pp = maxI == -1 ? t0f : tmin + maxI;
        const int os = start;
        if (maxI >= 0) {
          start += pp;
          float max0, min0, max1, min1; int mI0, mI1;
          double pk0 = 0.0, pk1 = 0.0;
          float a0, a1, ad;
          if (p.shimmerUseRms) {                                               // :461-513 (sequential float sums, every lane alike)
            const float *x = wav + os, *y = wav + start;
            int i, mI = 1; float mxv = x[1];
            float rmsX = x[0] * x[0];
            for (i = 1; i < pp - 1; i++) { if (x[i] > mxv) { mxv = x[i]; mI = i; } rmsX += x[i] * x[i]; }
            rmsX = sqrtf((rmsX + x[i] * x[i]) / (float)pp);
            pk0 = quad3((double)(mI - 1), x[mI - 1], (double)mI, x[mI], (double)(mI + 1), x[mI + 1], nullptr, nullptr);
            mI = 1; mxv = y[1];
            float rmsY = y[0] * y[0];
            for (i = 1; i < pp - 1; i++) { if (y[i] > mxv) { mxv = y[i]; mI = i; } rmsY += y[i] * y[i]; }
            rmsY = sqrtf((rmsY + y[i] * y[i]) / (float)pp);
            pk1 = quad3((double)(mI - 1), y[mI - 1], (double)mI, y[mI], (double)(mI + 1), y[mI + 1], nullptr, nullptr);
            a0 = rmsX; a1 = rmsY; ad = fabsf(rmsX - rmsY);
          } else {                                                             // :418-456
            jit_extrema(wav + os, pp, lane, max0, mI0, min0);
            jit_extrema(wav + start, pp, lane, max1, mI1, min1);
            if (p.peakToPeak) {
              const float *x = wav + os, *y = wav + start;
              pk0 = quad3((double)(mI0 - 1), x[mI0 - 1], (double)mI0, x[mI0], (double)(mI0 + 1), x[mI0 + 1], nullptr, nullptr);
              pk1 = quad3((double)(mI1 - 1), y[mI1 - 1], (double)mI1, y[mI1], (double)(mI1 + 1), y[mI1 + 1], nullptr, nullptr);
            }
            a0 = max0 - min0; a1 = max1 - min1;
            ad = (float)fabs((double)((max0 - min0) - (max1 - min1)));
          }
          if (lane == 0) pb[numPeriods] = os;
          numPeriods++;
          for (int i = lane; i < t0f; i += 32) avgWf[i] += wav[os + i];
          double conf = 0.0, ccI = 0.0;
          const double maxId = fabs(((double)tmin + quad3((double)(maxI - 1), cc[maxI - 1], (double)maxI, cc[maxI],
                                                          (double)(maxI + 1), cc[maxI + 1], &ccI, &conf))) * Ts;
          sumCC += (float)ccI;
          if (minCC == -2.0f || minCC > (float)ccI) minCC = (float)ccI;
          if (maxCC == -2.0f || maxCC < (float)ccI) maxCC = (float)ccI;
          if (p.brokenThresh) threshCC = minCC;                                // :811-816
          if (ccI > threshCC) {
            float period;
            if (p.peakToPeak) period = (float)(((double)start + pk1 - (double)os - pk0) * Ts);
            else period = (float)maxId;
            avgPeriod += period;
            nPeriods += 1.0f;
            if (lastT0 > 0.0) {
              const float diff = fabsf(lastT0 - period);
              JitterLocal += diff;
              nPeriodsLocal += 1.0f;
              if (lastDiff > 0.0) { JitterDDP += fabsf(lastDiff - diff); nPeriodsDDP += 1.0f; }
              lastDiff = diff;
            }
            lastT0 = period;
            avgAmp += (a0 + a1) / 2.0f;
            avgAmpDiff += ad;
          }
        } else {
          start += t0f;
        }
        if (start < toRead0 - 1) lastPeriod = start;                           // :856-858
        __syncwarp();
      }
      if (lane == 0) { pb[numPeriods] = start; if (pp > 0) pb[numPeriods + 1] = start + pp; }
      numPeriods++;
      for (int i = lane; i < t0f && start + i < nT; i += 32) {                 // :865-870
        avgWf[i] += wav[start + i];
        avgWf[i] /= (float)numPeriods;
      }
      __syncwarp();
      float Eh = 0.0f;
      for (int i = 3; i < t0f - 2 && start + i < nT; i++) Eh += avgWf[i] * avgWf[i];
      if (t0f - 4 > 0) Eh /= (float)(t0f - 4);
      Eh = sqrtf(Eh);
      float En = 0.0f; int nEn = 0;
      for (int i = 0; i < numPeriods; i++) {                                   // :882-889
        int n = 2;
        const int hiJ = min(pb[i + 1], pb[i] + t0f);
        for (int j = pb[i] + 2; j < hiJ - 2; j++) {
          const float delta = wav[j] - avgWf[n++];
          En += delta * delta;
          nEn++;
        }
      }
      if (nEn > 0) En /= (float)nEn;
      En = sqrtf(En);
      eH = Eh; eN = En;
      if (En > 0.0) {
        HNR = Eh / En;
        if (HNR > 0.0) lgHNR = (float)(20.0 * log((double)HNR) / log(10.0));
        else lgHNR = p.lgHNRfloor;
      }
      if (numPeriods > 0) sumCC /= (float)numPeriods;
      lastMis = toRead0 - lastPeriod;
    } else {                                                                   // :918-943
      lastPeriod = toRead0; lastMis = 0;
      lastT0 = 0.0f; lastDiff = 0.0f; lastJitterDDP = 0.0f; lastJitterLocal = 0.0f; lastShimmerLocal = 0.0f;
      if (p.noiseERMS || p.linearHNR || p.logHNR) {
        // energy of an unvoiced frame: float products summed in double (lld/pitchJitter.cpp:930-936).  The lanes take strided
        // partial sums (a regrouping of double additions of exact float values: ~1e-16 relative, gone in the float result)
        // instead of every lane walking all nT samples
        double E = 0.0;
        for (int i = lane; i < nT; i += 32) E += wav[i] * wav[i];
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) E += __shfl_xor_sync(kFull, E, d);
        E /= (double)nT;
        eH = 0.0f; HNR = 0.0f; eN = (float)sqrt(E); lgHNR = p.lgHNRfloor;
      }
    }
    lastIdx += lastPeriod;
    // output vector (:950-1080)
    int n = 0;
    float ov[16];
    const bool okL = nPeriods > 0.0 && nPeriodsLocal > 0.0 && F0 > 0.0;
    if (okL) { JitterLocal /= nPeriodsLocal; lastJitterLocal_b = lastJitterLocal = JitterLocal / (avgPeriod / nPeriods); }
    if (p.jitterLocal) {
      if (okL || (nPeriods == 0.0 && F0 > 0.0)) { if (lastJitterLocal > 1.0) lastJitterLocal = 1.0f; ov[n] = lastJitterLocal; }
      else ov[n] = 0.0f;
      n++;
    }
    if (p.jitterLocalEnv) { if (lastJitterLocal_b > 1.0) lastJitterLocal_b = 1.0f; ov[n++] = lastJitterLocal_b; }
    const bool okD = nPeriods > 0.0 && nPeriodsDDP > 0.0 && F0 > 0.0;
    if (okD) { JitterDDP /= nPeriodsDDP; lastJitterDDP_b = lastJitterDDP = JitterDDP / (avgPeriod / nPeriods); }
    if (p.jitterDDP) {
      if (okD || (nPeriods == 0.0 && F0 > 0.0)) { if (lastJitterDDP > 1.0) lastJitterDDP = 1.0f; ov[n] = lastJitterDDP; }
      else ov[n] = 0.0f;
      n++;
    }
    if (p.jitterDDPEnv) { if (lastJitterDDP_b > 1.0) lastJitterDDP_b = 1.0f; ov[n++] = lastJitterDDP_b; }
    if (nPeriods > 0.0 && F0 > 0.0) {
      if (avgAmp > 0.0) lastShimmerLocal_b = lastShimmerLocal = (avgAmpDiff / avgAmp);
      else lastShimmerLocal = 0.0f;
    }
    if (p.shimmerLocal || p.shimmerLocalDB) {
      if (F0 > 0.0) {
        if (lastShimmerLocal > 1.0) lastShimmerLocal = 1.0f;
        if (p.shimmerLocal) ov[n++] = lastShimmerLocal;
        if (p.shimmerLocalDB) { const double a = lastShimmerLocal + 1.0; ov[n++] = (float)(a > 10e-50 ? 20.0 * log(a) / log(10.0) : -1000.0); }
      } else {
        if (p.shimmerLocal) ov[n++] = 0.0f;
        if (p.shimmerLocalDB) ov[n++] = 0.0f;
      }
    }
    if (p.shimmerLocalEnv) { if (lastShimmerLocal_b > 1.0) lastShimmerLocal_b = 1.0f; ov[n++] = lastShimmerLocal_b; }
    if (p.harmonicERMS) ov[n++] = eH;
    if (p.noiseERMS) ov[n++] = eN;
    if (p.linearHNR) ov[n++] = HNR;
    if (p.logHNR) { if (lgHNR < p.lgHNRfloor) lgHNR = p.lgHNRfloor; ov[n++] = lgHNR; }
    if (p.refinedF0) ov[n++] = (nPeriods > 0.0 && F0 > 0.0) ? 1.0f / (avgPeriod / nPeriods) : 0.0f;
    if (p.srcQualMean) ov[n++] = sumCC;
    if (p.srcQualRange) ov[n++] = fabsf(maxCC - minCC);
    if (lane == 0) for (int k = 0; k < n; k++) o[k] = ov[k];
  }
}

// ------------------------------------------------------------------------------------------ seq_post_kernel

struct SeqCtx { const float *x; int stride; int T; int V; };

// cContourSmoother (smaWin = 3) value of row m, column c (dspcore/contourSmoother.cpp:84-117) with the
// end-of-input behaviour of a reader over [pitch level ; jitter level]: rows V-1 and V are produced during the
// reference's first EOI pass, when the jitter level (lagKind 2) still ends at its row V-1
__device__ float seq_sma(const SeqCtx &c, const SeqGroup &G, int k, int m)
{
  const int col = G.srcCol + k, lagKind = G.lagKind, noZero = G.noZero;
  const bool lagged = lagKind == 2 && c.V >= 1 && (m == c.V - 1 || m == c.V);   // V == 0: nothing runs in the first pass
  auto g = [&](int i) -> float {
    i = min(max(i, 0), c.T - 1);
    if (lagged && i > c.V - 1) i = c.V - 1;
    if (G.gateCol >= 0) {                                                         // other/valbasedSelector.cpp:195-233
      const float sel = c.x[(size_t)i * c.stride + G.gateCol];
      const bool pass = ((G.gateFlags & 1) ? sel < G.gateThr : sel > G.gateThr) || ((G.gateFlags & 2) && sel == G.gateThr);
      if (!pass) return G.gateOut;
    }
    return c.x[(size_t)i * c.stride + col];
  };
  const float x0 = g(m);
  if (noZero) {
    if (x0 == 0.0f) return 0.0f;
    float y = x0; int N = 1;
    const float a = g(m - 1), b = g(m + 1);
    if (a != 0.0f) { y += a; N++; }
    if (b != 0.0f) { y += b; N++; }
    return y / (float)N;
  }
  float y = x0;
  y += g(m - 1);
  y += g(m + 1);
  return y / 3.0f;
}

constexpr int kSeqWarps = 4, kMaxSegCols = 32;

// one warp per utterance, lane = row of a 32-row chunk
__global__ void __launch_bounds__(kSeqWarps * 32) seq_post_kernel(const SeqPostParams p, int u0, int u1)
{
  const int lane = threadIdx.x & 31;
  const int u = u0 + blockIdx.x * kSeqWarps + (threadIdx.x >> 5);
  if (u >= u1) return;
  SeqCtx c;
  c.T = (int)frame_count(p.uttOff[u + 1] - p.uttOff[u], p.frameSize, p.frameStep, p.frameCenter);
  if (c.T <= 0) return;
  c.V = p.lag[u];
  c.x = p.stat + (size_t)p.statOff[u] * p.statStride;
  c.stride = p.statStride;
  const long long R = p.rowOff[u + 1] - p.rowOff[u];
  float *out = p.out + (size_t)p.rowOff[u] * p.outStride;
  const int T = c.T, V = c.V;
  // 1. smoothed levels
  for (int g = 0; g < p.nGroups; g++) {
    const SeqGroup &G = p.groups[g];
    if (G.nStages != 1) continue;
    for (int m = lane; m <= T && m < R; m += 32)
      for (int k = 0; k < G.n; k++) out[(size_t)m * p.outStride + G.outCol + k] = seq_sma(c, G, k, m);
  }
  // 2. deltas with onlyInSegments: one running norm per delta component (dspcore/deltaRegression.cpp:77-79,123-141),
  //    rows in order, elements in column order: norm(n, k) = 2*sum i^2 + (i^2 of every accepted pair before and
  //    including element (n, k)) -- integers, exact in float below 2^24 -- so the running sum is a prefix sum.
  //    Rows V-1..V+2 are produced during the reference's first EOI pass, when the smoothed level ends at its row V;
  //    row V+3 (for T-5 <= V <= T-2) in the first tick of the second pass, when it ends at row T-1
  //    (core/dataMemoryLevel.cpp:1020-1027,1698-1708).
  for (int seg = 0; seg < kMaxSegIds; seg++) {
    int W = 0;
    for (int g = 0; g < p.nGroups; g++) if (p.groups[g].nStages == 2 && p.groups[g].segId == seg) W = p.groups[g].deltaWin;
    if (W == 0) continue;
    int normInit = 0;
    for (int i = 1; i <= W; i++) normInit += i * i;
    normInit *= 2;
    int base = 0;
    for (int n0 = 0; n0 <= T + W; n0 += 32) {
      const int n = n0 + lane;
      const bool live = n <= T + W;
      int last = T;
      if (V >= 1 && n >= V - 1 && n <= V + 2) last = min(T, V);
      else if (n == V + 3 && V >= T - 5 && V <= T - 2) last = T - 1;
      float num[kMaxSegCols];
      int cnt[kMaxSegCols];
      int col = 0, rowTot = 0;
      for (int g = 0; g < p.nGroups; g++) {
        const SeqGroup &G = p.groups[g];
        if (G.nStages != 2 || G.segId != seg) continue;
        for (int k = 0; k < G.n && col < kMaxSegCols; k++, col++) {
          float nm = 0.0f; int ct = 0;
          if (live) {
            for (int i = 1; i <= W; i++) {
              const float a = seq_sma(c, G, k, min(max(n - i, 0), last));
              const float b = seq_sma(c, G, k, min(max(n + i, 0), last));
              if (!(a == 0.0f || a != a || b == 0.0f || b != b)) { nm += (float)i * (b - a); ct += i * i; }
            }
          }
          num[col] = nm; cnt[col] = ct; rowTot += ct;
        }
      }
      int incl = rowTot;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) { const int o = __shfl_up_sync(kFull, incl, d); if (lane >= d) incl += o; }
      int running = base + incl - rowTot;
      base += __shfl_sync(kFull, incl, 31);
      col = 0;
      for (int g = 0; g < p.nGroups; g++) {
        const SeqGroup &G = p.groups[g];
        if (G.nStages != 2 || G.segId != seg) continue;
        for (int k = 0; k < G.n && col < kMaxSegCols; k++, col++) {
          running += cnt[col];
          if (live && n < R) out[(size_t)n * p.outStride + G.outCol + k] = num[col] / (float)(normInit + running);
        }
      }
    }
  }
}

}  // namespace

cudaError_t launch_shs(const ShsParams &p, cudaStream_t st)
{
  if (p.nTiles <= 0) return cudaSuccess;
  const size_t perWarp = ((size_t)2 * (p.nMag + 2) * sizeof(double) + (size_t)p.nPts * sizeof(float) + 128 + 15) & ~(size_t)15;
  int warps = kShsWarps;
  while (warps > 1 && (perWarp * warps + 1024) * 3 > 227 * 1024) warps--;   // three CTAs per SM (7 warps each for 513 bins)
  if ((size_t)p.nPts * sizeof(float) > (size_t)(p.nMag + 2) * sizeof(double)) return cudaErrorInvalidValue;   // SS must fit the buffer it reuses
  const size_t smem = perWarp * warps;
  if (smem > 220 * 1024) return cudaErrorInvalidValue;
  cudaError_t e = cudaFuncSetAttribute(shs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  shs_kernel<<<p.nTiles, warps * 32, smem, st>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_viterbi(const ViterbiParams &p, int u0, int u1, cudaStream_t st)
{
  if (u1 <= u0) return cudaSuccess;
  if (p.nCand + 1 > kVitStates || p.bufLen > kVitBuf) return cudaErrorInvalidValue;
  viterbi_kernel<<<(u1 - u0 + 63) / 64, 64, 0, st>>>(p, u0, u1);
  return cudaGetLastError();
}

cudaError_t launch_jitter(const JitterParams &p, int u0, int u1, cudaStream_t st)
{
  if (u1 <= u0) return cudaSuccess;
  const size_t perWarp = (size_t)p.capCC * sizeof(double) + (size_t)(p.capWav + p.capAvg) * sizeof(float) + (size_t)p.capPb * sizeof(int);
  const size_t smem = perWarp * kJitWarps;
  if (smem > 200 * 1024) return cudaErrorInvalidValue;
  auto kern = p.pcmF32 ? jitter_kernel<true> : jitter_kernel<false>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  kern<<<(u1 - u0 + kJitWarps - 1) / kJitWarps, kJitWarps * 32, smem, st>>>(p, u0, u1);
  return cudaGetLastError();
}

cudaError_t launch_seq_post(const SeqPostParams &p, int u0, int u1, cudaStream_t st)
{
  if (u1 <= u0 || p.nGroups <= 0) return cudaSuccess;
  seq_post_kernel<<<(u1 - u0 + kSeqWarps - 1) / kSeqWarps, kSeqWarps * 32, 0, st>>>(p, u0, u1);
  return cudaGetLastError();
}

}  // namespace osm
