// functionals.cu -- cFunctionals in full-input mode on the GPU (include/osm_b200_functionals.h, SURVEY.md 8f-3).
//
// One warp per contour = (utterance, LLD element).  The contour is streamed from the row-major LLD matrix in chunks of 32
// frames (lane = frame); the reference's nonZeroFuncts filter (functionals.cpp:286-299) becomes an order-preserving warp
// compaction on the fly (ballot + prefix popcount give every kept value its index in the filtered contour, which the position
// and regression functionals need).  Two passes:
//   pass 1  count, sum, min / max with first positions, the power / sign / log sums of cFunctionalMeans, the moment sums
//           sum x i, sum x i^2 of cFunctionalRegression; the filtered contour is copied to shared memory when percentiles are
//           enabled
//   seq     the order-dependent functionals (functionals_seq.cuh) read the shared copy: cFunctionalTimes counts in parallel,
//           cFunctionalLpc with one lane per autocorrelation lag (the reference's sequential float sums), cFunctionalPeaks2
//           collects the local extrema in parallel (ordered compaction) and prunes them on lane 0, cFunctionalSegments runs
//           its state machine on lane 0
//   pass 2  central moments about the float mean (functionalMoments.cpp:96-108) and the regression residuals
//           (functionalRegression.cpp:263-290), which need the results of pass 1
// then a warp-wide bitonic sort of the shared copy for cFunctionalPercentiles (the reference sorts with std::sort,
// functionals.cpp:296-299), and lane 0 assembles the values in the reference's order.
// Contours longer than kMaxShort rows (long_contours.hpp) run the same statements with the copy in a work space slice in HBM, and
// their percentiles come from a radix rank selection (pctl_select_kernel, rank_select.cuh) instead of a sort.
// All accumulators are double like the reference's; the reference adds sequentially, a warp adds 32 strided partial sums and
// combines them by shuffles -- a reordering of double additions, 1e-16 relative, invisible in the float results.
// Compiled with -fmad=false (the float expressions of the percentile interpolation keep their two roundings).
#include <cuda_runtime.h>
#include <algorithm>
#include <math.h>
#include <string.h>

#include <memory>
#include <string>
#include <vector>

#include "../../include/osm_b200_functionals.h"
#include "cuda_owned.hpp"
#include "functionals_seq.cuh"
#include "long_contours.hpp"
#include "plan.hpp"
#include "rank_select.cuh"

namespace osm {
namespace {

constexpr int kFnWarps = 4;
constexpr int kFnThreads = kFnWarps * 32;
constexpr int kSelThreads = 512;

struct FnParams {
  const float *rows; int rowStride; int nIn;
  const int *cols;                          // device [nIn] column of every input element inside a row, or null (0 .. nIn-1)
  long long outStride;                      // floats between the output rows of consecutive utterances
  const long long *rowOff, *nRows;          // device [nUtt]
  float *out; int nVals;                    // out[u][e * nVals + v]
  int sortCap;                              // floats of the contour copy per warp in shared memory (0: not needed)
  int perWarp;                              // floats per warp in shared memory: contour copy + extrema list + segment lengths
  int listOff, lensOff;                     // float offsets of the Peaks2 list / Segments lengths inside a warp's block
  int valOff[OSM_B200_F_MAX_ENABLED];       // first value of every enabled functional inside a contour's output
  int timesNorm, segNorm, peaksNorm; int onsetNorm, peaksOldNorm;
  float period; double periodD;             // input level period as FLOAT_DMEM and as double
  osm_b200_functionals_spec s;
  int extNorm, meanNorm;                    // resolved time normalisations
  int needReg, enQreg;
  LongContour *lc; int nLong;               // long path: this chunk's contours, one slice of wsStride floats each in ws
  float *ws; long long wsStride;
};

__device__ __forceinline__ double wsum(double v)
{
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ long long wsumll(long long v)
{
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

struct Keep {
  int mode;
  __device__ __forceinline__ bool operator()(float x) const { return mode == 0 || (mode == 2 ? x > 0.0f : x != 0.0f); }
};

// getInterpPctl (functionalPercentiles.cpp:317-336)
__device__ float interp_pctl(double p, const float *s, long long N)
{
  const double idx = p * (double)(N - 1);
  long long i1 = (long long)floor(idx), i2 = (long long)ceil(idx);
  i1 = i1 < 0 ? 0 : (i1 >= N ? N - 1 : i1);
  i2 = i2 < 0 ? 0 : (i2 >= N ? N - 1 : i2);
  if (i1 != i2) {
    const double w1 = idx - (double)i1, w2 = (double)i2 - idx;
    return __fadd_rn(__fmul_rn(s[i1], (float)w2), __fmul_rn(s[i2], (float)w1));
  }
  return s[i1];
}
__device__ float index_pctl(double p, const float *s, long long N)          // getPctlIdx (:309-315): C round()
{
  long long r = (long long)round(p * (double)(N - 1));
  r = r < 0 ? 0 : (r >= N ? N - 1 : r);
  return s[r];
}

// kLong = false: one warp per (utterance, element) of the grid, the contour copy in shared memory (contours of at most kMaxShort
// rows).  kLong = true: one warp per contour of p.lc, the copy in that contour's work space slice in global memory (sortCap /
// listOff / lensOff describe the chunk's slice); the percentiles are left to pctl_select_kernel, which reads the same copy.  The
// statements are the same in both.
template <bool kLong>
__global__ void __launch_bounds__(kFnThreads) functionals_kernel(const FnParams p)
{
  extern __shared__ float fnSort[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nW = blockDim.x >> 5;                                   // 1 .. kFnWarps: fewer when long contours need the shared memory
  const int groups = (p.nIn + nW - 1) / nW;
  const int c = blockIdx.x * nW + warp;                             // long path: this warp's contour
  if (kLong && c >= p.nLong) return;
  const int u = kLong ? p.lc[c].u : blockIdx.x / groups, e = kLong ? p.lc[c].e : (blockIdx.x % groups) * nW + warp;
  if (e >= p.nIn) return;
  const long long T = p.nRows[u];
  const float *col = p.rows + p.rowOff[u] * (long long)p.rowStride + (p.cols ? p.cols[e] : e);
  float *out = p.out + (long long)u * p.outStride + (long long)e * p.nVals;
  // the long path's slice: segment lengths / lag buffer | contour copy | extrema list, so that lensOff = -lensFloats and every
  // offset from sbuf stays below 2^31 floats
  float *sbuf = kLong ? p.ws + (long long)c * p.wsStride - p.lensOff : fnSort + (size_t)warp * p.perWarp;
  const Keep keep{p.s.nonZeroFuncts};
  const unsigned ltMask = (1u << lane) - 1u;

  // ---------------- pass 1 ----------------
  long long cnt = 0;
  double sum = 0, sAbs = 0, sSq = 0, sLog = 0, sPos = 0, sNeg = 0, sPosSq = 0, sNegSq = 0, sNz = 0, sNzAbs = 0, sNzSq = 0;
  double num = 0, num2 = 0, numAbs = 0;
  long long nPos = 0, nNeg = 0, nNz = 0;
  float mn = INFINITY, mx = -INFINITY;
  long long mnI = 0x7fffffffffffffffLL, mxI = 0x7fffffffffffffffLL;
  for (long long t0 = 0; t0 < T; t0 += 32) {
    const long long t = t0 + lane;
    const float x = t < T ? col[t * p.rowStride] : 0.0f;
    const bool k = t < T && keep(x);
    const unsigned m = __ballot_sync(0xffffffffu, k);
    if (k) {
      const long long i = cnt + __popc(m & ltMask);
      const double xd = (double)x, fa = fabs(xd), ii = (double)i;
      sum += xd; sAbs += fa;
      if (x < mn) { mn = x; mnI = i; }
      if (x > mx) { mx = x; mxI = i; }
      if (x > 0.0f) { sPos += xd; sPosSq += xd * xd; nPos++; }
      if (x < 0.0f) { sNeg += xd; sNegSq += xd * xd; nNeg++; }
      if (x != 0.0f) { sNz += xd; sNzAbs += fa; sNzSq += xd * xd; sLog += log(fa); nNz++; sSq += xd * xd; }
      double tmp = xd * ii;
      num += tmp; num2 += tmp * ii;
      numAbs += fa * ii;
      if (p.sortCap > 0 && i < p.sortCap) sbuf[i] = x;
    }
    cnt += __popc(m);
  }
  const long long N = cnt;                 // uniform
  if (kLong && lane == 0) p.lc[c].n = (int)N;
  if (N == 0) {                            // every sub-component returns nothing: zero fill (functionals.cpp:316-320)
    for (int v = lane; v < p.nVals; v += 32) out[v] = 0.0f;
    return;
  }
  sum = wsum(sum); sAbs = wsum(sAbs); sSq = wsum(sSq); sLog = wsum(sLog); sPos = wsum(sPos); sNeg = wsum(sNeg);
  sPosSq = wsum(sPosSq); sNegSq = wsum(sNegSq); sNz = wsum(sNz); sNzAbs = wsum(sNzAbs); sNzSq = wsum(sNzSq);
  num = wsum(num); num2 = wsum(num2); numAbs = wsum(numAbs);
  nPos = wsumll(nPos); nNeg = wsumll(nNeg); nNz = wsumll(nNz);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {       // extremes with the first position (functionalExtremes.cpp:96-101)
    const float omn = __shfl_xor_sync(0xffffffffu, mn, o), omx = __shfl_xor_sync(0xffffffffu, mx, o);
    const long long omnI = __shfl_xor_sync(0xffffffffu, mnI, o), omxI = __shfl_xor_sync(0xffffffffu, mxI, o);
    if (omn < mn || (omn == mn && omnI < mnI)) { mn = omn; mnI = omnI; }
    if (omx > mx || (omx == mx && omxI < mxI)) { mx = omx; mxI = omxI; }
  }
  const double Nd = (double)N;
  const float mean = (float)(sum / Nd);    // functionals.cpp:300-306, handed on as FLOAT_DMEM
  const double meanD = (double)mean;

  // ---------------- regression coefficients (functionalRegression.cpp:150-262) ----------------
  const auto &R = p.s.regression;
  double rm = 0, rt = 0, ra = 0, rb = 0, rc = 0, rinv = 0, centroid = 0;
  const double asum = meanD * Nd;
  if (p.needReg) {
    const double range = (double)__fsub_rn(mx, mn);         // max - min is a FLOAT_DMEM expression (:151)
    rinv = range > 0.0 ? 1.0 / range : 0.0;
    if (R.centroidUseAbsValues) centroid = sAbs != 0.0 ? numAbs / sAbs : 0.0;
    else centroid = asum != 0.0 ? num / asum : 0.0;
    if (R.centroidRatioLimit) centroid = (double)fseq::ratio_limit((float)centroid, (float)Nd, (float)Nd);   // :206-209
    if (R.centroidNorm == OSM_B200_TIMENORM_SECOND) centroid *= p.periodD;
    else if (R.centroidNorm == OSM_B200_TIMENORM_SEGMENT) centroid /= Nd;
    if (N > 1) {
      const double NNm1 = Nd * (Nd - 1.0);
      const double S1 = NNm1 / 2.0, S2 = NNm1 * (2.0 * Nd - 1.0) / 6.0;
      const double S1dS2 = S1 / S2;
      const double tmp = Nd - S1 * S1dS2;
      rt = tmp == 0.0 ? 0.0 : (asum - num * S1dS2) / tmp;
      rm = (num - rt * S1) / S2;
      const double S3 = S1 * S1, Nind1 = Nd - 1.0;
      const double S4 = S2 * (3.0 * (Nind1 * Nind1 + Nind1) - 1.0) / 5.0;
      if (p.enQreg) {
        const double S3S3 = S3 * S3, S2S2 = S2 * S2, S1S2 = S1 * S2, S1S1 = S3;
        const double det = S4 * S2 * Nd + 2.0 * S3 * S1S2 - S2S2 * S2 - S3S3 * Nd - S1S1 * S4;
        if (det != 0.0) {
          ra = ((S2 * Nd - S1S1) * num2 + (S1S2 - S3 * Nd) * num + (S3 * S1 - S2S2) * asum) / det;
          rb = ((S1S2 - S3 * Nd) * num2 + (S4 * Nd - S2S2) * num + (S3 * S2 - S4 * S1) * asum) / det;
          rc = ((S3 * S1 - S2S2) * num2 + (S3 * S2 - S4 * S1) * num + (S4 * S2 - S3S3) * asum) / det;
        }
      }
    } else {
      // a contour of one value: m = 0, t = c = that value
      float x0 = 0.0f;
      for (long long t = 0; t < T; t++) { const float x = col[t * p.rowStride]; if (keep(x)) { x0 = x; break; } }
      rm = 0.0; rt = rc = (double)x0;
    }
  }

  // ---------------- order-dependent functionals on the copy of the filtered contour ----------------
  __syncwarp();
  for (int fi = 0; fi < p.s.n_enabled; fi++) {
    float *o = out + p.valOff[fi];
    const int kind = p.s.enabled[fi];
    if (kind == OSM_B200_F_TIMES) {                                   // functionalTimes.cpp:245-371
      const auto &Tm = p.s.times;
      const float Nind = (float)N;
      float Norm = Nind, Norm1 = Nind - 1.0f, Norm2 = Nind - 2.0f, Tp = 1.0f;
      if (p.timesNorm == OSM_B200_TIMENORM_SECOND) {
        Tp = p.period;
        if (Tp != 0.0f) {
          if (Tm.buggySecNorm) { Norm = Norm / Tp; Norm1 = Norm1 / Tp; Norm2 = Norm2 / Tp; }
          else { Norm = 1.0f / Tp; Norm1 = Norm1 / (Nind * Tp); Norm2 = Norm2 / (Nind * Tp); }
        }
      }
      if (p.timesNorm == OSM_B200_TIMENORM_FRAME) { Norm = 1.0f; Norm1 = Norm1 / Nind; Norm2 = Norm2 / Nind; }
      const float range = mx - mn;
      const float l25 = 0.25f * range + mn, l50 = 0.50f * range + mn, l75 = 0.75f * range + mn, l90 = 0.90f * range + mn;
      long long n25 = 0, n50 = 0, n75 = 0, n90 = 0, nR = 0, nF = 0, nLC = 0, nRC = 0;
      for (long long i = lane; i < N; i += 32) {
        const float x = sbuf[i];
        n25 += x <= l25; n50 += x <= l50; n75 += x <= l75; n90 += x <= l90;
        if (i >= 1) {
          const float xp = sbuf[i - 1];
          nR += xp < x; nF += xp > x;
          if (i + 1 < N) {
            const float a1 = x - xp, a2 = sbuf[i + 1] - x;
            nRC += a2 < a1; nLC += a1 < a2;
          }
        }
      }
      n25 = wsumll(n25); n50 = wsumll(n50); n75 = wsumll(n75); n90 = wsumll(n90);
      nR = wsumll(nR); nF = wsumll(nF); nLC = wsumll(nLC); nRC = wsumll(nRC);
      if (lane == 0) {
        int n = 0;
        if (Tm.upleveltime25) o[n++] = (float)(N - n25) / Norm;
        if (Tm.downleveltime25) o[n++] = (float)n25 / Norm;
        if (Tm.upleveltime50) o[n++] = (float)(N - n50) / Norm;
        if (Tm.downleveltime50) o[n++] = (float)n50 / Norm;
        if (Tm.upleveltime75) o[n++] = (float)(N - n75) / Norm;
        if (Tm.downleveltime75) o[n++] = (float)n75 / Norm;
        if (Tm.upleveltime90) o[n++] = (float)(N - n90) / Norm;
        if (Tm.downleveltime90) o[n++] = (float)n90 / Norm;
        if (Tm.risetime) o[n++] = Norm1 != 0.0f ? (float)nR / Norm1 : 0.0f;
        if (Tm.falltime) o[n++] = Norm1 != 0.0f ? (float)nF / Norm1 : 0.0f;
        if (Tm.leftctime) o[n++] = Norm2 != 0.0f ? (float)nLC / Norm2 : 0.0f;
        if (Tm.rightctime) o[n++] = Norm2 != 0.0f ? (float)nRC / Norm2 : 0.0f;
        if (Tm.duration) o[n++] = p.timesNorm == OSM_B200_TIMENORM_SECOND ? (float)N * Tp : (float)N;
      }
    } else if (kind == OSM_B200_F_LPC) {                              // functionalLpc.cpp:98-125
      const int order = p.s.lpc.order;
      float *acf = sbuf + p.lensOff;                                   // the segment-length scratch doubles as the lag buffer
      if (lane <= order) {                                            // smileDsp_autoCorr (smileUtil.c:1560-1569): sequential float sum per lag
        float acc = 0.0f;
        for (long long i = lane; i < N; i++) acc = acc + sbuf[i] * sbuf[i - lane];
        acf[lane] = acc;
      }
      __syncwarp();
      if (lane == 0) fseq::lpc(p.s.lpc, acf, (long)N, o);
      __syncwarp();
    } else if (kind == OSM_B200_F_PEAKS2) {                           // functionalPeaks2.cpp:320-327 in parallel, then :330-915 on lane 0
      float *ly = sbuf + p.listOff;
      int *lx = reinterpret_cast<int *>(ly + p.sortCap);              // up to N - 4 extrema (a zigzag)
      int nl = 0;
      for (long long i0 = 2; i0 < N - 2; i0 += 32) {
        const long long i = i0 + lane;
        int type = -1;
        float x = 0.0f;
        if (i < N - 2) {
          x = sbuf[i];
          const float a = sbuf[i - 1], b = sbuf[i + 1];
          if (x > a && x > b) type = 1;
          else if (x < a && x < b) type = 0;
        }
        const unsigned m = __ballot_sync(0xffffffffu, type >= 0);
        if (type >= 0) { const int k = nl + __popc(m & ltMask); ly[k] = x; lx[k] = (int)(i << 1) | type; }
        nl += __popc(m);
      }
      __syncwarp();
      if (lane == 0) fseq::peaks2(p.s.peaks2, sbuf, (long)N, mn, mx, mean, p.period, p.peaksNorm, ly, lx, nl, o);
      __syncwarp();
    } else if (kind == OSM_B200_F_SEGMENTS) {
      if (lane == 0) fseq::segments(p.s.segments, sbuf, (long)N, mn, mx, p.period, p.segNorm, sbuf + p.lensOff, o);
      __syncwarp();
    } else if (kind == OSM_B200_F_ONSET) {                            // state machines / float running sums in frame order: lane 0
      if (lane == 0) fseq::onset(p.s.onset, sbuf, (long)N, p.period, p.onsetNorm, o);
      __syncwarp();
    } else if (kind == OSM_B200_F_PEAKS) {
      if (lane == 0) fseq::peaks(p.s.peaks, sbuf, (long)N, p.period, p.peaksOldNorm, reinterpret_cast<int *>(sbuf + p.listOff), o);
      __syncwarp();
    } else if (kind == OSM_B200_F_CROSSINGS) {
      if (lane == 0) fseq::crossings(p.s.crossings, sbuf, (long)N, o);
      __syncwarp();
    } else if (kind == OSM_B200_F_SAMPLES) {
      if (lane == 0) fseq::samples(p.s.samples, sbuf, (long)N, o);
      __syncwarp();
    } else if (kind == OSM_B200_F_DCT) {                              // one coefficient per lane, each a sequential float sum over the contour
      for (int k = p.s.dct.firstCoeff + lane; k <= p.s.dct.lastCoeff; k += 32) o[k - p.s.dct.firstCoeff] = fseq::dct_coeff(sbuf, (long)N, k);
      __syncwarp();
    }
  }

  // ---------------- pass 2 ----------------
  double m2 = 0, m3 = 0, m4 = 0, lea = 0, leq = 0, qea = 0, qeq = 0;
  cnt = 0;
  for (long long t0 = 0; t0 < T; t0 += 32) {
    const long long t = t0 + lane;
    const float x = t < T ? col[t * p.rowStride] : 0.0f;
    const bool k = t < T && keep(x);
    const unsigned m = __ballot_sync(0xffffffffu, k);
    if (k) {
      const double xd = (double)x, ii = (double)(cnt + __popc(m & ltMask));
      const double d = xd - meanD;
      double d2 = d * d;
      m2 += d2; d2 *= d; m3 += d2; m4 += d2 * d;
      if (p.needReg) {
        double er = xd - (rm * ii + rt);
        if (R.normInputs) er *= rinv;
        lea += fabs(er); leq += er * er;
        if (p.enQreg) {
          double eq = xd - (ra * ii * ii + rb * ii + rc);
          if (R.normInputs) eq *= rinv;
          qea += fabs(eq); qeq += eq * eq;
        }
      }
    }
    cnt += __popc(m);
  }
  m2 = wsum(m2); m3 = wsum(m3); m4 = wsum(m4);
  lea = wsum(lea); leq = wsum(leq); qea = wsum(qea); qeq = wsum(qeq);

  // ---------------- sorted copy for the percentiles ----------------
  bool needSort = false;
  for (int i = 0; i < p.s.n_enabled; i++) needSort = needSort || p.s.enabled[i] == OSM_B200_F_PERCENTILES;
  if (!kLong && needSort) {
    int n2 = 32;
    while (n2 < N) n2 <<= 1;
    __syncwarp();
    for (int i = (int)N + lane; i < n2; i += 32) sbuf[i] = INFINITY;
    __syncwarp();
    for (int k = 2; k <= n2; k <<= 1)
      for (int j = k >> 1; j > 0; j >>= 1) {
        for (int i = lane; i < n2; i += 32) {
          const int q = i ^ j;
          if (q > i) {
            const float a = sbuf[i], b = sbuf[q];
            const bool up = (i & k) == 0;
            if ((a > b) == up) { sbuf[i] = b; sbuf[q] = a; }
          }
        }
        __syncwarp();
      }
  }
  if (lane != 0) return;

  // ---------------- values, in the order of functionalsEnabled ----------------
  for (int fi = 0; fi < p.s.n_enabled; fi++) {
    int n = p.valOff[fi];
    switch (p.s.enabled[fi]) {
      case OSM_B200_F_EXTREMES: {
        const auto &E = p.s.extremes;
        float maxpos = (float)mxI, minpos = (float)mnI;
        if (p.extNorm == OSM_B200_TIMENORM_SEGMENT) { maxpos = __fdiv_rn(maxpos, (float)N); minpos = __fdiv_rn(minpos, (float)N); }
        else if (p.extNorm == OSM_B200_TIMENORM_SECOND && p.period != 0.0f) { maxpos = __fmul_rn(maxpos, p.period); minpos = __fmul_rn(minpos, p.period); }
        if (E.max) out[n++] = mx;
        if (E.min) out[n++] = mn;
        if (E.range) out[n++] = __fsub_rn(mx, mn);
        if (E.maxpos) out[n++] = maxpos;
        if (E.minpos) out[n++] = minpos;
        if (E.amean) out[n++] = mean;
        if (E.maxameandist) out[n++] = __fsub_rn(mx, mean);
        if (E.minameandist) out[n++] = __fsub_rn(mean, mn);
      } break;
      case OSM_B200_F_MEANS: {
        const auto &M = p.s.means;
        const double absmean = sAbs / Nd, qmean = sSq / Nd;
        double nzamean = 0, nzabsmean = 0, nzqmean = 0, nzgmean = 0;
        if (nNz > 0) { const double d = (double)nNz; nzamean = sNz / d; nzabsmean = sNzAbs / d; nzqmean = sNzSq / d; nzgmean = exp(sLog / d); }
        const double posamean = nPos > 0 ? sPos / (double)nPos : 0.0, posqmean = nPos > 0 ? sPosSq / (double)nPos : 0.0;
        const double negamean = nNeg > 0 ? sNeg / (double)nNeg : 0.0, negqmean = nNeg > 0 ? sNegSq / (double)nNeg : 0.0;
        if (M.amean) out[n++] = mean;
        if (M.absmean) out[n++] = (float)absmean;
        if (M.qmean) out[n++] = (float)qmean;
        if (M.nzamean) out[n++] = (float)nzamean;
        if (M.nzabsmean) out[n++] = (float)nzabsmean;
        if (M.nzqmean) out[n++] = (float)nzqmean;
        if (M.nzgmean) out[n++] = (float)nzgmean;
        if (M.nnz) {
          const float c = (float)nNz;
          out[n++] = p.meanNorm == OSM_B200_TIMENORM_FRAME ? c : (p.meanNorm == OSM_B200_TIMENORM_SEGMENT ? __fdiv_rn(c, (float)N) : __fdiv_rn(c, p.period));
        }
        if (M.flatness) out[n++] = absmean != 0.0 ? (float)(nzgmean / absmean) : 1.0f;
        if (M.posamean) out[n++] = (float)posamean;
        if (M.negamean) out[n++] = (float)negamean;
        if (M.posqmean) out[n++] = (float)posqmean;
        if (M.posrqmean) out[n++] = (float)sqrt(posqmean);
        if (M.negqmean) out[n++] = (float)negqmean;
        if (M.negrqmean) out[n++] = (float)sqrt(negqmean);
        if (M.rqmean) out[n++] = (float)sqrt(qmean);
        if (M.nzrqmean) out[n++] = (float)sqrt(nzqmean);
      } break;
      case OSM_B200_F_MOMENTS: {
        const auto &M = p.s.moments;
        const double v2 = m2 / Nd, sq = sqrt(v2);
        if (M.variance) out[n++] = (float)v2;
        if (M.stddev) out[n++] = v2 > 0.0 ? (float)sq : 0.0f;
        if (M.skewness) out[n++] = v2 > 0.0 ? (float)(m3 / (Nd * v2 * sq)) : 0.0f;
        if (M.kurtosis) out[n++] = v2 > 0.0 ? (float)(m4 / (Nd * v2 * v2)) : 0.0f;
        if (M.amean) out[n++] = mean;
        if (M.stddevNorm == 1 || M.stddevNorm == 2) {
          if (v2 > 0.0) {
            double ml = M.stddevNorm == 1 ? (double)fabsf(mean) : meanD;
            if (M.doRatioLimit) {                                      // functionalMoments.cpp:144-151
              out[n++] = ml != 0.0 ? fseq::ratio_limit((float)(sq / ml), 10.0f, 20.0f) : 20.0f;
            } else {
              if (ml == 0.0) ml = 1.0;
              out[n++] = (float)(sq / ml);
            }
          } else out[n++] = 0.0f;
        }
      } break;
      case OSM_B200_F_PERCENTILES: {
        if (kLong) break;                                              // pctl_select_kernel
        const auto &P = p.s.percentiles;
        const float q1 = P.interp ? interp_pctl(0.25, sbuf, N) : index_pctl(0.25, sbuf, N);
        const float q2 = P.interp ? interp_pctl(0.50, sbuf, N) : index_pctl(0.50, sbuf, N);
        const float q3 = P.interp ? interp_pctl(0.75, sbuf, N) : index_pctl(0.75, sbuf, N);
        if (P.quartile1) out[n++] = q1;
        if (P.quartile2) out[n++] = q2;
        if (P.quartile3) out[n++] = q3;
        if (P.iqr12) out[n++] = __fsub_rn(q2, q1);
        if (P.iqr23) out[n++] = __fsub_rn(q3, q2);
        if (P.iqr13) out[n++] = __fsub_rn(q3, q1);
        const int n0 = n;
        for (int i = 0; i < P.n_percentile; i++) out[n++] = P.interp ? interp_pctl(P.percentile[i], sbuf, N) : index_pctl(P.percentile[i], sbuf, N);
        for (int i = 0; i < P.n_pctlrange; i++) out[n++] = fabsf(__fsub_rn(out[n0 + P.pctlrange[i][1]], out[n0 + P.pctlrange[i][0]]));
      } break;
      case OSM_B200_F_REGRESSION: {
        double m = rm, t = rt, a = ra, b = rb, c = rc;
        if (R.doRatioLimit) {                                          // functionalRegression.cpp:328-335
          double rg = (double)__fsub_rn(mx, mn);
          if (rg <= 0.0) rg = 1.0;
          m = (double)fseq::ratio_limit((float)m, (float)(rg / 10.0), (float)(rg / 10.0 + 0.01));
          a = (double)fseq::ratio_limit((float)a, (float)sqrt(rg / 10.0), (float)(sqrt(rg / 10.0) + 0.01));
          b = (double)fseq::ratio_limit((float)b, (float)(rg / 10.0), (float)(rg / 10.0 + 0.01));
        }
        if (R.normRegCoeff == 1) { m *= Nd - 1.0; a *= (Nd - 1.0) * (Nd - 1.0); b *= Nd - 1.0; }
        else if (R.normRegCoeff == 2) { const double one = 1.0 / p.periodD; m *= one; a *= one * one; b *= one; }
        if (R.normInputs) { m *= rinv; t = (t - (double)mn) * rinv; a *= rinv; b *= rinv; c = (c - (double)mn) * rinv; }
        auto fin = [](double v) { return isfinite(v) ? v : 0.0; };
        if (R.linregc1) out[n++] = (float)fin(m);
        if (R.linregc2) out[n++] = (float)fin(t);
        if (R.linregerrA) out[n++] = (float)(isfinite(lea / Nd) ? lea / Nd : 0.0);
        if (R.linregerrQ) out[n++] = (float)(isfinite(leq / Nd) ? leq / Nd : 0.0);
        if (R.qregc1) out[n++] = (float)fin(a);
        if (R.qregc2) out[n++] = (float)fin(b);
        if (R.qregc3) out[n++] = (float)fin(c);
        const double qa = isfinite(qea / Nd) ? qea : 0.0, qq = isfinite(qeq / Nd) ? qeq : 0.0;
        if (R.qregerrA) out[n++] = (float)(R.oldBuggyQerr ? qa : qa / Nd);
        if (R.qregerrQ) out[n++] = (float)(R.oldBuggyQerr ? qq : qq / Nd);
        if (R.centroid) out[n++] = (float)fin(centroid);
      } break;
    }
  }
}

// cFunctionalPercentiles of the long path: one CTA per contour of the chunk finds every rank the percentile block reads in one
// MSB-first radix walk over the contour's copy (rank_select.cuh) and writes the block.  Walkers whose prefixes agree share a histogram.
struct SelParams {
  const LongContour *lc; const float *ws; long long wsStride; int copyOff;
  float *out; long long outStride; int nVals, valOff;
  decltype(osm_b200_functionals_spec::percentiles) P;
};

__global__ void __launch_bounds__(kSelThreads) pctl_select_kernel(const __grid_constant__ SelParams p)
{
  __shared__ unsigned hist[rsel::kMaxRanks][rsel::kDigits];
  __shared__ long long rank[rsel::kMaxRanks], rem[rsel::kMaxRanks];
  __shared__ uint32_t pre[rsel::kMaxRanks];
  __shared__ int lead[rsel::kMaxRanks];
  const LongContour &d = p.lc[blockIdx.x];
  const long long N = d.n;
  if (N == 0) return;                                                // functionals_kernel wrote the zero fill
  const float *x = p.ws + (long long)blockIdx.x * p.wsStride + p.copyOff;
  const int t = threadIdx.x, nr = 2 * (3 + p.P.n_percentile);
  if (t == 0) rsel::pctl_walkers(p.P, N, rank);
  __syncthreads();
  if (t < nr) { rem[t] = rank[t]; pre[t] = 0; }
  for (int shift = 24; shift >= 0; shift -= 8) {
    __syncthreads();
    if (t < nr) { int l = 0; while (pre[l] != pre[t]) l++; lead[t] = l; }
    for (int i = t; i < nr * rsel::kDigits; i += blockDim.x) hist[i / rsel::kDigits][i % rsel::kDigits] = 0u;
    __syncthreads();
    for (long long i = t; i < N; i += blockDim.x) {
      const uint32_t k = rsel::key(x[i]), hi = rsel::prefix(k, shift);
      for (int w = 0; w < nr; w++)
        if (lead[w] == w && pre[w] == hi) { atomicAdd(&hist[w][rsel::digit(k, shift)], 1u); break; }
    }
    __syncthreads();
    uint32_t next = 0;
    if (t < nr) { long long r = rem[t]; next = (pre[t] << 8) | (uint32_t)rsel::digit_of_rank(hist[lead[t]], r); rem[t] = r; }
    __syncthreads();
    if (t < nr) pre[t] = next;
  }
  __syncthreads();
  if (t == 0) {
    float sel[rsel::kMaxRanks];
    for (int w = 0; w < nr; w++) sel[w] = rsel::value(pre[w]);
    rsel::pctl_block(p.P, N, rank, sel, p.out + (long long)d.u * p.outStride + (long long)d.e * p.nVals + p.valOff);
  }
}

int resolve_norm(int own, int ownSet, int master)            // functionalComponent.hpp:67-76
{
  if (ownSet) return own;
  return master != OSM_B200_TIMENORM_UNSET ? master : own;
}

// summary glue: gather + cVectorOperation dBp / dBv (other/vectorOperation.cpp:508-527)
struct AssembleParams {
  const float *in; float *out;
  long long inStride, outStride, nRows;
  int nOut;
  short src[OSM_B200_SUMMARY_MAX_OUT];
  unsigned char op[OSM_B200_SUMMARY_MAX_OUT];
  float floorv[OSM_B200_SUMMARY_MAX_OUT];
};

__global__ void __launch_bounds__(128) summary_assemble_kernel(const __grid_constant__ AssembleParams p)
{
  const long long total = p.nRows * p.nOut;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / p.nOut;
    const int k = (int)(i - r * p.nOut);
    float x = p.in[r * p.inStride + p.src[k]];
    const int op = p.op[k];
    if (op != OSM_B200_VOP_COPY) {
      const float factor = op == OSM_B200_VOP_DBP ? (float)(10.0 / 2.302585092994046) : (float)(20.0 / 2.302585092994046);
      const float fl = p.floorv[k];
      x = factor * logf(x > fl ? x : fl);
    }
    p.out[r * p.outStride + k] = x;
  }
}

}  // namespace
}  // namespace osm

using namespace osm;

struct osm_b200_functionals {
  osm_b200_functionals_spec spec;
  int nIn = 0, nVals = 0, device = -1;
  double period = 0;
  std::vector<std::string> names;
  bool hasPct = false, hasSeq = false, hasPeaks = false, hasSeg = false;
  DevBuf<long long> dMeta;
  DevBuf<float> dIn, dOut;                     // run_host staging: one float more than the largest batch so far
  DevBuf<int> dCols; std::vector<int> hCols;
  DevBuf<float> dWs;                           // long contours: work space, at most kLongWsCapFloats unless one contour needs more
  DevBuf<LongContour> dLong; std::vector<LongContour> longs; std::vector<LongChunk> chunks;

  ~osm_b200_functionals() { if (device >= 0) cudaSetDevice(device); }
};

namespace {

std::vector<std::string> value_names(const osm_b200_functionals_spec &s)
{
  std::vector<std::string> v;
  char buf[64];
  for (int i = 0; i < s.n_enabled; i++) {
    switch (s.enabled[i]) {
      case OSM_B200_F_EXTREMES: {
        const auto &E = s.extremes;
        const int on[8] = {E.max, E.min, E.range, E.maxpos, E.minpos, E.amean, E.maxameandist, E.minameandist};
        const char *nm[8] = {"max", "min", "range", "maxPos", "minPos", "amean", "maxameandist", "minameandist"};   // functionalExtremes.cpp:37
        for (int k = 0; k < 8; k++) if (on[k]) v.push_back(nm[k]);
      } break;
      case OSM_B200_F_MEANS: {
        const auto &M = s.means;
        const int on[17] = {M.amean, M.absmean, M.qmean, M.nzamean, M.nzabsmean, M.nzqmean, M.nzgmean, M.nnz, M.flatness, M.posamean, M.negamean,
                            M.posqmean, M.posrqmean, M.negqmean, M.negrqmean, M.rqmean, M.nzrqmean};
        const char *nm[17] = {"amean", "absmean", "qmean", "nzamean", "nzabsmean", "nzqmean", "nzgmean", "nnz", "flatness", "posamean", "negamean",
                              "posqmean", "posrqmean", "negqmean", "negrqmean", "rqmean", "nzrqmean"};                  // functionalMeans.cpp:45
        for (int k = 0; k < 17; k++) if (on[k]) v.push_back(nm[k]);
      } break;
      case OSM_B200_F_MOMENTS: {
        const auto &M = s.moments;
        if (M.variance) v.push_back("variance");
        if (M.stddev) v.push_back("stddev");
        if (M.skewness) v.push_back("skewness");
        if (M.kurtosis) v.push_back("kurtosis");
        if (M.amean) v.push_back("amean");
        if (M.stddevNorm == 2) v.push_back("stddevNorm");
        else if (M.stddevNorm == 1) v.push_back("coeffOfVariation");                                                    // functionalMoments.cpp:34
      } break;
      case OSM_B200_F_PERCENTILES: {
        const auto &P = s.percentiles;
        if (P.quartile1) v.push_back("quartile1");
        if (P.quartile2) v.push_back("quartile2");
        if (P.quartile3) v.push_back("quartile3");
        if (P.iqr12) v.push_back("iqr1-2");
        if (P.iqr23) v.push_back("iqr2-3");
        if (P.iqr13) v.push_back("iqr1-3");
        for (int k = 0; k < P.n_percentile; k++) { snprintf(buf, sizeof buf, "percentile%.1f", P.percentile[k] * 100.0); v.push_back(buf); }   // :268-290
        for (int k = 0; k < P.n_pctlrange; k++) { snprintf(buf, sizeof buf, "pctlrange%i-%i", P.pctlrange[k][0], P.pctlrange[k][1]); v.push_back(buf); }
      } break;
      case OSM_B200_F_REGRESSION: {
        const auto &R = s.regression;
        const int on[10] = {R.linregc1, R.linregc2, R.linregerrA, R.linregerrQ, R.qregc1, R.qregc2, R.qregc3, R.qregerrA, R.qregerrQ, R.centroid};
        const char *nm[10] = {"linregc1", "linregc2", "linregerrA", "linregerrQ", "qregc1", "qregc2", "qregc3", "qregerrA", "qregerrQ", "centroid"};
        for (int k = 0; k < 10; k++) if (on[k]) v.push_back(nm[k]);
      } break;
      case OSM_B200_F_TIMES: {
        const auto &T = s.times;
        const int on[13] = {T.upleveltime25, T.downleveltime25, T.upleveltime50, T.downleveltime50, T.upleveltime75, T.downleveltime75,
                            T.upleveltime90, T.downleveltime90, T.risetime, T.falltime, T.leftctime, T.rightctime, T.duration};
        const char *nm[13] = {"upleveltime25", "downleveltime25", "upleveltime50", "downleveltime50", "upleveltime75", "downleveltime75",
                              "upleveltime90", "downleveltime90", "risetime", "falltime", "leftctime", "rightctime", "duration"};   // functionalTimes.cpp:39
        for (int k = 0; k < 13; k++) if (on[k]) v.push_back(nm[k]);
      } break;
      case OSM_B200_F_LPC: {                                                                                            // functionalLpc.cpp:84-96
        if (s.lpc.lpGain) v.push_back("lpgain");
        if (s.lpc.lpc) for (int k = s.lpc.firstCoeff; k < s.lpc.order; k++) { snprintf(buf, sizeof buf, "lpc%i", k); v.push_back(buf); }
      } break;
      case OSM_B200_F_SEGMENTS: {
        const auto &G = s.segments;
        const int on[5] = {G.numSegments, G.meanSegLen, G.maxSegLen, G.minSegLen, G.segLenStddev};
        const char *nm[5] = {"numSegments", "meanSegLen", "maxSegLen", "minSegLen", "segLenStddev"};                    // functionalSegments.cpp:39
        for (int k = 0; k < 5; k++) if (on[k]) v.push_back(nm[k]);
      } break;
      case OSM_B200_F_PEAKS2: {
        const char *nm[OSM_B200_F_PEAKS2_VALUES] = {"numPeaks", "meanPeakDist", "meanPeakDistDelta", "peakDistStddev", "peakRangeAbs", "peakRangeRel",
            "peakMeanAbs", "peakMeanMeanDist", "peakMeanRel", "ptpAmpMeanAbs", "ptpAmpMeanRel", "ptpAmpStddevAbs", "ptpAmpStddevRel", "minRangeAbs",
            "minRangeRel", "minMeanAbs", "minMeanMeanDist", "minMeanRel", "mtmAmpMeanAbs", "mtmAmpMeanRel", "mtmAmpStddevAbs", "mtmAmpStddevRel",
            "meanRisingSlope", "maxRisingSlope", "minRisingSlope", "stddevRisingSlope", "meanFallingSlope", "maxFallingSlope", "minFallingSlope",
            "stddevFallingSlope", "covFallingSlope", "covRisingSlope"};                                                  // functionalPeaks2.cpp:58-66
        for (int k = 0; k < OSM_B200_F_PEAKS2_VALUES; k++) if (s.peaks2.value[k]) v.push_back(nm[k]);
      } break;
      case OSM_B200_F_ONSET: {                                                                                          // functionalOnset.cpp:29
        const auto &O = s.onset;
        const int on[5] = {O.onsetPos, O.offsetPos, O.numOnsets, O.numOffsets, O.onsetRate};
        const char *nm[5] = {"onsetPos", "offsetPos", "numOnsets", "numOffsets", "onsetRate"};
        for (int k = 0; k < 5; k++) if (on[k]) v.push_back(nm[k]);
      } break;
      case OSM_B200_F_PEAKS: {                                                                                          // functionalPeaks.cpp:29
        const auto &K = s.peaks;
        const int on[5] = {K.numPeaks, K.meanPeakDist, K.peakMean, K.peakMeanMeanDist, K.peakDistStddev};
        const char *nm[5] = {"numPeaks", "meanPeakDist", "peakMean", "peakMeanMeanDist", "peakDistStddev"};
        for (int k = 0; k < 5; k++) if (on[k]) v.push_back(nm[k]);
      } break;
      case OSM_B200_F_CROSSINGS: {                                                                                      // functionalCrossings.cpp:26
        if (s.crossings.zcr) v.push_back("zcr");
        if (s.crossings.mcr) v.push_back("mcr");
        if (s.crossings.amean) v.push_back("amean");
      } break;
      case OSM_B200_F_SAMPLES: {                                                                                        // functionalSamples.cpp:89-95
        for (int k = 0; k < s.samples.n_samplepos; k++) { snprintf(buf, sizeof buf, "samples%.3f", s.samples.samplepos[k]); v.push_back(buf); }
      } break;
      case OSM_B200_F_DCT: {                                                                                            // functionalDCT.cpp:103-110
        for (int k = s.dct.firstCoeff; k <= s.dct.lastCoeff; k++) { snprintf(buf, sizeof buf, "dct%i", k); v.push_back(buf); }
      } break;
    }
  }
  return v;
}

// number of values functional `fi` of the enabled list contributes
int value_count(const osm_b200_functionals_spec &s, int fi)
{
  osm_b200_functionals_spec one = s;
  one.n_enabled = 1; one.enabled[0] = s.enabled[fi];
  return (int)value_names(one).size();
}

}  // namespace

extern "C" {

int32_t osm_b200_functionals_sizeof_spec(void) { return (int32_t)sizeof(osm_b200_functionals_spec); }

void osm_b200_functionals_defaults(osm_b200_functionals_spec *s)
{
  if (!s) return;
  memset(s, 0, sizeof *s);
  s->masterTimeNorm = OSM_B200_TIMENORM_UNSET;
  auto &E = s->extremes;
  E.max = E.min = E.range = E.maxpos = E.minpos = E.maxameandist = E.minameandist = 1; E.amean = 0; E.norm = OSM_B200_TIMENORM_FRAME;
  auto &M = s->means;
  M.amean = M.absmean = M.qmean = M.nzamean = M.nzabsmean = M.nzqmean = M.nzgmean = M.nnz = 1; M.norm = OSM_B200_TIMENORM_FRAME;
  auto &Q = s->moments;
  Q.variance = Q.stddev = Q.skewness = Q.kurtosis = 1;
  s->percentiles.interp = 1;
  auto &R = s->regression;
  R.linregc1 = R.linregc2 = R.linregerrA = R.linregerrQ = R.qregc1 = R.qregc2 = R.qregc3 = R.qregerrA = R.qregerrQ = R.centroid = 1;
  R.centroidNorm = OSM_B200_TIMENORM_SEGMENT; R.centroidUseAbsValues = 1; R.centroidRatioLimit = 1; R.oldBuggyQerr = 1;
  auto &T = s->times;                                             // functionalTimes.cpp:60-78
  T.upleveltime25 = T.downleveltime25 = T.upleveltime50 = T.downleveltime50 = T.upleveltime75 = T.downleveltime75 = T.upleveltime90 =
      T.downleveltime90 = T.risetime = T.falltime = T.leftctime = T.rightctime = T.duration = 1;
  T.buggySecNorm = 1; T.norm = OSM_B200_TIMENORM_SEGMENT;
  s->lpc.lpc = 1; s->lpc.order = 5;                                // functionalLpc.cpp:38-41
  auto &G = s->segments;                                          // functionalSegments.cpp:48-73
  G.maxNumSeg = 20; G.segMinLng = 3; G.pauseMinLng = 2; G.norm = OSM_B200_TIMENORM_SEGMENT; G.algorithm = OSM_B200_SEG_RELTH;
  auto &K = s->peaks2;                                            // functionalPeaks2.cpp:84-130
  K.relThresh = 0.1f; K.doRatioLimit = 1; K.norm = OSM_B200_TIMENORM_FRAME;
  s->onset.numOnsets = 1; s->onset.norm = OSM_B200_TIMENORM_SEGMENT;                                    // functionalOnset.cpp:43-54
  auto &QP = s->peaks;                                            // functionalPeaks.cpp:45-53
  QP.numPeaks = QP.meanPeakDist = QP.peakMean = QP.peakMeanMeanDist = 1; QP.norm = OSM_B200_TIMENORM_FRAME;
  s->crossings.zcr = s->crossings.mcr = 1;                        // functionalCrossings.cpp:42-46
  s->samples.n_samplepos = 5;                                     // functionalSamples.cpp:24,68-75
  for (int i = 0; i < 5; i++) s->samples.samplepos[i] = (double)i / (5 - 1.0);
  s->dct.firstCoeff = 1; s->dct.lastCoeff = 6;                    // functionalDCT.cpp:38-40
}

// no exception crosses the C boundary (host allocation failures while the names are built)
osm_b200_status osm_b200_functionals_create(const osm_b200_functionals_spec *spec, int32_t n_in, const char *const *in_names,
                                            double input_period, int32_t device, osm_b200_functionals **out)
try {
  if (!spec || !out || n_in <= 0 || !in_names) return set_last_error(OSM_B200_ERR_INVALID, "null argument");
  *out = nullptr;
  const auto &s = *spec;
  if (s.n_enabled <= 0 || s.n_enabled > OSM_B200_F_MAX_ENABLED) return set_last_error(OSM_B200_ERR_INVALID, "cFunctionals: functionalsEnabled is empty");
  for (int i = 0; i < s.n_enabled; i++)
    if (s.enabled[i] < 0 || s.enabled[i] >= OSM_B200_F_COUNT_) return set_last_error(OSM_B200_ERR_INVALID, "cFunctionals: unknown functional");
  if (s.nonZeroFuncts < 0 || s.nonZeroFuncts > 2) return set_last_error(OSM_B200_ERR_INVALID, "cFunctionals.nonZeroFuncts must be 0, 1 or 2");
  const auto &P = s.percentiles;
  if (P.n_percentile < 0 || P.n_percentile > OSM_B200_F_MAX_PCTL || P.n_pctlrange < 0 || P.n_pctlrange > OSM_B200_F_MAX_PCTL)
    return set_last_error(OSM_B200_ERR_UNSUPPORTED, "cFunctionalPercentiles: at most 8 percentiles / ranges");
  for (int i = 0; i < P.n_pctlrange; i++)
    if (P.pctlrange[i][0] < 0 || P.pctlrange[i][0] >= P.n_percentile || P.pctlrange[i][1] < 0 || P.pctlrange[i][1] >= P.n_percentile)
      return set_last_error(OSM_B200_ERR_INVALID, "cFunctionalPercentiles.pctlrange refers to a percentile that does not exist");
  for (int i = 0; i < s.n_enabled; i++) {
    if (s.enabled[i] == OSM_B200_F_LPC && (s.lpc.order < 1 || s.lpc.order > OSM_B200_F_MAX_LPC || s.lpc.firstCoeff < 0 || s.lpc.firstCoeff >= s.lpc.order))
      return set_last_error(OSM_B200_ERR_UNSUPPORTED, "cFunctionalLpc: 0 <= firstCoeff < order <= 16");
    if (s.enabled[i] == OSM_B200_F_SAMPLES && (s.samples.n_samplepos < 1 || s.samples.n_samplepos > OSM_B200_F_MAX_SAMPLES))
      return set_last_error(OSM_B200_ERR_UNSUPPORTED, "cFunctionalSamples: 1 .. 16 sample positions");
    if (s.enabled[i] == OSM_B200_F_DCT && (s.dct.firstCoeff < 0 || s.dct.lastCoeff < s.dct.firstCoeff || s.dct.lastCoeff - s.dct.firstCoeff + 1 > OSM_B200_F_MAX_DCT))
      return set_last_error(OSM_B200_ERR_UNSUPPORTED, "cFunctionalDCT: 0 <= firstCoeff <= lastCoeff, at most 32 coefficients");
    if (s.enabled[i] == OSM_B200_F_SEGMENTS) {
      const auto &G = s.segments;
      if (G.algorithm < OSM_B200_SEG_RELTH || G.algorithm > OSM_B200_SEG_NARELTH) return set_last_error(OSM_B200_ERR_UNSUPPORTED, "cFunctionalSegments: segmentationAlgorithm must be relTh, NArelTh, nonX or eqX");
      if (G.maxNumSeg < 1 || G.maxNumSeg > 4096) return set_last_error(OSM_B200_ERR_UNSUPPORTED, "cFunctionalSegments: 1 <= maxNumSeg <= 4096");
      if (G.n_thresholds < 0 || G.n_thresholds > OSM_B200_F_MAX_THRESH) return set_last_error(OSM_B200_ERR_UNSUPPORTED, "cFunctionalSegments: at most 8 thresholds");
    }
  }
  auto f = std::make_unique<osm_b200_functionals>();
  f->spec = s; f->nIn = n_in; f->period = input_period;
  const std::vector<std::string> vn = value_names(s);
  f->nVals = (int)vn.size();
  if (f->nVals == 0) return set_last_error(OSM_B200_ERR_INVALID, "cFunctionals: no value enabled");
  for (int e = 0; e < n_in; e++)
    for (const std::string &v : vn)                                    // functionals.cpp:222-228
      f->names.push_back(s.functNameAppend[0] ? std::string(in_names[e]) + "__" + s.functNameAppend + "_" + v : std::string(in_names[e]) + "_" + v);
  for (int i = 0; i < s.n_enabled; i++) {
    f->hasPct = f->hasPct || s.enabled[i] == OSM_B200_F_PERCENTILES;
    f->hasSeq = f->hasSeq || s.enabled[i] >= OSM_B200_F_TIMES;
    f->hasPeaks = f->hasPeaks || s.enabled[i] == OSM_B200_F_PEAKS2 || s.enabled[i] == OSM_B200_F_PEAKS;   // the extrema / distance list
    f->hasSeg = f->hasSeg || s.enabled[i] == OSM_B200_F_SEGMENTS;
  }
  if (device >= 0) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || device >= n) return set_last_error(OSM_B200_ERR_CUDA, "no usable CUDA device (this library has no CPU fallback)");
  }
  f->device = device;
  *out = f.release();
  return OSM_B200_OK;
} catch (const std::bad_alloc &) { return set_last_error(OSM_B200_ERR_NOMEM, "out of host memory"); }
catch (const std::exception &e) { return set_last_error(OSM_B200_ERR_INVALID, e.what()); }

void osm_b200_functionals_destroy(osm_b200_functionals *f)
{
  if (!f) return;
  delete f;
}

int32_t osm_b200_functionals_num_values(const osm_b200_functionals *f) { return f ? f->nVals : 0; }
int32_t osm_b200_functionals_num_elements(const osm_b200_functionals *f) { return f ? f->nVals * f->nIn : 0; }
const char *osm_b200_functionals_element_name(const osm_b200_functionals *f, int32_t idx)
{
  return (f && idx >= 0 && idx < (int)f->names.size()) ? f->names[idx].c_str() : nullptr;
}

osm_b200_status osm_b200_functionals_run_device(osm_b200_functionals *f, const float *d_rows, int32_t row_stride, const int64_t *row_offsets,
                                                const int64_t *n_rows, int32_t n_utt, float *d_out, void *stream)
{
  return osm_b200_functionals_run_device_cols(f, d_rows, row_stride, nullptr, row_offsets, n_rows, n_utt, d_out,
                                              f ? (int64_t)f->nVals * f->nIn : 0, stream);
}

osm_b200_status osm_b200_functionals_run_device_cols(osm_b200_functionals *f, const float *d_rows, int32_t row_stride, const int32_t *cols,
                                                     const int64_t *row_offsets, const int64_t *n_rows, int32_t n_utt, float *d_out,
                                                     int64_t out_stride, void *stream)
{
  if (!f || !row_offsets || !n_rows || n_utt < 0) return set_last_error(OSM_B200_ERR_INVALID, "null argument");
  if (f->device < 0) return set_last_error(OSM_B200_ERR_CUDA, "description-only functionals object (device < 0) cannot run; no CPU fallback");
  if (n_utt == 0) return OSM_B200_OK;
  if (!d_rows || !d_out || (!cols && row_stride < f->nIn) || out_stride < (int64_t)f->nVals * f->nIn) return set_last_error(OSM_B200_ERR_INVALID, "bad row buffer");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CU(cudaSetDevice(f->device));
  if (cols) {
    for (int e = 0; e < f->nIn; e++) if (cols[e] < 0 || cols[e] >= row_stride) return set_last_error(OSM_B200_ERR_INVALID, "column index outside the row");
    if (!f->dCols.p || f->hCols.size() != (size_t)f->nIn || memcmp(f->hCols.data(), cols, sizeof(int) * f->nIn) != 0) {
      CU(f->dCols.reserve_exact((size_t)f->nIn));
      f->hCols.assign(cols, cols + f->nIn);
      CU(cudaMemcpy(f->dCols.p, f->hCols.data(), sizeof(int) * (size_t)f->nIn, cudaMemcpyHostToDevice));
    }
  }
  // meta: row offsets | row counts of the shared-memory launch (0 for a long contour: that launch zero-fills its row, the long path
  // overwrites it later on the stream) | row counts
  const bool needCopy = f->hasPct || f->hasSeq;
  long long maxT = 0;
  int nLongUtt = 0;
  std::vector<long long> meta(3 * (size_t)n_utt);
  for (int u = 0; u < n_utt; u++) {
    if (n_rows[u] < 0 || row_offsets[u] < 0) return set_last_error(OSM_B200_ERR_INVALID, "negative row offset / count");
    if (needCopy && n_rows[u] >= kMaxLongRows)
      return set_last_error(OSM_B200_ERR_UNSUPPORTED, "cFunctionals (Percentiles, Times, Lpc, Segments, Peaks2): contours of 2^30 = 1073741824 frames or more are not supported (Peaks2 packs a frame index and a type bit into 32 bits)");
    const bool isLong = needCopy && n_rows[u] > kMaxShort;
    nLongUtt += isLong;
    meta[u] = row_offsets[u]; meta[n_utt + u] = isLong ? 0 : n_rows[u]; meta[2 * (size_t)n_utt + u] = n_rows[u];
    maxT = std::max<long long>(maxT, meta[n_utt + u]);
  }
  int sortCap = 0;
  if (needCopy) {
    sortCap = 32;
    while (sortCap < maxT) sortCap <<= 1;
  }
  // per-warp shared memory: contour copy | Peaks2 extrema (values, then positions) | segment lengths / lag buffer
  const int listFloats = f->hasPeaks ? 2 * sortCap : 0;
  const int lensFloats = f->hasSeq ? std::max(32, f->hasSeg ? f->spec.segments.maxNumSeg : 0) : 0;
  const int perWarp = sortCap + listFloats + lensFloats;
  int nWarps = kFnWarps;
  while (nWarps > 1 && (size_t)nWarps * perWarp * sizeof(float) > 200 * 1024) nWarps--;
  if ((size_t)nWarps * perWarp * sizeof(float) > 200 * 1024) return set_last_error(OSM_B200_ERR_UNSUPPORTED, "cFunctionals: contour too long for the shared-memory work space");
  CU(f->dMeta.reserve_exact(meta.size()));
  CU(cudaMemcpyAsync(f->dMeta.p, meta.data(), meta.size() * sizeof(long long), cudaMemcpyHostToDevice, st));
  if (nLongUtt > 0) {
    const long long wsFloats = plan_long_contours(n_rows, n_utt, f->nIn, f->hasPeaks ? 2 : 0, lensFloats, kLongWsCapFloats, f->longs, f->chunks);
    CU(f->dWs.reserve_exact((size_t)wsFloats));
    CU(f->dLong.reserve_exact(f->longs.size()));
    CU(cudaMemcpyAsync(f->dLong.p, f->longs.data(), f->longs.size() * sizeof(LongContour), cudaMemcpyHostToDevice, st));
  }
  CU(cudaStreamSynchronize(st));                  // `meta` is a local: the copy must have left the host buffer
  FnParams p;
  memset(&p, 0, sizeof p);
  p.cols = cols ? f->dCols.p : nullptr; p.outStride = out_stride;
  p.rows = d_rows; p.rowStride = row_stride; p.nIn = f->nIn; p.rowOff = f->dMeta.p; p.nRows = f->dMeta.p + n_utt;
  p.perWarp = perWarp; p.listOff = sortCap; p.lensOff = sortCap + listFloats;
  for (int i = 0, o = 0; i < f->spec.n_enabled; i++) { p.valOff[i] = o; o += value_count(f->spec, i); }
  p.timesNorm = resolve_norm(f->spec.times.norm, f->spec.times.normIsSet, f->spec.masterTimeNorm);
  p.segNorm = resolve_norm(f->spec.segments.norm, f->spec.segments.normIsSet, f->spec.masterTimeNorm);
  p.peaksNorm = resolve_norm(f->spec.peaks2.norm, f->spec.peaks2.normIsSet, f->spec.masterTimeNorm);
  p.onsetNorm = resolve_norm(f->spec.onset.norm, f->spec.onset.normIsSet, f->spec.masterTimeNorm);
  p.peaksOldNorm = resolve_norm(f->spec.peaks.norm, f->spec.peaks.normIsSet, f->spec.masterTimeNorm);
  p.out = d_out; p.nVals = f->nVals; p.sortCap = sortCap; p.period = (float)f->period; p.periodD = f->period; p.s = f->spec;
  p.extNorm = resolve_norm(f->spec.extremes.norm, f->spec.extremes.normIsSet, f->spec.masterTimeNorm);
  p.meanNorm = resolve_norm(f->spec.means.norm, f->spec.means.normIsSet, f->spec.masterTimeNorm);
  const auto &R = f->spec.regression;
  for (int i = 0; i < f->spec.n_enabled; i++) p.needReg = p.needReg || f->spec.enabled[i] == OSM_B200_F_REGRESSION;
  p.enQreg = R.qregc1 || R.qregc2 || R.qregc3 || R.qregerrA || R.qregerrQ || R.centroid;     // functionalRegression.cpp:108-117
  if (nLongUtt < n_utt) {
    const size_t smem = (size_t)nWarps * perWarp * sizeof(float);
    if (smem > 48 * 1024) CU(cudaFuncSetAttribute(functionals_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int groups = (f->nIn + nWarps - 1) / nWarps;
    functionals_kernel<false><<<(unsigned)((long long)n_utt * groups), nWarps * 32, smem, st>>>(p);
    CU(cudaGetLastError());
  }
  if (nLongUtt == 0) return OSM_B200_OK;
  // long contours, chunk by chunk through the one work space: a warp per contour (one per CTA, so that a chunk spreads over the
  // SMs), then a CTA per contour for the percentiles
  p.nRows = f->dMeta.p + 2 * (size_t)n_utt;
  p.ws = f->dWs.p;
  SelParams sp;
  memset(&sp, 0, sizeof sp);
  sp.ws = f->dWs.p; sp.copyOff = lensFloats; sp.out = d_out; sp.outStride = out_stride; sp.nVals = f->nVals; sp.P = f->spec.percentiles;
  for (int i = 0; i < f->spec.n_enabled; i++) if (f->spec.enabled[i] == OSM_B200_F_PERCENTILES) sp.valOff = p.valOff[i];
  for (const LongChunk &ch : f->chunks) {
    const int nC = ch.end - ch.begin;
    p.lc = f->dLong.p + ch.begin; p.nLong = nC;
    p.sortCap = ch.cap; p.listOff = ch.cap; p.lensOff = -lensFloats; p.wsStride = long_slice_floats(ch.cap, f->hasPeaks ? 2 : 0, lensFloats);
    functionals_kernel<true><<<(unsigned)nC, 32, 0, st>>>(p);
    CU(cudaGetLastError());
    if (f->hasPct) {
      sp.lc = p.lc; sp.wsStride = p.wsStride;
      pctl_select_kernel<<<(unsigned)nC, kSelThreads, 0, st>>>(sp);
      CU(cudaGetLastError());
    }
  }
  return OSM_B200_OK;
}

osm_b200_status osm_b200_summary_assemble_device(const float *d_in, int64_t in_stride, const int32_t *src, const int32_t *op, const float *log_floor,
                                                 int32_t n_out, int64_t n_rows, float *d_out, int64_t out_stride, void *stream)
{
  if (!d_in || !d_out || !src || n_out < 1 || n_rows < 0) return set_last_error(OSM_B200_ERR_INVALID, "summary_assemble: null argument");
  if (n_out > OSM_B200_SUMMARY_MAX_OUT) return set_last_error(OSM_B200_ERR_UNSUPPORTED, "summary_assemble: more than OSM_B200_SUMMARY_MAX_OUT output values");
  if (n_rows == 0) return OSM_B200_OK;
  AssembleParams p;
  p.in = d_in; p.out = d_out; p.inStride = in_stride; p.outStride = out_stride; p.nRows = n_rows; p.nOut = n_out;
  for (int k = 0; k < n_out; k++) {
    if (src[k] < 0 || src[k] >= in_stride || src[k] > 32767) return set_last_error(OSM_B200_ERR_INVALID, "summary_assemble: source index out of range");
    const int o = op ? op[k] : OSM_B200_VOP_COPY;
    if (o < OSM_B200_VOP_COPY || o > OSM_B200_VOP_DBV) return set_last_error(OSM_B200_ERR_INVALID, "summary_assemble: unknown operation");
    p.src[k] = (short)src[k]; p.op[k] = (unsigned char)o; p.floorv[k] = log_floor ? log_floor[k] : 1e-12f;
  }
  const long long total = n_rows * n_out;
  const int blocks = (int)std::min<long long>((total + 127) / 128, 148LL * 8);
  summary_assemble_kernel<<<blocks, 128, 0, (cudaStream_t)stream>>>(p);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_last_error(OSM_B200_ERR_CUDA, std::string("summary_assemble: ") + cudaGetErrorString(e));
  return OSM_B200_OK;
}

osm_b200_status osm_b200_functionals_run_host(osm_b200_functionals *f, const float *rows, int32_t row_stride, const int64_t *row_offsets,
                                              const int64_t *n_rows, int32_t n_utt, int64_t total_rows, float *out)
{
  if (!f || !rows || !out || total_rows < 0) return set_last_error(OSM_B200_ERR_INVALID, "null argument");
  if (f->device < 0) return set_last_error(OSM_B200_ERR_CUDA, "description-only functionals object (device < 0) cannot run; no CPU fallback");
  CU(cudaSetDevice(f->device));
  const size_t nIn = (size_t)total_rows * row_stride, nOut = (size_t)n_utt * f->nVals * f->nIn;
  CU(f->dIn.reserve_exact(nIn + 1));
  CU(f->dOut.reserve_exact(nOut + 1));
  CU(cudaMemcpy(f->dIn.p, rows, nIn * sizeof(float), cudaMemcpyHostToDevice));
  osm_b200_status st = osm_b200_functionals_run_device(f, f->dIn.p, row_stride, row_offsets, n_rows, n_utt, f->dOut.p, nullptr);
  if (st != OSM_B200_OK) return st;
  CU(cudaMemcpy(out, f->dOut.p, nOut * sizeof(float), cudaMemcpyDeviceToHost));
  return OSM_B200_OK;
}

}  // extern "C"
