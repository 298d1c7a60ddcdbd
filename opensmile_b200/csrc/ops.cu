// ops.cu -- standalone per-frame LLD kernels (lane = frame) for components that are not fused
// into lld_kernel: cSpectral on the magnitude level, cEnergy and cMZcr on the framer / windower
// level.  Each thread owns one frame and walks it in the reference's loop order with the
// reference's accumulator types (double sums), so results differ from the CPU only through the
// FFT that produced the magnitudes.  Citations relative to /root/reference/src.
#include "kernels.cuh"
#include "frame_reader.cuh"

namespace osm {

// ------------------------------------------------------------------------------------------
// cSpectral (lldcore/spectral.cpp:586-1555), magnitude input with a linear bin-frequency axis
// ------------------------------------------------------------------------------------------
constexpr int kSpecWarps = 8;                    // staging and the log spectrum use all of them, the descriptors the first four
constexpr int kSpecThreads = 32 * kSpecWarps;   // one CTA = one tile; lane = frame, warps split the descriptors

struct SpecView {
  const float *mag;     // magnitudes of this frame: bin k at mag[k * mstride] (shared-memory tile, stride 32,
                        // or -- when both tiles do not fit -- the global tile, stride F)
  const float *logS;    // shared-memory log spectrum of this frame, bin k at logS[k * 32] (or null)
  int mstride;
  int squareInput, useLog;
  __device__ __forceinline__ float m(int k) const { return mag[(size_t)k * mstride]; }
  __device__ __forceinline__ float M(int k) const   // srcM (:677-690)
  {
    const float v = m(k);
    return squareInput ? v : (v > 0.0f ? __fsqrt_rn(v) : 0.0f);
  }
  __device__ __forceinline__ float P(int k) const   // srcP (:692-703)
  {
    const float v = m(k);
    return squareInput ? __fmul_rn(v, v) : v;
  }
  __device__ __forceinline__ float L(int k) const { return logS[k * 32]; }
  __device__ __forceinline__ float LP(int k) const { return useLog ? L(k) : P(k); }
};

// The tile's magnitudes (and, when needed, its log spectrum) are staged in shared memory once;
// (by all eight warps); the descriptors are then distributed over the first four warps.  Every descriptor is still
// evaluated by ONE thread per frame in the reference's loop order and accumulator types; a warp
// that needs a shared prerequisite (frame sum, sum of the spectrum, centroid) recomputes it with the
// same loop, so the split does not change any result.
__global__ void __launch_bounds__(kSpecThreads) spectral_kernel(const SpectralParams p)
{
  extern __shared__ float ssm[];       // [nSrc][32] magnitudes | [nSrc][32] log spectrum (when reqLog) | [32] previous frame's column is read from global
  const OpTile tl = p.tiles[blockIdx.x];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool active = lane < tl.nf;
  const int F = p.F, Nsrc = p.nSrc;
  const int fl = active ? lane : 0;    // inactive lanes shadow frame 0 (results discarded)
  const bool staged = p.stageMag != 0;
  float *smag = ssm, *slog = ssm + (staged ? (size_t)Nsrc * 32 : 0);
  const float *gmag = p.mag + ((size_t)blockIdx.x * Nsrc) * F;
  if (staged) {
    for (int idx = tid; idx < Nsrc * 32; idx += kSpecThreads) {
      const int k = idx >> 5, ff = idx & 31;
      smag[idx] = gmag[(size_t)k * F + (ff < F ? ff : 0)];
    }
    __syncthreads();
  }
  SpecView v;
  v.mag = staged ? (smag + fl) : (gmag + fl);
  v.mstride = staged ? 32 : F;
  v.logS = slog + fl;
  v.squareInput = p.squareInput; v.useLog = p.useLog;
  const double F0 = p.F0;
  const int lo = p.loBin, hi = p.hiBin, nBins = hi - lo + 1;
  const float specFloor = p.specFloor;

  if (p.reqLog) {                                                      // :704-729
    float fac = (float)(10.0 / log(10.0));
    int src = 0;                                                        // 0 = P, 1 = M, 2 = raw
    if (p.reqPow) src = 0;
    else if (p.reqMag) src = 1;
    else src = 2;
    SpecView vl = v;     // inactive lanes compute the shadow column too: every slog column is defined
    for (int k = warp; k < Nsrc; k += kSpecWarps) {
      const float x = (src == 0) ? vl.P(k) : ((src == 1) ? vl.M(k) : vl.m(k));
      slog[k * 32 + lane] = (x <= specFloor) ? p.logSpecFloor : __fmul_rn(fac, logf(x));
    }
    __syncthreads();
  }

  float *dst = p.stat + (p.statOff[tl.utt] + tl.f0 + fl) * (long long)p.statStride + p.outCol;
  auto frq = [&](int k) { return F0 * (double)k; };
  // output columns, in the order of spectral.cpp:378-584
  int col = 0;
  const int cBands = col; col += p.nBands;
  const int cSlopes = col; col += p.nSlopes;
  const int cAlpha = col; col += p.alphaRatio ? 1 : 0;
  const int cHamm = col; col += p.hammarberg ? 1 : 0;
  const int cRoll = col; col += p.nRollOff;
  const int cFlux = col; col += p.flux ? 1 : 0;
  const int cCentroid = col; col += p.centroid ? 1 : 0;
  const int cMaxPos = col; col += p.maxPos ? 1 : 0;
  const int cMinPos = col; col += p.minPos ? 1 : 0;
  const int cEntropy = col; col += p.entropy ? 1 : 0;
  const int cStd = col; col += p.stddev ? 1 : 0;
  const int cVar = col; col += p.variance ? 1 : 0;
  const int cSkew = col; col += p.skewness ? 1 : 0;
  const int cKurt = col; col += p.kurtosis ? 1 : 0;
  const int cSlope = col; col += p.slope ? 1 : 0;
  const int cSharp = col; col += p.sharpness ? 1 : 0;
  const int cHarm = col; col += p.harmonicity ? 1 : 0;
  const int cFlat = col;
  auto put = [&](int c, float x) { if (active) dst[c] = x; };

  auto frame_sum = [&]() {                                              // :766-771
    double fs = 0.0;
    for (int i = lo; i <= hi; i++) fs += v.P(i);
    return fs;
  };
  auto sum_b = [&](double frameSum) {                                   // :1092-1099
    double sb = 0.0;
    if (p.normBand && !p.useLog) sb = frameSum;
    else for (int j = lo; j <= hi; j++) sb += (double)v.LP(j);
    return sb;
  };
  auto sum_a = [&]() {                                                  // :1257-1312
    double sa = 0.0;
    for (int j = lo; j <= hi; j++) sa += frq(j) * (double)v.LP(j);
    return sa;
  };

  if (warp == 0) {
    // ---- frame sum -> band energies, roll-off points, sharpness ----
    double frameSum = 0.0;
    if (p.normBand || p.sharpness || p.nRollOff > 0) frameSum = frame_sum();
    for (int b = 0; b < p.nBands; b++) {                                // :775-870
      const int iL = p.bandIL[b], iR = p.bandIR[b];
      double sum = (double)v.P(iL) * p.bandWL[b];
      for (int j = iL + 1; j < iR; j++) sum += (double)v.P(j);
      sum += (double)v.P(iR) * p.bandWR[b];
      if (p.normBand) put(cBands + b, frameSum > 0.0 ? (float)(sum / frameSum) : 0.0f);
      else if (nBins > 0) put(cBands + b, p.useLog ? (float)(10.0 * log(sum / (double)nBins) / log(10.0)) : (float)(sum / (double)nBins));
      else put(cBands + b, 0.0f);
    }
    if (p.nRollOff > 0) {                                               // :1103-1122
      double sumC = 0.0;
      float ro[16];
#pragma unroll
      for (int i = 0; i < 16; i++) ro[i] = 0.0f;
      for (int j = lo; j <= hi; j++) {
        sumC += (double)v.P(j);
#pragma unroll
        for (int i = 0; i < 16; i++) {
          if (i < p.nRollOff) {
            if (p.buggyRollOff == 1 && i > 0) sumC += (double)v.P(j);
            if ((ro[i] == 0.0f) && (sumC >= p.rollOff[i] * frameSum)) ro[i] = (float)frq(j);
          }
        }
      }
#pragma unroll
      for (int i = 0; i < 16; i++) if (i < p.nRollOff) put(cRoll + i, ro[i]);
    }
    if (p.sharpness) {                                                  // :1429-1478 (float accumulation)
      float sumAA = 0.0f, c2 = 0.0f;
      for (int j = lo; j <= hi && j < Nsrc; j++) sumAA = __fadd_rn(sumAA, (float)(p.sharpW[j - lo] * (double)v.P(j)));
      if (frameSum != 0.0) c2 = (float)((double)sumAA / frameSum);
      put(cSharp, (float)(0.11 * (double)c2));
    }
  } else if (warp == 1) {
    // ---- flux, entropy ----
    if (p.flux) {                                                       // :1125-1254
      const bool first = (tl.f0 + fl) == 0;
      if (first) put(cFlux, 0.0f);
      else {
        // previous frame: the neighbouring column of this tile, or the last column of the tile before
        const float *prev = (fl > 0) ? (v.mag - 1) : (p.mag + ((size_t)(blockIdx.x - 1) * Nsrc) * F + (F - 1));
        const int pstride = (fl > 0) ? v.mstride : F;
        double myA = 0.0;
        for (int j = lo; j <= hi; j++) {
          const float pm = prev[(size_t)j * pstride];
          const float pM = p.squareInput ? pm : (pm > 0.0f ? __fsqrt_rn(pm) : 0.0f);
          const double myB = ((double)v.M(j) - (double)pM);
          myA += myB * myB;
        }
        const double fx = nBins > 0 ? myA / (double)nBins : 0.0;
        put(cFlux, fx > 0.0 ? (float)sqrt(fx) : 0.0f);
      }
    }
    if (p.entropy) {                                                    // smileutil/smileUtil.c:2082-2124
      const double entropy_floor = 0.0000001;
      double e = 0.0, dn = 0.0;
      const double l2 = log(2.0);
      float mn = 0.0f;
      for (int i = lo; i <= hi; i++) { const float x = v.LP(i); dn += (double)x; if (x < mn) mn = x; }
      if (mn < 0.0f) {
        const double mf = entropy_floor + mn;
        for (int i = lo; i <= hi; i++) { const float x = v.LP(i); if (x <= mf) dn += mf - x; dn -= (double)mn; }
      } else mn = 0.0f;
      if (dn < (float)entropy_floor) dn = (float)entropy_floor;
      for (int i = lo; i <= hi; i++) {
        double vv = __fsub_rn(v.LP(i), mn);
        if (vv <= entropy_floor) vv = entropy_floor;
        const double ln = vv / dn;
        if (ln > 0.0) e += ln * log(ln) / l2;
      }
      put(cEntropy, (float)(-e));
    }
  } else if (warp == 2) {
    // ---- centroid, moments, overall slope ----
    if (p.centroid || p.stddev || p.variance || p.skewness || p.kurtosis || p.slope) {
      const double frameSum = (p.normBand && !p.useLog) ? frame_sum() : 0.0;
      const double sumB = sum_b(frameSum);
      const double sumA = sum_a();
      float ctr = 0.0f;
      if (sumB != 0.0) ctr = (float)(sumA / sumB);
      if (p.centroid) put(cCentroid, ctr);
      if (p.stddev || p.variance || p.skewness || p.kurtosis) {         // :1338-1397
        const double u = ctr;
        double m2 = 0.0, m3 = 0.0, m4 = 0.0;
        for (int i = lo; i <= hi; i++) {
          const double t1 = (frq(i) - u);
          double m = t1 * t1 * (double)v.LP(i);
          m2 += m; m *= t1; m3 += m; m4 += m * t1;
        }
        double sigma2 = 0.0;
        if (sumB != 0.0) sigma2 = m2 / sumB;
        if (p.stddev) put(cStd, sigma2 > 0.0 ? (float)sqrt(sigma2) : 0.0f);
        if (p.variance) put(cVar, (float)sigma2);
        if (p.skewness) put(cSkew, sigma2 <= 0.0 ? 0.0f : (float)(m3 / (sumB * sigma2 * sqrt(sigma2))));
        if (p.kurtosis) put(cKurt, sigma2 == 0.0 ? 0.0f : (float)(m4 / (sumB * sigma2 * sigma2)));
      }
      if (p.slope) {                                                    // :1400-1427
        double Sf = 0.0, S2f = 0.0;
        const double Nind = (double)nBins;
        for (int i = lo; i <= hi && i < Nsrc; i++) { const double f = frq(i); S2f += f * f; Sf += f; }
        const double deno = (Nind * S2f - Sf * Sf);
        double slope = 0.0;
        if (deno != 0.0) slope = (Nind * sumA - Sf * sumB) / deno;
        put(cSlope, p.oldSlopeScale ? (float)(slope * (Nind - 1.0)) : (float)slope);
      }
    }
  } else if (warp == 3) {
    // ---- band slopes, alpha ratio, Hammarberg index, extrema, harmonicity, flatness ----
    for (int b = 0; b < p.nSlopes; b++) {                               // :873-993
      const int iL = p.slopeIL[b], iR = p.slopeIR[b];
      const double wL = p.slopeWL[b], wR = p.slopeWR[b], Nind = p.slopeNind[b];
      double Sf = frq(iL) * wL, S2f = Sf * Sf;
      double sumA = frq(iL) * wL * (double)v.LP(iL), sumB = wL * v.LP(iL);
      for (int ii = iL + 1; ii < iR && ii < Nsrc; ii++) {
        const double f = frq(ii), x = (double)v.LP(ii);
        S2f += f * f; Sf += f; sumA += f * x; sumB += x;
      }
      S2f += frq(iR) * wR * frq(iR) * wR;
      Sf += frq(iR) * wR;
      sumA += frq(iR) * wR * (double)v.LP(iR);
      sumB += wR * (double)v.LP(iR);
      const double deno = (Nind * S2f - Sf * Sf);
      double slope = 0.0;
      if (deno != 0.0) slope = (Nind * sumA - Sf * sumB) / deno;
      put(cSlopes + b, p.oldSlopeScale ? (float)(slope * (Nind - 1.0)) : (float)slope);
    }
    if (p.alphaRatio) {                                                 // :996-1037 (float sums)
      float sum01 = 0.0f, sum15 = 0.0f;
      for (int j = 0; j < Nsrc; j++) {
        const double f = frq(j);
        if (f > 5000.0) break;
        if (f < 1000.0) sum01 = __fadd_rn(sum01, v.P(j)); else sum15 = __fadd_rn(sum15, v.P(j));
      }
      if (sum01 > 0.0f) {
        if (p.useLog) put(cAlpha, (sum15 > specFloor) ? (float)(10.0 * log((double)__fdiv_rn(sum15, sum01)) / log(10.0))
                                                      : (float)(10.0 * (log((double)specFloor) - log((double)sum01)) / log(10.0)));
        else put(cAlpha, __fdiv_rn(sum15, sum01));
      } else put(cAlpha, 0.0f);
    }
    if (p.hammarberg) {                                                 // :1040-1089
      float max02 = 0.0f, max25 = 0.0f;
      for (int j = 0; j < Nsrc; j++) {
        const double f = frq(j);
        if (f > 5000.0) break;
        const float x = v.P(j);
        if (f < 2000.0) { if (x > max02) max02 = x; } else { if (x > max25) max25 = x; }
      }
      if (max25 > 0.0f) {
        if (p.useLog) put(cHamm, (max02 > specFloor) ? (float)(10.0 * log((double)__fdiv_rn(max02, max25)) / log(10.0))
                                                     : (float)(10.0 * (log((double)specFloor) - log((double)max25)) / log(10.0)));
        else put(cHamm, __fdiv_rn(max02, max25));
      } else put(cHamm, 0.0f);
    }
    if (p.maxPos || p.minPos) {                                         // :1314-1330
      int maP = lo, miP = lo;
      float mx = v.LP(lo), mn = mx;
      for (int j = lo + 1; j < hi; j++) {
        const float x = v.LP(j);
        if (x < mn) { mn = x; miP = j; }
        if (x > mx) { mx = x; maP = j; }
      }
      if (p.maxPos) put(cMaxPos, (float)frq(maP));
      if (p.minPos) put(cMinPos, (float)frq(miP));
    }
    if (p.harmonicity || p.flatness) {
      const double frameSum = (p.normBand && !p.useLog) || (p.harmonicity && p.normBand) ? frame_sum() : 0.0;
      const double sumB = sum_b(frameSum);
      if (p.harmonicity) {                                              // :1484-1513
        float ptpSum = 0.0f, lastPeak = -99.0f;
        for (int j = lo + 2; j < hi - 1; j++) {
          const float a = v.LP(j - 2), b = v.LP(j - 1), c = v.LP(j), d = v.LP(j + 1), e = v.LP(j + 2);
          if ((a < c && b < c && c > d && c > e) || (a > c && b > c && c < d && c < e)) {
            if (lastPeak != -99.0f) ptpSum = __fadd_rn(ptpSum, fabsf(__fsub_rn(c, lastPeak)));
            lastPeak = c;
          }
        }
        ptpSum = __fdiv_rn(ptpSum, 2.0f);
        if (p.normBand && sumB != 0.0) {
          if (p.useLog) ptpSum = __fdiv_rn(ptpSum, (float)fabs(sumB)); else ptpSum = __fdiv_rn(ptpSum, (float)frameSum);
        } else ptpSum = __fdiv_rn(ptpSum, (float)nBins);
        put(cHarm, ptpSum);
      }
      if (p.flatness) {                                                 // :1515-1544
        float sf = 0.0f, gmean = 0.0f;
        int nGm = 0;
        if (sumB != 0.0) {
          for (int j = lo; j <= hi; j++) {
            const float x = v.LP(j);
            if (x != 0.0f) { gmean = (float)((double)gmean + log((double)fabsf(x))); nGm++; }
          }
          if (nGm > 0) gmean = __fdiv_rn(gmean, (float)nGm);
          gmean = (float)exp((double)gmean);
          sf = __fdiv_rn(gmean, (float)fabs(sumB / (double)nBins));
        }
        if (p.logFlatness) put(cFlat, sf > 0.0f ? (float)log((double)sf) : 0.0f); else put(cFlat, sf);
      }
    }
  }
}

cudaError_t launch_spectral(const SpectralParams &p, cudaStream_t st)
{
  if (p.nTiles <= 0) return cudaSuccess;
  // Stage the magnitude tile in shared memory only together with a log spectrum (measured: without
  // one, the extra shared memory costs more occupancy than the cached global reads cost time), and
  // only when both tiles fit (they do up to FFT 1024)
  const size_t tile = (size_t)p.nSrc * 32 * sizeof(float);
  SpectralParams q = p;
  q.stageMag = (p.reqLog && tile * 2 <= 200 * 1024) ? 1 : 0;
  const size_t smem = tile * ((p.reqLog ? 1 : 0) + q.stageMag);
  cudaError_t e = cudaFuncSetAttribute(spectral_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  spectral_kernel<<<p.nTiles, kSpecThreads, smem, st>>>(q);
  return cudaGetLastError();
}

// cFFTmagphase as an output level (spectrogram): transposes a magnitude tile [nSrc][F] into rows of the
// static level, 32 bins at a time through shared memory so that both sides are coalesced
// mode (dspcore/fftmagphase.cpp:215-255, float statements): 0 magnitude, 1 normalise (|X| / N), 2 power, 3 normalise + power
// (|X|^2 / N^2), 4 dBpsd = max(mindBp, dBpnorm + 10 log10(|X|^2 / N^2)) (bins 0 and N/2: 20 log10(|X| / N)); N = FFT size
__device__ __forceinline__ float mag_variant(float m, int mode, bool edgeBin, float N, float dBpnorm, float mindBp)
{
  switch (mode) {
    case 1: return __fmul_rn(__fdiv_rn(1.0f, N), m);
    case 2: return __fmul_rn(m, m);
    case 3: if (edgeBin) { const float v = __fmul_rn(__fdiv_rn(1.0f, N), m); return __fmul_rn(v, v); }
            return __fmul_rn(__fdiv_rn(1.0f, __fmul_rn(N, N)), __fmul_rn(m, m));
    case 4: {
      const float v = edgeBin ? __fadd_rn(dBpnorm, __fmul_rn(20.0f, log10f(__fmul_rn(__fdiv_rn(1.0f, N), m))))
                              : __fadd_rn(dBpnorm, __fmul_rn(10.0f, log10f(__fmul_rn(__fdiv_rn(1.0f, __fmul_rn(N, N)), __fmul_rn(m, m)))));
      return v > mindBp ? v : mindBp;                 // MAX(mindBp, v): a NaN (log10 of 0 * ...) compares false and yields mindBp like the macro
    }
    default: return m;
  }
}

__global__ void __launch_bounds__(256) mag_rows_kernel(const float *mag, const OpTile *tiles, int F, int nSrc,
                                                       const long long *statOff, float *stat, int statStride, int outCol,
                                                       int mode, float fftN, float dBpnorm, float mindBp)
{
  __shared__ float t[32][33];
  const OpTile tl = tiles[blockIdx.x];
  const float *src = mag + ((size_t)blockIdx.x * nSrc) * F;
  float *dst = stat + (statOff[tl.utt] + tl.f0) * (long long)statStride + outCol;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;            // 32 x 8
  for (int k0 = 0; k0 < nSrc; k0 += 32) {
    for (int kk = ty; kk < 32; kk += 8)
      t[kk][tx] = (k0 + kk < nSrc && tx < F) ? src[(size_t)(k0 + kk) * F + tx] : 0.f;
    __syncthreads();
    for (int ff = ty; ff < tl.nf; ff += 8)
      if (k0 + tx < nSrc) dst[(long long)ff * statStride + k0 + tx] = mag_variant(t[tx][ff], mode, k0 + tx == 0 || k0 + tx == nSrc - 1, fftN, dBpnorm, mindBp);
    __syncthreads();
  }
}

cudaError_t launch_mag_rows(const float *mag, const OpTile *tiles, int nTiles, int F, int nSrc, const long long *statOff,
                            float *stat, int statStride, int outCol, cudaStream_t st, int mode, float fftN, float dBpnorm, float mindBp)
{
  if (nTiles <= 0) return cudaSuccess;
  mag_rows_kernel<<<nTiles, 256, 0, st>>>(mag, tiles, F, nSrc, statOff, stat, statStride, outCol, mode, fftN, dBpnorm, mindBp);
  return cudaGetLastError();
}

template <bool F32>
__global__ void __launch_bounds__(32) energy_kernel(const TimeOpParams p)
{
  const OpTile tl = p.tiles[blockIdx.x];
  const int lane = threadIdx.x;
  if (lane >= tl.nf) return;
  const long long uo = p.uttOff[tl.utt];
  FrameReader<F32> fr{p, p.pcm + uo * p.nChan, frame_first_sample(tl.f0 + lane, p.frameStep, p.frameCenter)};
  const int N = p.frameSize;
  double d = 0.0;                                     // lldcore/energy.cpp:157-161
  for (int i = 0; i < N; i++) { const float t = fr.at(i); d += (double)__fmul_rn(t, t); }
  float *dst = p.stat + (p.statOff[tl.utt] + tl.f0 + lane) * (long long)p.statStride + p.outCol;
  int n = 0;
  if (p.eRms) dst[n++] = __fadd_rn(__fmul_rn((float)sqrt(d / (double)(float)N), p.escaleRms), p.ebiasRms);
  if (p.eEnergy2) dst[n++] = __fadd_rn(__fmul_rn((float)(d / (double)N), p.escaleSquare), p.ebiasSquare);
  if (p.eLog) {
    const double minE = 8.674676e-019;
    if (!p.eHtk) {
      d /= (double)(float)N;
      if (d < minE) d = minE;
    } else {
      d *= 32767.0 * 32767.0;
      if (d <= 1.0) d = 1.0;
    }
    dst[n++] = __fadd_rn(__fmul_rn((float)log(d), p.escaleLog), p.ebiasLog);
  }
}

template <bool F32>
__global__ void __launch_bounds__(32) mzcr_kernel(const TimeOpParams p)
{
  const OpTile tl = p.tiles[blockIdx.x];
  const int lane = threadIdx.x;
  if (lane >= tl.nf) return;
  const long long uo = p.uttOff[tl.utt];
  FrameReader<F32> fr{p, p.pcm + uo * p.nChan, frame_first_sample(tl.f0 + lane, p.frameStep, p.frameCenter)};
  const int N = p.frameSize;
  float mean = fr.at(0), nzc = 0.0f, nmc = 4.0f, mx = 0.f, mn = 0.f, absmax = 0.f;   // lldcore/mzcr.cpp:113-115
  if (p.zZcr || p.zMcr || p.zDc) {
    float a = fr.at(0), b = (N > 1) ? fr.at(1) : 0.f;
    for (int i = 1; i < N - 1; i++) {
      const float c = fr.at(i + 1);
      mean = __fadd_rn(mean, b);
      if (((__fmul_rn(a, c) <= 0.0f) && (b == 0.0f)) || (__fmul_rn(a, b) < 0.0f)) nzc = __fadd_rn(nzc, 1.0f);
      a = b; b = c;
    }
    nzc = __fdiv_rn(nzc, (float)N);
    mean = __fdiv_rn(mean, (float)N);
  }
  if (p.zMcr) {
    float a = __fsub_rn(fr.at(0), mean), b = (N > 1) ? __fsub_rn(fr.at(1), mean) : 0.f;
    for (int i = 1; i < N - 1; i++) {
      const float c = __fsub_rn(fr.at(i + 1), mean);
      if (((__fmul_rn(a, c) <= 0.0f) && (b == 0.0f)) || (__fmul_rn(a, b) < 0.0f)) nmc = __fadd_rn(nmc, 1.0f);
      a = b; b = c;
    }
    nmc = __fdiv_rn(nmc, (float)N);
  }
  if (p.zAmax || p.zMaxmin) {
    mx = mn = fr.at(0);
    for (int i = 1; i < N; i++) { const float x = fr.at(i); if (x < mn) mn = x; if (x > mx) mx = x; }
    absmax = (fabsf(mn) > fabsf(mx)) ? fabsf(mn) : fabsf(mx);
  }
  float *dst = p.stat + (p.statOff[tl.utt] + tl.f0 + lane) * (long long)p.statStride + p.outCol;
  int n = 0;
  if (p.zZcr) dst[n++] = nzc;
  if (p.zMcr) dst[n++] = nmc;
  if (p.zAmax) dst[n++] = absmax;
  if (p.zMaxmin) { dst[n++] = mx; dst[n++] = mn; }
  if (p.zDc) dst[n++] = mean;
}

// cIntensity (lldcore/intensity.cpp:124-146).  The reference bounds its summation loop by
// MIN(Nsrc, MIN(nWin, Ndst)) with Ndst = number of OUTPUT values (1 or 2), i.e. only the first one or
// two samples of the frame enter the "mean": reproduced as is, this is what the shipped configs emit.
template <bool F32>
__global__ void __launch_bounds__(32) intensity_kernel(const TimeOpParams p)
{
  const OpTile tl = p.tiles[blockIdx.x];
  const int lane = threadIdx.x;
  if (lane >= tl.nf) return;
  const long long uo = p.uttOff[tl.utt];
  FrameReader<F32> fr{p, p.pcm + uo * p.nChan, frame_first_sample(tl.f0 + lane, p.frameStep, p.frameCenter)};
  const int nOut = (p.iIntensity ? 1 : 0) + (p.iLoudness ? 1 : 0);
  const int safeN = min(p.frameSize, nOut);
  double Im = 0.0;
  if (safeN > 0) { const float x = fr.at(0); Im += p.iW0 * (double)x * (double)x; }
  if (safeN > 1) { const float x = fr.at(1); Im += p.iW1 * (double)x * (double)x; }
  Im /= p.iWinSum;
  float *dst = p.stat + (p.statOff[tl.utt] + tl.f0 + lane) * (long long)p.statStride + p.outCol;
  int n = 0;
  if (p.iIntensity) dst[n++] = (float)Im;
  if (p.iLoudness) dst[n++] = (float)pow(Im / 0.000001, 0.3);
}

cudaError_t launch_intensity(const TimeOpParams &p, cudaStream_t st)
{
  if (p.nTiles <= 0) return cudaSuccess;
  (p.pcmF32 ? intensity_kernel<true> : intensity_kernel<false>)<<<p.nTiles, 32, 0, st>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_energy(const TimeOpParams &p, cudaStream_t st)
{
  if (p.nTiles <= 0) return cudaSuccess;
  (p.pcmF32 ? energy_kernel<true> : energy_kernel<false>)<<<p.nTiles, 32, 0, st>>>(p);
  return cudaGetLastError();
}
cudaError_t launch_mzcr(const TimeOpParams &p, cudaStream_t st)
{
  if (p.nTiles <= 0) return cudaSuccess;
  (p.pcmF32 ? mzcr_kernel<true> : mzcr_kernel<false>)<<<p.nTiles, 32, 0, st>>>(p);
  return cudaGetLastError();
}

}  // namespace osm
