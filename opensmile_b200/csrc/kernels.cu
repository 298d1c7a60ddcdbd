// kernels.cu -- launch_lld and the int16 instances of lld_kernel (lld_kernel.cuh), the temporal post-processing
// (post_kernel), the ACF pitch kernels, the cPlp RASTA filter and tail, and the small per-row helpers (sm_90a).
#include <cstdio>
#include <cstdlib>

#include "fft_radix.cuh"
#include "kernels.cuh"

#include "lld_common.cuh"
#include "lld_kernel.cuh"

namespace osm {

template cudaError_t launch_lld_kernel<false>(const LldParams &, int, int, cudaStream_t, LldLaunchInfo *, bool);

// ------------------------------------------------------------------------------------------
// temporal post-processing
// ------------------------------------------------------------------------------------------
// Tick-order model of chained window processors (cWindowProcessor with blocksize=1, components
// ticking in data-flow order; core/windowProcessor.cpp:85-119,167-230, core/componentManager.cpp:
// 1233-1262).  For the level produced by stage s:  final_s = final_{s-1} + W_s frames in total,
// c0_s = max(c0_{s-1} - W_s, 0) of them produced before EOI is raised (c0_0 = final_0 = T).
// When the consumer computes frame t >= c0_s its input level holds
//     navail = min(c0_{s-1} + (t - c0_s) + 1, final_{s-1})
// frames.  Matrix reads (core/dataMemoryLevel.cpp:1651-1738): window start >= 0: rows >= navail
// replicate row navail-1; window start < 0: rows < 0 replicate row 0 and rows >= navail come
// from the zero-initialised, not yet written level buffer (0.0).  For c0_{s-1} >= W_s this is the
// plain "clamp to [0, final-1]" rule; the rest only triggers for utterances shorter than the
// summed window lengths and is reproduced because the reference does it.
//
// post_kernel: one CTA per tile of kPostRows output rows of one utterance.  The static rows the
// tile depends on (halo = summed half windows) are staged in shared memory once, every stage of
// every group is then evaluated level by level in shared memory (O(window) per element) and
// the finished rows are written out.
constexpr int kPostRows = 64;      // at most; see post_tile_rows()
constexpr int kPostMaxHalo = 12;
constexpr int kPostThreads = 256;

__device__ __forceinline__ float post_read(const float *lvl, int n, int rowBase, int t, int W, int navail, int i, int c)
{
  // lvl: smem rows of the input level, row index (absolute frame - rowBase), n columns
  if (t - W < 0) {
    if (i < 0) i = 0;
    else if (i >= navail) return 0.f;
  } else if (i > navail - 1) {
    i = navail - 1;
  }
  return lvl[(i - rowBase) * n + c];
}

__global__ void __launch_bounds__(kPostThreads) post_kernel(const PostParams p)
{
  extern __shared__ float psm[];
  const TileRef tr = p.tiles[blockIdx.x];
  const int u = tr.utt, r0 = tr.f0;
  const long long Ls = p.uttOff[u + 1] - p.uttOff[u];
  const int Tout = (int)(p.rowOff[u + 1] - p.rowOff[u]);
  const int r1 = min(r0 + p.rows, Tout);
  const int H = p.halo;
  const int rowBase = r0 - H;                       // absolute frame of smem row 0 (may be < 0)
  const int nRowsBuf = p.rows + 2 * H;
  float *S0 = psm;                                  // [nRowsBuf][nStat]
  float *A = S0 + nRowsBuf * p.nStat;               // [nRowsBuf][maxN]
  float *B = A + nRowsBuf * p.maxN;
  const int tid = threadIdx.x;

  // ---- static rows [r0-H, r1+H) /\ [0, Tmax) -> smem (Tmax = rows of the static buffer) ----
  {
    const int Tmax = (int)(p.statOff[u + 1] - p.statOff[u]);
    const int lo = max(rowBase, 0), hi = min(r1 + H, Tmax);
    const float *src = p.stat + p.statOff[u] * (long long)p.statStride;
    const int tot = (hi - lo) * p.nStat;
    for (int idx = tid; idx < tot; idx += kPostThreads) {
      const int rr = idx / p.nStat, c = idx - rr * p.nStat;
      S0[(lo + rr - rowBase) * p.nStat + c] = src[(long long)(lo + rr) * p.statStride + c];
    }
  }
  __syncthreads();

  for (int gi = 0; gi < p.nGroups; gi++) {
    const PostGroup &g = p.groups[gi];
    const int n = g.n;
    const int T = (int)frame_count(Ls, g.frameSize, g.frameStep, g.frameCenter);   // frames of this group's source level
    // a multi-level reader delivers min over its levels: that bounds how many frames the first stage
    // produces (before EOI and in total), while reads of THIS level still clamp at its own end
    int Tlim = T;
    for (int k = 0; k < g.nLim; k++) Tlim = min(Tlim, (int)frame_count(Ls, g.limSize[k], g.limStep[k], g.limCenter[k]));
    // level 0 view of this group: copy its columns so that every level has row stride n
    const float *cur;
    {
      const int lo = max(rowBase, 0), hi = min(r1 + H, T);
      const int tot = (hi - lo) * n;
      for (int idx = tid; idx < tot; idx += kPostThreads) {
        const int rr = idx / n, c = idx - rr * n;
        A[(lo + rr - rowBase) * n + c] = S0[(lo + rr - rowBase) * p.nStat + g.srcCol + c];
      }
      cur = A;
    }
    __syncthreads();
    int Tprev = T, n0 = T;                          // input level: total frames, frames before EOI
    int Tcnt = Tlim, n0cnt = Tlim;                  // the same as seen through the reader (min over its levels)
    int Hrem = 0;
    for (int s = 0; s < g.nStages; s++) Hrem += g.win[s];
    for (int s = 0; s < g.nStages; s++) {
      const int W = g.win[s];
      Hrem -= W;
      const int c0 = max(n0cnt - W, 0);
      const int Tcur = Tcnt + W;
      float *dst = (cur == A) ? B : A;
      const int lo = max(r0 - Hrem, 0), hi = min(r1 + Hrem, Tcur);   // rows of this level needed
      const int tot = (hi - lo) * n;
      float norm = 0.f;
      for (int i = 1; i <= W; i++) norm = __fadd_rn(norm, __fmul_rn((float)i, (float)i));
      norm = __fmul_rn(norm, 2.0f);                 // deltaRegression.cpp:77-80
      for (int idx = tid; idx < tot; idx += kPostThreads) {
        const int rr = idx / n, c = idx - rr * n;
        const int t = lo + rr;
        const int navail = (t < c0) ? Tprev : min(n0 + (t - c0) + 1, Tprev);
        float y;
        if (g.kind[s] == 2) {
          // fullinputMean.cpp:516-522 : vec->data[i] -= means[i]
          y = __fsub_rn(post_read(cur, n, rowBase, t, 0, navail, t, c), p.means[(long long)u * p.nStat + g.srcCol + c]);
        } else if (g.kind[s] == 0) {
          // deltaRegression.cpp:139-146 : num = sum_i i*(x[t+i]-x[t-i]) ; y = num / norm
          float num = 0.f;
          const int fl = g.flags[s];                 // bit 1 relativeDelta, bit 2 absOutput, bit 3 halfWaveRect (:100-108,157-165)
          for (int i = 1; i <= W; i++) {
            const float later = post_read(cur, n, rowBase, t, W, navail, t + i, c);
            const float prior = post_read(cur, n, rowBase, t, W, navail, t - i, c);
            float delta = __fsub_rn(later, prior);
            if (fl & 2) delta = prior != 0.0f ? __fdiv_rn(delta, fabsf(prior)) : 0.0f;
            num = __fadd_rn(num, __fmul_rn((float)i, delta));
          }
          y = __fdiv_rn(num, norm);
          if (fl & 8) { if (y < 0.0f) y = 0.0f; }
          else if (fl & 4) { if (y < 0.0f) y = -y; }
        } else {
          // contourSmoother.cpp:84-117 : y = x[n]; y += x[n-w]; y += x[n+w]; y /= smaWin
          const int noZero = g.flags[s];
          const float x0 = post_read(cur, n, rowBase, t, W, navail, t, c);
          if (noZero && x0 == 0.f) {
            y = 0.f;
          } else {
            y = x0;
            int cnt = 1;
            for (int w = 1; w <= W; w++) {
              const float a = post_read(cur, n, rowBase, t, W, navail, t - w, c);
              const float b = post_read(cur, n, rowBase, t, W, navail, t + w, c);
              if (!noZero || a != 0.f) { y = __fadd_rn(y, a); cnt++; }
              if (!noZero || b != 0.f) { y = __fadd_rn(y, b); cnt++; }
            }
            y = __fdiv_rn(y, noZero ? (float)cnt : (float)(2 * W + 1));
          }
        }
        dst[(t - rowBase) * n + c] = y;
      }
      __syncthreads();
      cur = dst;
      n0 = c0; n0cnt = c0;
      Tprev = Tcur; Tcnt = Tcur;
    }
    // ---- write rows [r0, r1) of this group ----
    {
      float *o = p.out + (p.rowOff[u] + r0) * (long long)p.outStride + g.outCol;
      const int tot = (r1 - r0) * n;
      for (int idx = tid; idx < tot; idx += kPostThreads) {
        const int rr = idx / n, c = idx - rr * n;
        o[(long long)rr * p.outStride + c] = cur[(r0 + rr - rowBase) * n + c];
      }
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------
// cAcf (ACF + cepstrum) + cPitchACF, per-frame part.
//   dspcore/acf.cpp:250-345: both levels are the inverse real FFT of a real, even spectrum
//   (power resp. log(1+x)), i.e. cosine transforms.  With z[n] = Pfull[n] + i*Cfull[n] over the
//   symmetric extension n = 0..N-1, ONE complex FFT of size N gives both at once:
//   Re Z[j] = 2*acf_ooura[j], Im Z[j] = 2*cep_ooura[j]  (real even input -> real even output).
//   lldcore/pitchACF.cpp:137-361 then scans the two arrays per frame.
// One CTA per tile, lane = frame, same batched in-place FFT as lld_kernel.
// ------------------------------------------------------------------------------------------
template <int N, int F, int NT>
__global__ void __launch_bounds__(NT, 1) acf_pitch_kernel(const AcfPitchParams p)
{
  constexpr int NW = NT / 32, G = 32 / F, NVW = NW * G;
  using Fc = Fact<N>;
  extern __shared__ __align__(16) unsigned char smem[];
  float2 *Z = reinterpret_cast<float2 *>(smem);
  float2 *sTw = reinterpret_cast<float2 *>(smem + (size_t)N * F * 8);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int f = lane & (F - 1);
  const int vw = warp * G + lane / F;
  // the magnitude level is stored in tiles of p.F frames; this CTA handles F of them (sub-tile)
  const int SUB = p.F / F;
  const int tileIdx = blockIdx.x / SUB, sub = blockIdx.x - tileIdx * SUB;
  OpTile tl = p.tiles[tileIdx];
  tl.f0 += sub * F;
  tl.nf = min(max(tl.nf - sub * F, 0), F);
  const int nSrc = p.nSrc;
  for (int i = tid; i < p.twCount; i += NT) sTw[i] = p.twiddles[i];
  // ---- spectrum -> symmetric complex input ----
  {
    const float *mg = p.mag + (size_t)tileIdx * nSrc * p.F + sub * F;
    for (int idx = tid; idx < nSrc * F; idx += NT) {
      const int k = idx / F, ff = idx - k * F;
      const float m = mg[(size_t)k * p.F + ff];
      const float pw = p.acfUsePower ? __fmul_rn(m, m) : m;                       // acf.cpp:253-261
      const float cs = p.cepUsePower ? __fmul_rn(m, m) : m;
      float cv;
      if (p.oldCompatCepstrum) cv = (k == 0 || k == nSrc - 1) ? cs : ((cs > 0.0f) ? logf(cs) : 0.0f);   // acf.cpp:276-286 (float log)
      else cv = (cs > 0.0f) ? (float)log((double)cs + 1.0) : 0.0f;                 // acf.cpp:289-305
      const float2 v = make_float2(pw, cv);
      Z[k * F + ff] = v;
      if (k > 0 && k < N / 2) Z[(N - k) * F + ff] = v;
    }
  }
  __syncthreads();
  // oldCompatCepstrum: the two transforms share one complex FFT, whose rounding is relative to the larger channel, and log(x) of
  // the tiny powers of a quiet frame (|log x| ~ 20) would swamp its ACF channel (x ~ 1e-9).  The cepstrum channel of each frame is
  // weighted by the power of two that brings both channels to the same magnitude (exact) and the weight is undone on output.
  __shared__ float sCepUnscale[32];
  if (p.oldCompatCepstrum) {
    for (int ff = tid; ff < F; ff += NT) {
      float mp = 0.0f, mc = 0.0f;
      for (int k = 0; k <= N / 2; k++) { const float2 v = Z[k * F + ff]; mp = fmaxf(mp, fabsf(v.x)); mc = fmaxf(mc, fabsf(v.y)); }
      const int e = (mp > 0.0f && mc > 0.0f) ? max(min(ilogbf(mp) - ilogbf(mc), 100), -100) : 0;
      sCepUnscale[ff] = ldexpf(1.0f, -e);
      const float w = ldexpf(1.0f, e);
      for (int k = 0; k < N; k++) Z[k * F + ff].y *= w;
    }
    __syncthreads();
  }
  {
    LldParams dummy;     // fft_stage only reads it in its FIRST (sample loading) specialisation
    fft_stage<N, F, NVW, Fc::R0, N, false, false, false>(Z, nullptr, nullptr, nullptr, sTw + p.twOff[0], dummy, vw, f);
    __syncthreads();
    fft_stage<N, F, NVW, Fc::R1, N / Fc::R0, false, false, false>(Z, nullptr, nullptr, nullptr, sTw + p.twOff[1], dummy, vw, f);
    __syncthreads();
    fft_stage<N, F, NVW, Fc::R2, N / (Fc::R0 * Fc::R1), false, true, false>(Z, nullptr, nullptr, nullptr, nullptr, dummy, vw, f);
  }
  __syncthreads();
  // ---- per-frame analysis (lldcore/pitchACF.cpp:137-183) ----
  // lane = frame as everywhere; the lag range [0, n) is cut into NVW slices, one per virtual warp.
  // Counts, maxima and the first-peak index combine exactly; the two double sums (mean of the ACF,
  // mean |cepstrum|) are added slice by slice instead of lag by lag (differences at the 1e-16 level).
  const int n = N / 2;                                     // length of each cAcf level (Ndst = Nsrc - 1)
  const float fNsrc = (float)nSrc;
  auto acf = [&](int j) {
    float d = 0.5f * Z[fft_pos<N>(j) * F + f].x;
    if (p.normOutput) d = __fdiv_rn(d, fNsrc);             // acf.cpp:321-325
    return fabsf(d);                                       // :342-344
  };
  auto cep = [&](int j) {
    float d = 0.5f * Z[fft_pos<N>(j) * F + f].y;
    if (p.oldCompatCepstrum) d *= sCepUnscale[f];
    if (p.normOutput) d = __fdiv_rn(d, fNsrc);
    return p.absCepstrum ? fabsf(d) : d;                   // :327-341
  };
  // per-slice partial results, [NVW][F] each, behind the twiddles
  double *sD = reinterpret_cast<double *>(smem + (((size_t)N * F * 8 + (size_t)p.twCount * 8 + 15) & ~(size_t)15));
  double *sMx = sD, *sMean = sD + NVW * F, *sCmax = sD + 2 * NVW * F, *sCsum = sD + 3 * NVW * F;
  int *sI = reinterpret_cast<int *>(sD + 4 * NVW * F);
  int *sZcr = sI, *sMcr = sI + NVW * F, *sIdx = sI + 2 * NVW * F;
  const double Nd = (double)(2 * n);
  const double Tsamp = (double)p.fsSec / Nd;
  const int preskip = (p.maxPitch <= 0.0) ? 0 : (int)(1.0 / (p.maxPitch * Tsamp));
  const int skip = preskip + 1;
  const int j0 = (int)(((long long)n * vw) / NVW), j1 = (int)(((long long)n * (vw + 1)) / NVW);
  {
    // voicingProb pass (:249-284): sign changes, rising maximum, sum; cepstrum maximum and |.| sum (:286-297)
    int zcr = 0;
    double mx = -1.0, mean = 0.0;                          // ACF values are >= 0
    const int i0 = max(j0, 1);
    float a0 = acf(i0 - 1);
    for (int i = i0; i < j1; i++) {
      const float a1 = acf(i);
      if (__fmul_rn(a0, a1) < 0.0f) zcr++;
      if (i >= preskip) {
        if (((double)a1 > mx) && (a0 < a1)) mx = a1;
        mean += (double)a1;
      }
      a0 = a1;
    }
    double cmax = -1e300, csum = 0.0;
    for (int i = j1 - 1; i >= j0; i--) {
      const double buf = cep(i);
      csum += fabs(buf);
      if (i >= skip && buf > cmax) cmax = buf;
    }
    sZcr[vw * F + f] = zcr; sMx[vw * F + f] = mx; sMean[vw * F + f] = mean;
    sCmax[vw * F + f] = cmax; sCsum[vw * F + f] = csum;
  }
  __syncthreads();
  // the reference starts the mean with element preskip of the concatenated input [acf ; cepstrum] (:258): past the ACF's n
  // lags that is a cepstrum value.  The plan refuses preskip >= 2n, where the reference reads outside its input
  double mean = preskip < n ? acf(preskip) : cep(preskip - n), mx = acf(n - 1), cmax = cep(n - 1), csum = 0.0;
  int zcr = 0;
  for (int w = 0; w < NVW; w++) {
    zcr += sZcr[w * F + f];
    mean += sMean[w * F + f];
    if (sMx[w * F + f] > mx) mx = sMx[w * F + f];
    if (sCmax[w * F + f] > cmax) cmax = sCmax[w * F + f];
  }
  for (int w = NVW - 1; w >= 0; w--) csum += sCsum[w * F + f];     // the reference walks the lags downwards
  mean /= (double)(n - preskip + 1);
  csum /= (double)n;
  {
    // mean crossings (:266-273) and the first cepstral peak above the threshold (:299-310)
    int mcr = 0;
    const int i0 = max(j0, 1);
    float a0 = acf(i0 - 1);
    for (int i = i0; i < j1; i++) {
      const float a1 = acf(i);
      if (((double)a0 - mean) * ((double)a1 - mean) < 0.0) mcr++;
      a0 = a1;
    }
    int first = 0x7fffffff;
    const double thr = (cmax + csum) * 0.6;
    const int lo = max(j0, skip + 1), hi = min(j1, n - 1);
    if (lo < hi) {
      float cm = cep(lo - 1), c0 = cep(lo);
      for (int i = lo; i < hi; i++) {
        const float c1 = cep(i + 1);
        if ((double)c0 > thr && (cm < c0) && (c0 > c1)) { first = i; break; }
        cm = c0; c0 = c1;
      }
    }
    sMcr[vw * F + f] = mcr; sIdx[vw * F + f] = first;
  }
  __syncthreads();
  if (vw == 0 && f < tl.nf) {
    int mcr = 0, maxIdx = 0x7fffffff;
    for (int w = 0; w < NVW; w++) { mcr += sMcr[w * F + f]; maxIdx = min(maxIdx, sIdx[w * F + f]); }
    if (maxIdx == 0x7fffffff) maxIdx = 0;
    const double acfZcr = (mcr > zcr) ? (double)mcr / (double)n : (double)zcr / (double)n;
    const float acf0 = acf(0);
    const double voicing = (acf0 > 0.0f) ? mx / (double)acf0 : 0.0;
    PitchRaw r;
    r.voicing = voicing; r.acfZcr = acfZcr; r.maxIdx = maxIdx;
    const float aI = acf(maxIdx);
    r.hnr = 0.f; r.hnrDB = 0.f; r.hnrLin = 0.f;
    if (p.HNR) {                                           // :312-326
      const float dd = __fsub_rn(acf0, aI);
      const double buf = (dd == 0.0f) ? 100000000000000000000.0 : (double)__fdiv_rn(aI, dd);
      r.hnr = (float)((buf > 0.00000000001) ? 10.0 * log(buf) : 10.0 * log(0.00000000001));
    }
    if (p.HNRdB) {                                         // :329-343
      double buf = (double)__fsub_rn(acf0, aI);
      buf = (buf == 0.0) ? 10e10 : (double)aI / buf;
      r.hnrDB = (float)((buf <= 10e-10) ? -100.0 : ((buf >= 10e10) ? +100.0 : 10.0 * log(buf) / log(10.0)));
    }
    if (p.linHNR) {                                        // :346-360
      double buf = (double)__fsub_rn(acf0, aI);
      buf = (buf == 0.0) ? 10e3 : (double)aI / buf;
      r.hnrLin = (float)((buf <= 10e-3) ? 10e-3 : ((buf >= 10e3) ? 10e3 : buf));
    }
    p.raw[p.statOff[tl.utt] + tl.f0 + f] = r;
  }
}

// per-utterance pitch contour smoothing state machine (lldcore/pitchACF.cpp:184-245): sequential in
// time, one thread per utterance
__global__ void pitch_smooth_kernel(const AcfPitchParams p, int u0, int u1)
{
  const int u = u0 + blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= u1) return;
  const long long Ls = p.uttOff[u + 1] - p.uttOff[u];
  const int T = (int)frame_count(Ls, p.frameSize, p.frameStep, p.frameCenter);
  const int n = p.nfft / 2;
  const double Tsamp = (double)p.fsSec / (double)(2 * n);
  float lastPitch = 0.f, lastlastPitch = 0.f, glMeanPitch = 0.f, pitchEnv = 0.f;
  int onsFlag = 0;
  const double maxPitch = p.maxPitch;
  for (int t = 0; t < T; t++) {
    const PitchRaw r = p.raw[p.statOff[u] + t];
    float *dst = p.stat + (p.statOff[u] + t) * (long long)p.statStride + p.outCol;
    int k = 0;
    if (p.voiceProb) dst[k++] = (float)r.voicing;
    if (p.HNR) dst[k++] = r.hnr;
    if (p.HNRdB) dst[k++] = r.hnrDB;
    if (p.linHNR) dst[k++] = r.hnrLin;
    if (p.F0 || p.F0env || p.voiceQual || p.F0raw) {
      int maxIdx = r.maxIdx;
      const float invT = __fdiv_rn(1.0f, __fmul_rn((float)maxIdx, (float)Tsamp));
      float vq = __fmul_rn(__fsub_rn((float)maxPitch, (float)fabs((r.acfZcr * maxPitch) - (double)invT)), (float)r.voicing);
      if (maxIdx == 0) vq = 0.0f;
      if (p.voiceQual) dst[k++] = vq;
      float pitch = 0.0f, rawF0 = 0.0f;
      if (maxIdx > 0) { pitch = invT; rawF0 = pitch; }
      if (r.voicing < p.voicingCutoff) { maxIdx = 0; pitch = 0.0f; }
      if ((lastPitch == 0.0f) && (pitch > 0.0f)) onsFlag = 1;
      if ((lastPitch > 0.0f) && (pitch == 0.0f) && (onsFlag == 0)) onsFlag = -1;
      if ((lastPitch > 0.0f) && (pitch > 0.0f)) onsFlag = 0;
      if ((lastPitch == 0.0f) && (pitch == 0.0f)) onsFlag = 0;
      if ((pitch == 0.0f) && (onsFlag == 1)) lastPitch = 0.0f;
      const float oPitch = pitch;
      const float tol = 0.4f;
      float alpha = 0.3f;
      if (pitch > 0.0f) {
        if (glMeanPitch == 0.0f) glMeanPitch = pitch;
        if (!((pitch < __fmul_rn(__fadd_rn(1.0f, tol), glMeanPitch)) && (pitch > __fmul_rn(__fsub_rn(1.0f, tol), glMeanPitch)))) {
          pitch = glMeanPitch;
          alpha = __fdiv_rn(alpha, 3.0f);
        }
        if (onsFlag && (lastPitch > pitch)) lastPitch = __fmul_rn(lastPitch, 0.85f);
      }
      if ((pitch > 0.0f) && (onsFlag == -1)) lastPitch = pitch;
      if (oPitch > 0.0f) glMeanPitch = __fadd_rn(__fmul_rn(__fsub_rn(1.0f, alpha), glMeanPitch), __fmul_rn(alpha, oPitch));
      float out;
      if ((lastlastPitch != 0.0f) && (lastPitch != 0.0f)) out = __fmul_rn(0.5f, __fadd_rn(lastlastPitch, lastPitch));
      else out = lastPitch;
      if (p.F0) dst[k++] = out;
      if (p.F0raw) dst[k++] = rawF0;
      lastlastPitch = lastPitch;
      lastPitch = pitch;
      if (p.F0env) {
        if (out > 0.0f) pitchEnv = __fadd_rn(__fmul_rn(0.75f, pitchEnv), __fmul_rn(0.25f, out));
        dst[k++] = pitchEnv;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------
int lld_tile_frames(int nfft, bool narrow)
{
  const int F = nfft == 4096 ? 8 : (nfft == 2048 ? 16 : 32);
  return (narrow && nfft >= 1024) ? F / 2 : F;
}
int lld_virtual_warps(int nfft) { return nfft == 512 ? 8 : (nfft == 1024 ? 16 : 32); }
int lld_max_chunk_tiles() { return 16; }
bool lld_supported_fft(int nfft) { return nfft == 512 || nfft == 1024 || nfft == 2048 || nfft == 4096; }

size_t lld_smem_bytes(const LldParams &p, int nfft)
{
  return (size_t)make_layout(p, nfft / 2, lld_tile_frames(nfft, p.narrow != 0)).total;
}

cudaError_t launch_lld(const LldParams &p, int nfft, int numSMs, cudaStream_t st, LldLaunchInfo *info, bool launch)
{
  {
    static const bool fastOn = [] { const char *e = getenv("OSM_B200_LLD_FAST"); return !(e && e[0] == '0'); }();
    if (fastOn && lld_fast_applies(p, nfft)) return launch_lld_fast(p, numSMs, st, info, launch);
  }
  return p.pcmF32 ? launch_lld_kernel<true>(p, nfft, numSMs, st, info, launch) : launch_lld_kernel<false>(p, nfft, numSMs, st, info, launch);
}

int post_tile_rows(int nStat, int maxN, int halo)
{
  int rows = kPostRows;
  while (rows > 4 && (size_t)(rows + 2 * halo) * (nStat + 2 * maxN) * sizeof(float) > 160 * 1024) rows /= 2;
  return rows;
}

cudaError_t launch_post(const PostParams &p, cudaStream_t st)
{
  if (p.nTiles <= 0 || p.nGroups <= 0) return cudaSuccess;
  if (p.halo > kPostMaxHalo) return cudaErrorInvalidValue;
  const size_t smem = (size_t)(p.rows + 2 * p.halo) * (p.nStat + 2 * p.maxN) * sizeof(float);
  cudaError_t e = cudaFuncSetAttribute(post_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  post_kernel<<<p.nTiles, kPostThreads, smem, st>>>(p);
  return cudaGetLastError();
}

bool acf_pitch_supported_fft(int nfft) { return nfft == 512 || nfft == 1024 || nfft == 2048; }

template <int N, int F, int NT>
static cudaError_t launch_acf_t(const AcfPitchParams &p, cudaStream_t st)
{
  constexpr int NVW = (NT / 32) * (32 / F);
  // FFT tile | twiddles | per-slice partials of the analysis (4 doubles + 3 ints per slice and frame)
  const size_t smem = (((size_t)N * F * 8 + (size_t)p.twCount * 8 + 15) & ~(size_t)15) + (size_t)NVW * F * (4 * 8 + 3 * 4) + 16;
  auto kern = acf_pitch_kernel<N, F, NT>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  kern<<<p.nTiles * (p.F / F), NT, smem, st>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_acf_pitch(const AcfPitchParams &p, cudaStream_t st)
{
  if (p.nTiles <= 0) return cudaSuccess;
  switch (p.nfft) {
    case 512:  return launch_acf_t<512, 32, 512>(p, st);
    case 1024: return launch_acf_t<1024, 16, 512>(p, st);
    case 2048: return launch_acf_t<2048, 8, 256>(p, st);
    default:   return cudaErrorInvalidValue;
  }
}

// ------------------------------------------------------------------------------------------
// cPlp RASTA filter (lldcore/plp.cpp:446-483): a 5-tap FIR + one-pole IIR along time on every band,
// state reset per utterance; the first 5 outputs are forced to 0.  Sequential in time by
// construction -> one thread per (utterance, band); float operations in the reference's order.
// ------------------------------------------------------------------------------------------
__global__ void rasta_kernel(const RastaParams p, int u0, int u1)
{
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int nB = p.nBands;
  const int u = u0 + (int)(idx / nB), b = (int)(idx % nB);
  if (u >= u1) return;
  const long long L = p.uttOff[u + 1] - p.uttOff[u];
  const long long T = frame_count(L, p.frameSize, p.frameStep, p.frameCenter);
  float *x = p.band + p.statOff[u] * nB + b;
  if (p.mode == 1) {
    float fir[5] = {0.f, 0.f, 0.f, 0.f, 0.f};   // circular input history, slot ptr = newest
    float iir = 0.f;
    int ptr = 0;
    for (long long t = 0; t < T; t++) {
      const float s = x[t * nB];
      fir[ptr] = s;
      float sum = __fmul_rn(p.fir[0], s);
#pragma unroll
      for (int m = 1; m < 5; m++) sum = __fadd_rn(sum, __fmul_rn(p.fir[m], fir[(5 - m + ptr) % 5]));
      sum = __fadd_rn(sum, __fmul_rn(p.iir, iir));
      iir = sum;
      x[t * nB] = (t >= 5) ? sum : 0.f;
      ptr = (ptr + 1) % 5;
    }
  } else {
    float b0 = 0.f, b1 = 0.f, b2 = 0.f, b3 = 0.f;
    for (long long t = 0; t < T; t++) {
      const float s = x[t * nB];
      const float out = __fadd_rn(__fmul_rn(p.fir[0], s), b0);
      const float fb = (t >= 5) ? __fmul_rn(p.iir, out) : __fmul_rn(__fmul_rn(0.f, p.iir), out);   // (init>=5) * iir * out
      b0 = __fadd_rn(__fadd_rn(__fmul_rn(p.fir[1], s), b1), fb);
      b1 = __fadd_rn(__fmul_rn(p.fir[2], s), b2);
      b2 = __fadd_rn(__fmul_rn(p.fir[3], s), b3);
      b3 = __fmul_rn(p.fir[4], s);
      x[t * nB] = (t >= 5) ? out : 0.f;
    }
  }
}

cudaError_t launch_rasta(const RastaParams &p, int u0, int u1, cudaStream_t st)
{
  const long long n = (long long)(u1 - u0) * p.nBands;
  if (n <= 0) return cudaSuccess;
  const int bs = 128;
  rasta_kernel<<<(unsigned)((n + bs - 1) / bs), bs, 0, st>>>(p, u0, u1);
  return cudaGetLastError();
}

// rest of cPlp after the RASTA filter (plp.cpp:486-590) for 32 static rows per CTA, lane = frame
constexpr int kTailF = 32, kTailWarps = 4;
__global__ void __launch_bounds__(kTailF * kTailWarps) plp_tail_kernel(const LldParams p, const float *band, float *stat,
                                                                       int statStride, int outCol, long long row0, long long row1)
{
  extern __shared__ __align__(16) unsigned char smem[];
  const int nB = p.nBands;
  float *melS = reinterpret_cast<float *>(smem);                    // [nB][F]
  float *acfS = melS + nB * kTailF;                                 // [nAuto][F]
  float *outS = acfS + (kMaxLp + 1) * kTailF;                       // [nStat][2F]
  const int tid = threadIdx.x, f = tid & 31, vw = tid >> 5;
  const long long r0 = row0 + (long long)blockIdx.x * kTailF;
  const int nf = (int)min((long long)kTailF, row1 - r0);
  for (int idx = tid; idx < nB * kTailF; idx += blockDim.x) {
    const int ff = idx / nB, b = idx - ff * nB;
    float v = 0.f;
    if (ff < nf) {
      v = band[(r0 + ff) * nB + b];
      if (p.plpAud) {                                               // plp.cpp:488-510
        if (p.doLog) {
          v = __fmul_rn(__fadd_rn(v, p.plpEql[b]), p.plpCompression);
        } else {
          if (v < p.melfloor) v = p.melfloor;
          v = __fmul_rn(v, p.plpEql[b]);
          v = (float)pow((double)v, (double)p.plpCompression);
        }
      }
      if (p.plpInvLog) v = expf(v);                                 // :513-518
    }
    melS[b * kTailF + ff] = v;
  }
  __syncthreads();
  plp_backend<kTailF, kTailWarps>(p, melS, p.dctCos, p.dctLift, acfS, outS, vw, f);
  __syncthreads();
  for (int idx = tid; idx < nf * p.nStat; idx += blockDim.x) {
    const int ff = idx / p.nStat, c = idx - ff * p.nStat;
    stat[(r0 + ff) * statStride + outCol + c] = outS[c * (2 * kTailF) + ff];
  }
}

cudaError_t launch_plp_tail(const LldParams &op, const float *band, float *stat, int statStride, int outCol,
                            long long row0, long long row1, cudaStream_t st)
{
  if (row1 <= row0) return cudaSuccess;
  const size_t smem = (size_t)(op.nBands + kMaxLp + 1 + 2 * op.nStat) * kTailF * sizeof(float);
  cudaError_t e = cudaFuncSetAttribute(plp_tail_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  const long long nb = (row1 - row0 + kTailF - 1) / kTailF;
  plp_tail_kernel<<<(unsigned)nb, kTailF * kTailWarps, smem, st>>>(op, band, stat, statStride, outCol, row0, row1);
  return cudaGetLastError();
}

// cFullinputMean, single-loop mode (dspcore/fullinputMean.cpp:526-546): means = first frame, += every
// further frame (float, frame order), /= (float)n at EOI.  One thread per (utterance, column of a group
// that ends in a mean subtraction); T follows the group's reader (min over its levels' streams).
__global__ void cms_mean_kernel(const PostParams p, float *means, int u0, int u1)
{
  const int u = u0 + blockIdx.x;
  if (u >= u1) return;
  const long long Ls = p.uttOff[u + 1] - p.uttOff[u];
  const float *src = p.stat + p.statOff[u] * (long long)p.statStride;
  for (int gi = 0; gi < p.nGroups; gi++) {
    const PostGroup &g = p.groups[gi];
    if (g.nStages < 1 || g.kind[g.nStages - 1] != 2) continue;
    int T = (int)frame_count(Ls, g.frameSize, g.frameStep, g.frameCenter);
    for (int k = 0; k < g.nLim; k++) T = min(T, (int)frame_count(Ls, g.limSize[k], g.limStep[k], g.limCenter[k]));
    for (int c = threadIdx.x; c < g.n; c += blockDim.x) {
      float m = 0.f;
      if (T > 0) {
        m = src[g.srcCol + c];
        for (int t = 1; t < T; t++) m = __fadd_rn(m, src[(long long)t * p.statStride + g.srcCol + c]);
        m = __fdiv_rn(m, (float)T);
      }
      means[(long long)u * p.nStat + g.srcCol + c] = m;
    }
  }
}

cudaError_t launch_cms_means(const PostParams &p, float *means, int u0, int u1, cudaStream_t st)
{
  if (u1 <= u0) return cudaSuccess;
  cms_mean_kernel<<<u1 - u0, 64, 0, st>>>(p, means, u0, u1);
  return cudaGetLastError();
}

__global__ void vecop_ll1_kernel(float *stat, int statStride, int srcCol, int n, int outCol, long long row0, long long row1)
{
  const long long r = row0 + (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= row1) return;
  const float *x = stat + r * statStride + srcCol;
  float d = 0.f;
  for (int i = 0; i < n; i++) d = __fadd_rn(d, x[i]);               // vectorOperation.cpp:475-481
  if (n > 0) d = __fdiv_rn(d, (float)n);
  stat[r * statStride + outCol] = d;
}

cudaError_t launch_vecop_ll1(float *stat, int statStride, int srcCol, int n, int outCol, long long row0, long long row1,
                             cudaStream_t st)
{
  if (row1 <= row0) return cudaSuccess;
  const int bs = 128;
  vecop_ll1_kernel<<<(unsigned)((row1 - row0 + bs - 1) / bs), bs, 0, st>>>(stat, statStride, srcCol, n, outCol, row0, row1);
  return cudaGetLastError();
}

cudaError_t launch_pitch_smooth(const AcfPitchParams &p, int u0, int u1, cudaStream_t st)
{
  if (u1 <= u0) return cudaSuccess;
  const int bs = 64;
  pitch_smooth_kernel<<<(u1 - u0 + bs - 1) / bs, bs, 0, st>>>(p, u0, u1);
  return cudaGetLastError();
}

}  // namespace osm
