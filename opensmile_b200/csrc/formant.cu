// formant.cu -- the formant chain of the GeMAPS graphs as one kernel (sm_90a):
//   cWindower level -> [cTransformFFT -> cSpecResample] -> cLpc (acf) -> cFormantLpc        (SURVEY.md 8f-2)
//
// The reference transforms every windowed frame (zero padded to the FFT size), and cSpecResample evaluates an
// inverse DFT of the low bins on a coarser time grid (dsp/specResample.cpp:175-185, smileDsp_irdft
// smileutil/smileUtil.c:1800-1820).  Both steps are linear and no other component reads that FFT level's
// resampled copy, so the kernel applies their composition directly: res[i] = sum_m xw[m] * D[m][i] with the
// table D built in double on the host (tables.cpp build_formant).  That is one dense [frames x N] * [N x I]
// product per tile -- fp32 FMA on purpose: order-11 LPC amplifies input noise of 1e-7 to ~1e-2 in the formants
// (DESIGN.md), so reduced-precision tensor-core formats are not an option here.
// Then one warp per frame: autocorrelation (one lane per lag, the reference's float summation order), Levinson-
// Durbin on lane 0, the roots of the predictor polynomial with one lane per root (formant_math.cuh), and the
// formant frequencies / bandwidths of the roots in the upper half plane.
// Compiled with -fmad=false: the float recursions keep the reference's statement order.
#include "kernels.cuh"
#include "frame_reader.cuh"
#include "formant_math.cuh"
#include "fft_ref_order.cuh"

namespace osm {

namespace {

using fm::kFmtWarps;                       // CTA shape and scratch: formant_math.cuh (the graph pass sizes the shared memory)
using fm::kFmtFpw;
using fm::kFmtBatch;
using fm::FmtWarpWs;
constexpr int kFmtThreads = kFmtWarps * 32;

template <bool F32>
__global__ void __launch_bounds__(kFmtThreads) formant_kernel(const FormantParams p)
{
  extern __shared__ __align__(16) unsigned char fmtSmem[];
  const TimeOpParams &tp = p.tp;
  const int N = tp.frameSize, I = p.nRes, IP = p.nResPad;
  FmtWarpWs *ws = reinterpret_cast<FmtWarpWs *>(fmtSmem);
  float *xw = reinterpret_cast<float *>(ws + kFmtBatch);        // [kFmtWarps][N]
  float *res0 = xw + (size_t)kFmtWarps * (p.refOrder ? 4 * ro::kPlane : N);  // [kFmtBatch][IP]
  const OpTile tl = tp.tiles[blockIdx.x];
  const long long uo = tp.uttOff[tl.utt];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  // two frames per warp need a half warp per frame: one lane per lag 0..p
  const int fpw = (p.p + 1 <= 16) ? kFmtFpw : 1;
  for (int fb0 = 0; fb0 < tl.nf; fb0 += kFmtWarps * fpw) {
   // transform + resampling in batches of kFmtWarps frames; the per-frame phase then takes fpw batches at once
   for (int part = 0; part < fpw; part++) {
    const int fb = fb0 + part * kFmtWarps;
    const int nb = min(kFmtWarps, tl.nf - fb);
    if (nb <= 0) break;
    float *res = res0 + (size_t)part * kFmtWarps * IP;
    if (p.refOrder) {
      // Reference-order path (fft_ref_order.cuh): the zero padded windowed frame goes through a 512-point real FFT with the
      // reference's rounding sequence; then cSpecResample's inverse sum over the reference's float tables, in its order.
      float *planes = xw;                                        // [kFmtWarps][4][kPlane]: in / out, real / imaginary
      const float *wc = p.D, *cosT = p.D + ro::kNw + ro::kNc, *sinT = cosT + (size_t)p.kHalf * IP;
      for (int f = 0; f < nb; f++) {
        FrameReader<F32> fr{tp, tp.pcm + uo * tp.nChan, frame_first_sample(tl.f0 + fb + f, tp.frameStep, tp.frameCenter)};
        float *re = planes + (size_t)f * 4 * ro::kPlane, *im = re + ro::kPlane;
        for (int n = tid; n < ro::kN; n += kFmtThreads) {
          const int m = n - p.padLeft;
          const float v = (m >= 0 && m < N) ? fr.at(m) : 0.0f;
          ((n & 1) ? im : re)[ro::phys(n >> 1)] = v;
        }
      }
      __syncthreads();
      auto frame_planes = [&](int f, int which) { float *b = planes + ((size_t)f * 4 + 2 * which) * ro::kPlane; return ro::Planes{b, b + ro::kPlane}; };
      for (int it = tid; it < ro::kItemsA * nb; it += kFmtThreads) ro::phase_a(frame_planes(it / ro::kItemsA, 0), wc, it % ro::kItemsA);
      __syncthreads();
      for (int it = tid; it < ro::kItemsB * nb; it += kFmtThreads) ro::phase_b(frame_planes(it / ro::kItemsB, 0), wc, it % ro::kItemsB);
      __syncthreads();
      for (int it = tid; it < ro::kItemsC * nb; it += kFmtThreads) ro::phase_c(frame_planes(it / ro::kItemsC, 0), wc, it % ro::kItemsC);
      __syncthreads();
      for (int it = tid; it < ro::kItemsD * nb; it += kFmtThreads)
        ro::phase_d(frame_planes(it / ro::kItemsD, 0), frame_planes(it / ro::kItemsD, 1), wc + ro::kNw, it % ro::kItemsD);
      __syncthreads();
      // smileDsp_irdft (smileutil/smileUtil.c:1800-1820): out = DC; out += Re_k cos; out += Im_k sin (k ascending); out /= K/2
      // The bins the sum reads are first gathered per bin as (Re of the 8 frames | Im of the 8 frames) into the transform's input
      // planes, which are dead now (34 rows of 16 floats in each of the first four frames' input planes): the sum then reads four
      // 128-bit words per bin instead of sixteen scalars.  Same operands, same order per frame.
      constexpr int kRowsPerPiece = (2 * ro::kPlane) / 16;
      const bool gathered = p.kHalf <= 4 * kRowsPerPiece;
      if (gathered) {
        for (int idx = tid; idx < p.kHalf * 16; idx += kFmtThreads) {
          const int k2 = idx >> 4, c = idx & 15, f = c & 7, im = c >> 3;
          planes[(size_t)(k2 / kRowsPerPiece) * 4 * ro::kPlane + (k2 % kRowsPerPiece) * 16 + c] =
              planes[((size_t)f * 4 + 2 + im) * ro::kPlane + ro::phys(k2)];
        }
        __syncthreads();
      }
      for (int i = tid; i < I; i += kFmtThreads) {
        float acc[kFmtWarps];
        if (gathered) {
          {
            const float4 *r4 = reinterpret_cast<const float4 *>(planes);                 // bin 0: DC of every frame
            const float4 a = r4[0], b = r4[1];
            acc[0] = a.x; acc[1] = a.y; acc[2] = a.z; acc[3] = a.w; acc[4] = b.x; acc[5] = b.y; acc[6] = b.z; acc[7] = b.w;
          }
          const float *row = planes + 16;
          int within = 1;
          for (int k2 = 1; k2 < p.kHalf; k2++) {
            const float cv = __ldg(cosT + (size_t)k2 * IP + i), sv = __ldg(sinT + (size_t)k2 * IP + i);
            const float4 *r4 = reinterpret_cast<const float4 *>(row);
            const float4 re0 = r4[0], re1 = r4[1], im0 = r4[2], im1 = r4[3];
            acc[0] = __fadd_rn(acc[0], __fmul_rn(re0.x, cv)); acc[0] = __fadd_rn(acc[0], __fmul_rn(im0.x, sv));
            acc[1] = __fadd_rn(acc[1], __fmul_rn(re0.y, cv)); acc[1] = __fadd_rn(acc[1], __fmul_rn(im0.y, sv));
            acc[2] = __fadd_rn(acc[2], __fmul_rn(re0.z, cv)); acc[2] = __fadd_rn(acc[2], __fmul_rn(im0.z, sv));
            acc[3] = __fadd_rn(acc[3], __fmul_rn(re0.w, cv)); acc[3] = __fadd_rn(acc[3], __fmul_rn(im0.w, sv));
            acc[4] = __fadd_rn(acc[4], __fmul_rn(re1.x, cv)); acc[4] = __fadd_rn(acc[4], __fmul_rn(im1.x, sv));
            acc[5] = __fadd_rn(acc[5], __fmul_rn(re1.y, cv)); acc[5] = __fadd_rn(acc[5], __fmul_rn(im1.y, sv));
            acc[6] = __fadd_rn(acc[6], __fmul_rn(re1.z, cv)); acc[6] = __fadd_rn(acc[6], __fmul_rn(im1.z, sv));
            acc[7] = __fadd_rn(acc[7], __fmul_rn(re1.w, cv)); acc[7] = __fadd_rn(acc[7], __fmul_rn(im1.w, sv));
            row += 16;
            if (++within == kRowsPerPiece) { within = 0; row += 4 * ro::kPlane - kRowsPerPiece * 16; }
          }
        } else {
#pragma unroll
          for (int f = 0; f < kFmtWarps; f++) acc[f] = planes[((size_t)f * 4 + 2) * ro::kPlane];
          for (int k2 = 1; k2 < p.kHalf; k2++) {
            const float cv = __ldg(cosT + (size_t)k2 * IP + i), sv = __ldg(sinT + (size_t)k2 * IP + i);
            const int ph = ro::phys(k2);
#pragma unroll
            for (int f = 0; f < kFmtWarps; f++) {
              const float *b = planes + ((size_t)f * 4 + 2) * ro::kPlane;
              acc[f] = __fadd_rn(acc[f], __fmul_rn(b[ph], cv));
              acc[f] = __fadd_rn(acc[f], __fmul_rn(b[ro::kPlane + ph], sv));
            }
          }
        }
#pragma unroll
        for (int f = 0; f < kFmtWarps; f++) res[f * IP + i] = __fdiv_rn(acc[f], p.halfK);
      }
      __syncthreads();
    } else {
    // 1. windowed frames (dspcore/windower.cpp:226) into shared memory
    for (int f = 0; f < nb; f++) {
      FrameReader<F32> fr{tp, tp.pcm + uo * tp.nChan, frame_first_sample(tl.f0 + fb + f, tp.frameStep, tp.frameCenter)};
      for (int m = tid; m < N; m += kFmtThreads) xw[f * N + m] = fr.at(m);
    }
    __syncthreads();
    // 2. resampled frames: thread i owns output sample i of all frames of the batch
    for (int i = tid; i < I; i += kFmtThreads) {
      float acc[kFmtWarps];
#pragma unroll
      for (int f = 0; f < kFmtWarps; f++) acc[f] = 0.0f;
      const float *dcol = p.D + i;
      for (int m = 0; m < N; m++) {
        const float dv = __ldg(dcol + (size_t)m * IP);
#pragma unroll
        for (int f = 0; f < kFmtWarps; f++) acc[f] = __fmaf_rn(xw[f * N + m], dv, acc[f]);
      }
#pragma unroll
      for (int f = 0; f < kFmtWarps; f++) res[f * IP + i] = acc[f];
    }
    __syncthreads();
    }
   }
    // 3. one (half) warp per frame
    {
      const int h = (fpw == 2) ? (lane >> 4) : 0, hl = (fpw == 2) ? (lane & 15) : lane;
      const unsigned hm = (fpw == 2) ? (0xffffu << (16 * h)) : 0xffffffffu;
      const int fi = warp * fpw + h;                                   // frame of the batch [fb0, fb0 + kFmtWarps * fpw)
      const int part = fi / kFmtWarps, fin = fi - part * kFmtWarps;    // resampled by batch `part` as its frame `fin`
      // frames are dealt so that a warp's two frames come from the two batches: fi -> (part, fin) below keeps res contiguous
      // The sequential per-frame steps (Durbin recursion, candidate selection / sort / store) run as "one LANE per frame" on the
      // first warp for the whole batch of frames -- one instruction stream for up to 16 frames instead of one per half warp with a
      // single active lane (ncu: those two steps were 45 % of the kernel's warp-instructions) -- the steps with per-frame
      // parallelism (autocorrelation lags, the simultaneous root refinement) stay "one half warp per frame".
      const bool live = fb0 + fi < tl.nf;
      FmtWarpWs &w = ws[live ? fi : 0];
      const int P = p.p;
      auto lpc_setup = [&](FmtWarpWs &q) {
        fm::durbin(q.r, P, q.a);
        for (int i = 0; i < P; i++) q.c[i] = -(double)q.a[P - 1 - i];  // lld/formantLpc.cpp:258-262
        int z0 = 0;
        while (z0 < P && q.c[z0] == 0.0) z0++;                         // roots at the origin yield no candidate
        q.z0 = z0; q.n = P - z0;
      };
      auto emit = [&](FmtWarpWs &q, int frameInBatch) {
        // smileDsp_lpcrootsToFormants (smileutil/smileUtil.c:2019-2054): candidates in root order, then the
        // ascending sort of lld/formantLpc.cpp:277-296 over the leading non-zero entries
        double f[fm::kMaxLpcOrder], b[fm::kMaxLpcOrder];
        const int nF = p.nFormants, n = q.n;
        int nv = 0;
        for (int k = 0; k < n && nv < nF; k++) if (q.ok[k]) { f[nv] = q.f[k]; b[nv] = q.b[k]; nv++; }
        for (int i = nv; i < nF; i++) { f[i] = 0.0; b[i] = 0.0; }
        int nz = 0;
        while (nz < nF && f[nz] != 0.0) nz++;
        for (int i = 0; i < nz; i++)
          for (int j = i + 1; j < nz; j++)
            if (f[j] < f[i]) { double t = f[j]; f[j] = f[i]; f[i] = t; t = b[j]; b[j] = b[i]; b[i] = t; }
        float *dst = tp.stat + (tp.statOff[tl.utt] + tl.f0 + fb0 + frameInBatch) * (long long)tp.statStride + tp.outCol;
        int o = 0;
        if (p.saveNValid) dst[o++] = (float)nv;                        // lld/formantLpc.cpp:376-392
        if (p.saveFormants) for (int i = 0; i < nF; i++) dst[o++] = (float)f[i];
        if (p.saveBandwidths) for (int i = 0; i < nF; i++) dst[o++] = (float)b[i];
      };
      if (live) {
        const float *x = res0 + ((size_t)part * kFmtWarps + fin) * IP;
        if (hl <= P) w.r[hl] = fm::acf_lag(x, I, hl);                  // lld/lpc.cpp:156-215 (method acf)
      }
      __syncthreads();
      if (warp == 0 && lane < kFmtWarps * fpw && fb0 + lane < tl.nf) lpc_setup(ws[lane]);
      __syncthreads();
      if (live) {
      const int n = w.n;
      const double *c = w.c + w.z0;
      double zr = 0.0, zi = 0.0, prev = 1e300;
      if (hl < n) { fm::aberth_init(c, n, hl, &zr, &zi); w.zr[hl] = zr; w.zi[hl] = zi; }
      __syncwarp(hm);
      bool last = false;
      for (int it = 0; it < fm::kAberthMaxIter && n > 0; it++) {
        bool done = true;
        if (hl < n) {
          const double c2 = fm::aberth_step(c, n, w.zr, w.zi, hl, &zr, &zi);
          done = fm::aberth_done(c2, prev, zr, zi);
          prev = c2;
        }
        __syncwarp(hm);
        if (hl < n) { w.zr[hl] = zr; w.zi[hl] = zi; }
        const bool all = __all_sync(hm, done);
        __syncwarp(hm);
        if (last) break;
        last = all;
      }
      if (hl < n) {
        double f = 0.0, b = 0.0;
        w.ok[hl] = fm::root_to_formant(zr, zi, p.T, p.minF, p.maxF, &f, &b) ? 1 : 0;
        w.f[hl] = f; w.b[hl] = b;
      }
      }
      __syncthreads();
      if (warp == 0 && lane < kFmtWarps * fpw && fb0 + lane < tl.nf) emit(ws[lane], lane);
    }
    __syncthreads();
  }
}

}  // namespace

size_t formant_smem_bytes(const FormantParams &p)
{
  return fm::formant_smem_bytes(p.refOrder != 0, p.tp.frameSize, p.nResPad);
}

cudaError_t launch_formant(const FormantParams &p, cudaStream_t st)
{
  if (p.tp.nTiles <= 0) return cudaSuccess;
  const size_t smem = formant_smem_bytes(p);
  auto kern = p.tp.pcmF32 ? formant_kernel<true> : formant_kernel<false>;
  if (smem > 48 * 1024) {   // per device / context attribute: set on every launch like the other launchers
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  kern<<<p.tp.nTiles, kFmtThreads, smem, st>>>(p);
  return cudaGetLastError();
}

}  // namespace osm
