// harmonics.cu -- cHarmonics (lld/harmonics.cpp:743-900) for the switch set of the GeMAPS graphs (sm_90a):
// reads, per frame t, the F0 of the Viterbi-smoothed pitch level, the formant frequencies of the cFormantLpc level
// (static rows of this plan) and the 60 ms magnitude spectrum (tile-major level in HBM), writes
//   [HarmonicsToNoiseRatioACFLogdB] | HarmonicDifferenceLogRel* | FormantAmplitudeByMaxHarmonicLogRelF0[start..end].
// One warp per frame (CTA = one tile of the magnitude level, 8 frames at a time):
//   - the frame's magnitudes are transposed into shared memory once;
//   - HNR: the reference takes an inverse FFT of the whole power spectrum and then looks at a handful of lags around
//     fs / F0 (getClosestPeak).  Only those lags are evaluated here, each as a cosine sum over the bins with the lanes
//     of the warp striding the bins (double accumulation, table of cos(2 pi m / N)); every lane holds the reduced
//     value, so the peak search runs uniformly on all lanes;
//   - harmonic peak search with one lane per harmonic (the reference's "start at the previous harmonic's bin" never binds on
//     a linear frequency axis; checked per frame, sequential fallback), log magnitudes per lane, warp arg-max per formant.
// Compiled with -fmad=false.
#include "kernels.cuh"
#include "harmonics_math.cuh"

namespace osm {

namespace {

constexpr int kHmWarps = 8;
constexpr int kHmThreads = kHmWarps * 32;

struct MagS { const float *m; __device__ __forceinline__ float operator()(int b) const { return m[b]; } };

// warp-collective autocorrelation lag j of the power spectrum (computeAcf, lld/harmonics.cpp:590-630, as a cosine sum):
// |p0/2 + p(N/2)/2 (-1)^j + sum_{k=1}^{N/2-1} p_k cos(2 pi j k / N)| / nb, p_k = mag_k^2 (float product)
struct AcfWarp {
  const float *m; int nb, N; const double *cosTab; int lane;
  // The peak search probes neighbouring lags again and again (isPeak reads x(n) twice and x(n-1), x(n+1); the outward walk then
  // moves by one): the last four lags are kept.  Every lane holds the same (lag, value) pairs, so the look-up is warp uniform.
  mutable int cj0 = -1, cj1 = -1, cj2 = -1, cj3 = -1, nextSlot = 0;
  mutable float cv0 = 0.f, cv1 = 0.f, cv2 = 0.f, cv3 = 0.f;
  __device__ __forceinline__ float operator()(int j) const
  {
    if (j == cj0) return cv0;
    if (j == cj1) return cv1;
    if (j == cj2) return cv2;
    if (j == cj3) return cv3;
    double s = 0.0;
    for (int k = 1 + lane; k < N / 2; k += 32) s += (double)(m[k] * m[k]) * cosTab[(j * k) & (N - 1)];
    if (lane == 0) s += 0.5 * (double)(m[0] * m[0]) + 0.5 * (double)(m[N / 2] * m[N / 2]) * ((j & 1) ? -1.0 : 1.0);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float v = (float)fabs(s) / (float)nb;
    if (nextSlot == 0) { cj0 = j; cv0 = v; } else if (nextSlot == 1) { cj1 = j; cv1 = v; } else if (nextSlot == 2) { cj2 = j; cv2 = v; } else { cj3 = j; cv3 = v; }
    nextSlot = (nextSlot + 1) & 3;
    return v;
  }
};

__global__ void __launch_bounds__(kHmThreads) harmonics_kernel(const HarmonicsParams p)
{
  extern __shared__ __align__(16) unsigned char hmSmem[];
  const int nb = p.nb, N = (nb - 1) * 2;
  const int nbP = nb + 1;                                      // odd pitch: the transposing stores spread over the banks
  float *magS = reinterpret_cast<float *>(hmSmem);             // [kHmWarps][nbP]
  hm::Harm *HS = reinterpret_cast<hm::Harm *>(magS + (size_t)kHmWarps * nbP);   // [kHmWarps][nHarm]
  const OpTile tl = p.tiles[blockIdx.x];
  const float *tile = p.mag + (size_t)blockIdx.x * nb * p.F;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  for (int fb = 0; fb < tl.nf; fb += kHmWarps) {
    const int nf = min(kHmWarps, tl.nf - fb);
    for (int idx = tid; idx < nb * kHmWarps; idx += kHmThreads) {
      const int b = idx / kHmWarps, f = idx % kHmWarps;
      if (f < nf) magS[f * nbP + b] = tile[(size_t)b * p.F + fb + f];
    }
    __syncthreads();
    if (warp < nf) {
      const float *m = magS + warp * nbP;
      const long long row = p.statOff[tl.utt] + tl.f0 + fb + warp;
      float *srow = p.stat + row * (long long)p.statStride;
      const float F0 = srow[p.f0Col];
      float *dst = srow + p.outCol;
      int o = 0;
      if (p.doHnr) {
        AcfWarp A{m, nb, N, p.cosTab, lane};
        const double fs = (double)(nb - 1) * p.binHz * 2.0;
        const int f0bin = F0 > 0.0f ? (int)floor(fs / (double)F0) : 0;       // freqToAcfBinLin (:393-401)
        int ref = 0;
        if (f0bin > 0) ref = hm::closest_peak(A, nb, f0bin);
        float v = 0.0f;
        if (ref > 0) { const float a0 = A(0), ar = A(ref); v = hm::hnr_db(a0, ar); }
        if (lane == 0) dst[o] = v;
        o++;
      }
      if (F0 > 0.0f) {
        // Harmonic peaks, lane = harmonic (i = lane, lane + 32, ...).  The reference searches harmonic i upward from the
        // candidate bin of harmonic i-1 (freqToBin's start argument).  On the linear axis that lower bound never binds
        // (candidate i-1 <= first bin above (i f0) <= the bin freqToBin finds for any later frequency), so every lane takes
        // its predecessor's candidate from the closed form; each lane checks that its own candidate equals that closed form,
        // and if any lane disagrees the warp falls back to the sequential statements on lane 0.
        hm::Harm *H = HS + (size_t)warp * p.nHarm;
        MagS M{m};
        const int last0 = hm::freq_to_bin(p.binHz, nb, 0.5f * F0, 1);
        const int first = hm::freq_to_bin(p.binHz, nb, 0.5f * F0, last0);
        bool consistent = true;
        for (int i = lane; i < p.nHarm; i += 32) {
          const int prev = i == 0 ? last0 : hm::freq_to_bin(p.binHz, nb, (float)i * F0, 0);
          hm::Harm h;
          const int cand = hm::find_one_harmonic(F0, M, nb, p.binHz, i, prev, first, &h);
          consistent = consistent && cand == hm::freq_to_bin(p.binHz, nb, (float)(i + 1) * F0, 0);
          H[i] = h;
        }
        consistent = __all_sync(0xffffffffu, consistent);
        __syncwarp();
        if (!consistent) {
          if (lane == 0) hm::find_harmonics(F0, M, nb, p.binHz, p.nHarm, H);
        } else {
          const float m0 = H[0].mag;
          const bool logRel = m0 != 0.0f;
          const float m0log = logRel ? log10f(m0) : 0.0f;
          __syncwarp();
          for (int i = lane; i < p.nHarm; i += 32) H[i].lr = i == 0 ? 0.0f : hm::log_rel(H[i].magi, logRel, m0log);
          __syncwarp();
          if (lane == 0) hm::dedup(H, p.nHarm);
        }
        __syncwarp();
        // strongest harmonic within +-20 % of each formant (getFormantAmplitudeIndices): lanes stride the harmonics, warp
        // arg-max with the lowest index among equal magnitudes (the sequential scan keeps the first of the largest)
        int fa[hm::kMaxFormants];
        for (int k = 0; k < p.nFmt; k++) {
          const float f = srow[p.fmtCol + k], lo = 0.8f * f, hi = 1.2f * f;
          int best = -1;
          float bm = 0.0f;
          for (int h = lane; h < p.nHarm; h += 32)
            if (lo <= H[h].fi && H[h].fi <= hi && H[h].mag > bm) { best = h; bm = H[h].mag; }
#pragma unroll
          for (int off = 16; off > 0; off >>= 1) {
            const float om = __shfl_xor_sync(0xffffffffu, bm, off);
            const int ob = __shfl_xor_sync(0xffffffffu, best, off);
            if (ob >= 0 && (best < 0 || om > bm || (om == bm && ob < best))) { bm = om; best = ob; }
          }
          fa[k] = best;
        }
        if (lane == 0) {
          for (int i = 0; i < p.nDiffs; i++)
            dst[o++] = hm::harmonic_difference(H, p.nHarm, fa, p.nFmt, hm::Diff{p.diffs[4 * i], p.diffs[4 * i + 1], p.diffs[4 * i + 2], p.diffs[4 * i + 3]});
          if (p.doFa) for (int k = p.faStart; k <= p.faEnd; k++) dst[o++] = (k >= 1 && k <= p.nFmt && fa[k - 1] >= 0) ? H[fa[k - 1]].lr : 0.0f;
        }
      } else if (lane == 0) {
        for (int i = 0; i < p.nDiffs; i++) dst[o++] = 0.0f;
        if (p.doFa) for (int k = p.faStart; k <= p.faEnd; k++) dst[o++] = p.floorUnvoiced;
      }
    }
    __syncthreads();
  }
}

}  // namespace

size_t harmonics_smem_bytes(const HarmonicsParams &p)
{
  return (size_t)kHmWarps * (p.nb + 1) * sizeof(float) + (size_t)kHmWarps * p.nHarm * sizeof(hm::Harm);
}

cudaError_t launch_harmonics(const HarmonicsParams &p, cudaStream_t st)
{
  if (p.nTiles <= 0) return cudaSuccess;
  const size_t smem = harmonics_smem_bytes(p);
  if (smem > 48 * 1024) {   // per device / context attribute: set on every launch like the other launchers
    cudaError_t e = cudaFuncSetAttribute(harmonics_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  harmonics_kernel<<<p.nTiles, kHmThreads, smem, st>>>(p);
  return cudaGetLastError();
}

}  // namespace osm
