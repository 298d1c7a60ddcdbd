// lsp.cu -- stand-alone cLpc (method acf) and cLsp on a time-domain frame level (sm_90a), e.g. emobase's
//   cFramer -> cVectorPreemphasis -> cLpc (p = 8) -> cLsp
// cLpc and cLsp are cVectorProcessors: one output frame per input frame, so the op writes columns of the static rows of
// the frame level's stream.  One CTA per tile of frames:
//   1. one warp per frame: the (pre-emphasised) frame is staged in shared memory, lanes 0..p each sum one autocorrelation
//      lag in the reference's sequential float order (formant_math.cuh acf_lag, smileutil/smileUtil.c:1560-1569);
//   2. one thread per frame: Levinson-Durbin (formant_math.cuh durbin, :1572-1627) and, for a cLsp level, the LSP root
//      search (lsp_math.cuh, lld/lsp.cpp:113-313).
// Compiled with -fmad=false: the float recursions keep the reference's statement order.
#include "kernels.cuh"
#include "frame_reader.cuh"
#include "formant_math.cuh"
#include "lsp_math.cuh"

namespace osm {

namespace {

constexpr int kLpcWarps = 8;
constexpr int kLpcThreads = kLpcWarps * 32;

template <bool F32>
__global__ void __launch_bounds__(kLpcThreads) lpc_kernel(const LpcParams p)
{
  extern __shared__ __align__(16) float lpcSmem[];
  const TimeOpParams &tp = p.tp;
  const int N = tp.frameSize, P = p.p;
  float *xs = lpcSmem + (size_t)(threadIdx.x >> 5) * N;                 // [kLpcWarps][N] staged frames
  float *rs = lpcSmem + (size_t)kLpcWarps * N;                          // [F][P + 1] autocorrelations
  const OpTile tl = tp.tiles[blockIdx.x];
  const long long uo = tp.uttOff[tl.utt];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int f = warp; f < tl.nf; f += kLpcWarps) {
    FrameReader<F32> fr{tp, tp.pcm + uo * tp.nChan, frame_first_sample(tl.f0 + f, tp.frameStep, tp.frameCenter)};
    for (int n = lane; n < N; n += 32) xs[n] = tp.windowed ? fr.at(n) : fr.pre(n);
    __syncwarp();
    if (lane <= P) rs[f * (P + 1) + lane] = fm::acf_lag(xs, N, lane);
    __syncwarp();
  }
  __syncthreads();
  for (int f = threadIdx.x; f < tl.nf; f += kLpcThreads) {
    float a[fm::kMaxLpcOrder];
    const float gain = fm::durbin(rs + f * (P + 1), P, a);               // lld/lpc.cpp:156-168
    float *dst = tp.stat + (tp.statOff[tl.utt] + tl.f0 + f) * (long long)tp.statStride + tp.outCol;
    int o = 0;
    if (p.outLpc) for (int i = 0; i < P; i++) dst[o++] = a[i];          // :189-194
    if (p.outGain) dst[o++] = gain;                                      // :197-200
    if (p.outLsp) {
      float lsf[lsp::kMaxOrder];
      lsp::lsp_from_lpc(a, P, lsf);
      for (int i = 0; i < P; i++) dst[o++] = lsf[i];
    }
  }
}

}  // namespace

size_t lpc_smem_bytes(const LpcParams &p)
{
  return ((size_t)kLpcWarps * p.tp.frameSize + (size_t)p.tp.F * (p.p + 1)) * sizeof(float);
}

cudaError_t launch_lpc(const LpcParams &p, cudaStream_t st)
{
  if (p.tp.nTiles <= 0) return cudaSuccess;
  const size_t smem = lpc_smem_bytes(p);
  auto kern = p.tp.pcmF32 ? lpc_kernel<true> : lpc_kernel<false>;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  kern<<<p.tp.nTiles, kLpcThreads, smem, st>>>(p);
  return cudaGetLastError();
}

}  // namespace osm
