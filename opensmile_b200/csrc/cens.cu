// cens.cu -- cCens (lld/cens.cpp:139-222) on the columns of a cChroma op of the static level (sm_90a, built with -fmad=false).
//
// Every output row depends only on the quantised rows t-W+1 .. t of its utterance, so the rows are independent: one CTA per tile
// of up to kCensRows rows of one utterance.  The CTA quantises its rows and the W-1 rows of left halo once into shared memory
// (bytes: q is 0..4), then one thread per (row, element) runs the window in the reference's order (float, j ascending, from 0),
// one thread per row takes the double norm, and the normalised values overwrite the CENS columns of the static level.  Rows
// before the utterance start are the zeros of the reference's calloc'd ring buffer.  The tiles are cut from each utterance's
// own length (prepare_batch), so a row's value does not depend on the batch.
#include "kernels.cuh"

namespace osm {

namespace {

constexpr int kCensThreads = 256;

// chromaDiscretise (:139-149): float against double constants
__device__ __forceinline__ unsigned char cens_quantise(float x)
{
  const double v = (double)x;
  return v >= 0.4 ? 4 : (v >= 0.2 ? 3 : (v >= 0.1 ? 2 : (v >= 0.05 ? 1 : 0)));
}

__global__ void __launch_bounds__(kCensThreads) cens_kernel(const CensParams p)
{
  extern __shared__ __align__(16) unsigned char csm[];
  const int N = p.N, W = p.W;
  float *sWin = reinterpret_cast<float *>(csm);                 // [W]
  float *sAcc = sWin + W;                                       // [kCensRows][N]
  float *sNorm = sAcc + kCensRows * N;                          // [kCensRows] (float)sqrt(n), -1 = not n > 0
  unsigned char *sQ = reinterpret_cast<unsigned char *>(sNorm + kCensRows);   // [kCensRows + W - 1][N]
  const OpTile tl = p.tiles[blockIdx.x];
  const int tid = threadIdx.x;
  const long long base = p.statOff[tl.utt];
  const int r0 = tl.f0 - (W - 1);                               // row of sQ row 0
  for (int j = tid; j < W; j += kCensThreads) sWin[j] = p.win[j];
  const int nq = (tl.nf + W - 1) * N;
  for (int idx = tid; idx < nq; idx += kCensThreads) {
    const int rr = idx / N, c = idx - rr * N;
    const int r = r0 + rr;
    sQ[idx] = r >= 0 ? cens_quantise(p.stat[(base + r) * p.statStride + p.srcCol + c]) : (unsigned char)0;
  }
  __syncthreads();
  // :180-187: _buf[i] = 0; _buf[i] += q[t-j][i] * (float)win[j], j = 0 .. W-1
  const int nOut = tl.nf * N;
  for (int idx = tid; idx < nOut; idx += kCensThreads) {
    const int i = idx / N, c = idx - i * N;
    const unsigned char *q = sQ + (i + W - 1) * N + c;
    float acc = 0.0f;
    for (int j = 0; j < W; j++) acc = __fadd_rn(acc, __fmul_rn((float)q[-j * N], sWin[j]));
    if (p.l2norm) sAcc[idx] = acc;
    else p.stat[(base + tl.f0 + i) * p.statStride + p.outCol + c] = acc;      // :209-214
  }
  if (!p.l2norm) return;
  __syncthreads();
  // :192-201: n = sum (double)x^2 in element order; n > 0: x / (float)sqrt(n)
  for (int i = tid; i < tl.nf; i += kCensThreads) {
    double n = 0.0;
    for (int c = 0; c < N; c++) {
      const double a = (double)sAcc[i * N + c];
      n = __dadd_rn(n, __dmul_rn(a, a));
    }
    sNorm[i] = n > 0.0 ? (float)sqrt(n) : -1.0f;
  }
  __syncthreads();
  for (int idx = tid; idx < nOut; idx += kCensThreads) {
    const int i = idx / N, c = idx - i * N;
    const float nf = sNorm[i];
    p.stat[(base + tl.f0 + i) * p.statStride + p.outCol + c] = nf >= 0.0f ? __fdiv_rn(sAcc[idx], nf) : p.unit;   // :202-207
  }
}

}  // namespace

size_t cens_smem_bytes(int N, int W)
{
  return (size_t)W * 4 + (size_t)kCensRows * N * 4 + (size_t)kCensRows * 4 + (size_t)(kCensRows + W - 1) * N;
}

cudaError_t cens_configure(int N, int W, size_t optinBytes)
{
  // most shapes fit the default 48 KB; a larger one raises the kernel's limit to the device's opt-in maximum, which no plan of
  // another shape can lower again
  if (cens_smem_bytes(N, W) <= 48 * 1024) return cudaSuccess;
  return cudaFuncSetAttribute(cens_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)optinBytes);
}

cudaError_t launch_cens(const CensParams &p, cudaStream_t st)
{
  if (p.nTiles <= 0) return cudaSuccess;
  cens_kernel<<<p.nTiles, kCensThreads, cens_smem_bytes(p.N, p.W), st>>>(p);
  return cudaGetLastError();
}

}  // namespace osm
