// tonefilt.cu -- cTonefilt [-> cChroma] on the wave level (sm_90a), the block form of tonefilt_math.cuh.
//
// Work unit: one segment = a run of output rows (blocks of P samples) of one utterance, one CTA.  Rows are taken 32 at a time
// (a chunk); per chunk:
//   1. G [32 blocks x 2 nNotes] = X [32 x P] W [P x 2 nNotes] on the FP64 tensor cores (mma.m8n8k4.f64): X is staged in shared
//      memory as float in slices of kSlice samples, one warp owns every 4th..8th column tile of 8 for all 32 rows;
//   2. every (block, note) multiplies its sum by the block phase e^{i theta_b} (one sincos each);
//   3. one thread per note carries z through the 32 blocks and writes the rows (or hands them to the chroma fold).
// Long utterances are cut into several segments (plan side): an aggregate pass runs 1-3 from a zero state and keeps each
// segment's end state, tonefilt_carry_kernel chains them per utterance and note (z_in of the next segment = a^n z_in + end
// state), and the output pass reruns 1-3 from that carry.  Segment cuts depend on the utterance's own length only, so an
// utterance gives the same rows alone and in a batch.
// Compiled with -fmad=false: the per-block statements are the host build's (tests/native/tonefilt_host.cpp).
#include "kernels.cuh"
#include "frame_reader.cuh"
#include "tonefilt_math.cuh"

namespace osm {

namespace {

constexpr int kThreads = 256, kWarps = kThreads / 32;
constexpr int kRows = 32;                 // blocks per chunk: 4 row tiles of 8
constexpr int kSlice = 256;               // samples of a block staged per slice
constexpr int kStride = kSlice + 4;       // row stride of the staged slice in floats (== 4 mod 32: conflict-free A fragments)
constexpr int kMaxColTiles = 4;           // column tiles of 8 per warp (2 nNotes <= 8 warps * 4 * 8)

__device__ __forceinline__ void dmma(double &c0, double &c1, double a, double b)
{
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

template <bool F32>
__global__ void __launch_bounds__(kThreads, 2) tonefilt_kernel(const TonefiltParams p, int aggregate)
{
  extern __shared__ __align__(16) unsigned char tfSmem[];
  const ChunkRef seg = p.segs[blockIdx.x];
  const long long uo = p.tp.uttOff[seg.utt];
  const long long L = p.tp.uttOff[seg.utt + 1] - uo;
  const int P = p.P, nN = p.nNotes, nc = p.nc;
  const long long Tu = (L + P - 1) / P;
  if (aggregate && seg.b >= Tu) return;            // the last segment of an utterance hands no state on
  float *xs = reinterpret_cast<float *>(tfSmem);   // [kRows][kStride] staged slice ...
  double *G = reinterpret_cast<double *>(tfSmem);  // ... and, after the product, [kRows][nc] block sums
  float *tone = reinterpret_cast<float *>(tfSmem + p.smemSums);   // [kRows][nNotes] (chroma)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nColT = nc / 8;
  const int16_t *pcm = p.tp.pcm + uo * p.tp.nChan;
  double zr = 0.0, zi = 0.0, ak = 0.0, fk = 0.0;
  if (tid < nN) {
    ak = p.a[tid]; fk = p.freq[tid];
    if (!aggregate && seg.a > 0) { zr = p.cin[(size_t)blockIdx.x * nN + tid].x; zi = p.cin[(size_t)blockIdx.x * nN + tid].y; }
  }
  for (int c0 = seg.a; c0 < seg.b; c0 += kRows) {
    const int nb = min(kRows, seg.b - c0);
    double acc[kMaxColTiles][4][2];
#pragma unroll
    for (int t = 0; t < kMaxColTiles; t++)
#pragma unroll
      for (int m = 0; m < 4; m++) acc[t][m][0] = acc[t][m][1] = 0.0;
    for (int ks = 0; ks < p.kp; ks += kSlice) {
      __syncthreads();
      for (int i = tid; i < kRows * kSlice; i += kThreads) {
        const int r = i / kSlice, jj = i - r * kSlice, j = ks + jj;
        float v = 0.f;
        if (r < nb && j < P) {
          long long m = (long long)(c0 + r) * P + j;
          if (m >= L) m = L - 1;                   // the last block is padded with copies of the last sample
          v = td_pcm<F32>(p.tp, pcm + m * p.tp.nChan);
        }
        xs[r * kStride + jj] = v;
      }
      __syncthreads();
      const int kn = min(kSlice, p.kp - ks);
      for (int kk = 0; kk < kn; kk += 4) {
        double af[4];
#pragma unroll
        for (int m = 0; m < 4; m++) af[m] = (double)xs[(m * 8 + (lane >> 2)) * kStride + kk + (lane & 3)];
        const double *wr = p.W + (size_t)(ks + kk + (lane & 3)) * nc + (lane >> 2);
#pragma unroll
        for (int t = 0; t < kMaxColTiles; t++) {
          const int ct = warp + kWarps * t;
          if (ct < nColT) {
            const double bf = __ldg(wr + ct * 8);
#pragma unroll
            for (int m = 0; m < 4; m++) dmma(acc[t][m][0], acc[t][m][1], af[m], bf);
          }
        }
      }
    }
    __syncthreads();                               // every warp is done with the slice: G takes its place
#pragma unroll
    for (int t = 0; t < kMaxColTiles; t++) {
      const int ct = warp + kWarps * t;
      if (ct < nColT)
#pragma unroll
        for (int m = 0; m < 4; m++) {
          double *g = G + (size_t)(m * 8 + (lane >> 2)) * nc + ct * 8 + (lane & 3) * 2;
          g[0] = acc[t][m][0]; g[1] = acc[t][m][1];
        }
    }
    __syncthreads();
    if (tid < nN) {
      for (int r = 0; r < nb; r++) {
        tf::block_step(zr, zi, ak, G[(size_t)r * nc + 2 * tid], G[(size_t)r * nc + 2 * tid + 1], fk, (long long)(c0 + r), P, p.T);
        if (aggregate) continue;
        const float y = tf::tone_value(zr, zi);
        if (p.chromaK > 0) tone[r * nN + tid] = y;
        else p.tp.stat[(p.tp.statOff[seg.utt] + c0 + r) * (long long)p.tp.statStride + p.tp.outCol + tid] = y;
      }
    }
    if (!aggregate && p.chromaK > 0) {
      __syncthreads();
      if (tid < nb)
        tf::chroma_row(tone + tid * nN, 1, nN, p.chromaK, p.silThresh,
                       p.tp.stat + (p.tp.statOff[seg.utt] + c0 + tid) * (long long)p.tp.statStride + p.tp.outCol, 1);
    }
  }
  if (aggregate && tid < nN) p.agg[(size_t)blockIdx.x * nN + tid] = make_double2(zr, zi);
}

// per (utterance, note): the state entering every segment of the utterance; one thread, in segment order
__global__ void __launch_bounds__(128) tonefilt_carry_kernel(const TonefiltParams p, const int32_t *uttSeg0, int u0, int u1)
{
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)(u1 - u0) * p.nNotes) return;
  const int u = u0 + (int)(i / p.nNotes), k = (int)(i % p.nNotes);
  const int s0 = uttSeg0[u], s1 = uttSeg0[u + 1];
  const int base = uttSeg0[u0];
  double zr = 0.0, zi = 0.0;
  for (int s = s0; s + 1 < s1; s++) {
    const double an = pow(p.a[k], (double)(p.segs[s - base].b - p.segs[s - base].a));
    const double2 e = p.agg[(size_t)(s - base) * p.nNotes + k];
    zr = an * zr + e.x;
    zi = an * zi + e.y;
    p.cin[(size_t)(s + 1 - base) * p.nNotes + k] = make_double2(zr, zi);
  }
}

}  // namespace

size_t tonefilt_smem_bytes(int nNotes, int chroma, size_t *sumsOffset)
{
  const size_t sums = std::max((size_t)kRows * kStride * sizeof(float), (size_t)kRows * tf::padded_cols(nNotes) * sizeof(double));
  if (sumsOffset) *sumsOffset = sums;
  return sums + (chroma ? (size_t)kRows * nNotes * sizeof(float) : 0);
}

cudaError_t launch_tonefilt(const TonefiltParams &p, const int32_t *uttSeg0, int u0, int u1, bool carry, cudaStream_t st)
{
  if (p.nSegs <= 0) return cudaSuccess;
  const size_t smem = tonefilt_smem_bytes(p.nNotes, p.chromaK > 0, nullptr);
  auto kern = p.tp.pcmF32 ? tonefilt_kernel<true> : tonefilt_kernel<false>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  if (carry) {
    kern<<<p.nSegs, kThreads, smem, st>>>(p, 1);
    const long long n = (long long)(u1 - u0) * p.nNotes;
    tonefilt_carry_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(p, uttSeg0, u0, u1);
  }
  kern<<<p.nSegs, kThreads, smem, st>>>(p, 0);
  return cudaGetLastError();
}

}  // namespace osm
