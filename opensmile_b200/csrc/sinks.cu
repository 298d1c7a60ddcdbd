// sinks.cu -- the value formatting of the reference's file sinks on the device (SURVEY.md 8f-4): rows that a plan run left in HBM
// are turned into the bytes of the files there, the host only adds the per-row prefix (name / index / time stamp) and writes.
//   cHtkSink  (iocore/htkSink.cpp:183-206): float32 big endian -> htk_pack_kernel swaps the bytes of every value
//   cCsvSink  (iocore/csvSink.cpp:195-233): "%.0f" for integer-valued values, "%e" otherwise, a delimiter between the values and a
//             newline after the last -> csv_format_kernel: one warp per row, lane = value (text_format.cuh, identical to printf on
//             every finite float it accepts), ordered by a warp prefix sum of the lengths into the row's slot of the text buffer.
//             Rows with a value the device leaves to the host (non-finite, |x| >= 1e15, an undecidable rounding: ~1e-7 of the
//             values) are flagged and formatted by the host writer.
//   cArffSink (iocore/arffSink.cpp:300-312): every value "%e", ',' between them -> the same kernel with alwaysE (integers >= 1e7 go to
//             the host writer as well)
// gather_rows_kernel picks an LLD sink's columns and rows out of the union level a summary configuration's plan leaves in HBM, into
// the packed [rows][columns] layout the two kernels above read (a session whose sinks read a summary and an LLD level).
#include <cuda_runtime.h>

#include "../../include/osm_b200_host.h"
#include "text_format.cuh"

namespace osm {
namespace {

constexpr int kSinkWarps = 8;

__global__ void __launch_bounds__(kSinkWarps * 32) csv_format_kernel(const float *__restrict__ rows, long long nRows, int K, char delim,
                                                                      char *__restrict__ text, long long slot, int *__restrict__ rowLen,
                                                                      unsigned char *__restrict__ rowHost, int alwaysE)
{
  const int lane = threadIdx.x & 31;
  const long long r = (long long)blockIdx.x * kSinkWarps + (threadIdx.x >> 5);
  if (r >= nRows) return;
  const float *row = rows + r * K;
  char *dst = text + r * slot;
  int off = 0;
  bool host = false;
  for (int k0 = 0; k0 < K; k0 += 32) {
    const int k = k0 + lane;
    char buf[tf::kMaxValueChars + 1];
    int n = 0;
    if (k < K) {
      n = tf::fmt_value(row[k], buf, alwaysE != 0);
      if (n < 0) { host = true; n = 0; }
      buf[n++] = (k == K - 1) ? '\n' : delim;
    }
    int incl = n;                                     // inclusive prefix sum of the lengths over the lanes
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    char *d = dst + off + incl - n;
    for (int i = 0; i < n; i++) d[i] = buf[i];
    off += __shfl_sync(0xffffffffu, incl, 31);
  }
  host = __any_sync(0xffffffffu, host);
  if (lane == 0) { rowLen[r] = off; rowHost[r] = host ? 1 : 0; }
}

__global__ void htk_pack_kernel(const uint32_t *__restrict__ in, uint32_t *__restrict__ out, long long n)
{
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = __byte_perm(in[i], 0, 0x0123);
}

// one warp per output row: row r of utterance u (dstOff[u] <= r < dstOff[u + 1]) is row srcOff[u] + r - dstOff[u] of `in`, columns
// cols[0 .. nCols); a copy, no arithmetic
__global__ void __launch_bounds__(kSinkWarps * 32) gather_rows_kernel(const float *__restrict__ in, int inStride, const long long *__restrict__ cols,
                                                                       int nCols, const long long *__restrict__ srcOff,
                                                                       const long long *__restrict__ dstOff, int nUtt, float *__restrict__ out)
{
  const long long r = (long long)blockIdx.x * kSinkWarps + (threadIdx.x >> 5);
  if (r >= dstOff[nUtt]) return;
  int lo = 0, hi = nUtt - 1;                          // the last u with dstOff[u] <= r
  while (lo < hi) { const int m = (lo + hi + 1) >> 1; if (dstOff[m] <= r) lo = m; else hi = m - 1; }
  const float *src = in + (srcOff[lo] + r - dstOff[lo]) * inStride;
  float *dst = out + r * nCols;
  for (int k = threadIdx.x & 31; k < nCols; k += 32) dst[k] = src[cols[k]];
}

}  // namespace
}  // namespace osm

using namespace osm;

extern "C" {

int64_t osm_b200_device_csv_slot_bytes(int32_t K) { return (int64_t)K * (tf::kMaxValueChars + 1); }

int32_t osm_b200_device_format_csv(const float *d_rows, int64_t n_rows, int32_t K, char delim, char *d_text, int64_t slot_bytes,
                                   int32_t *d_row_len, uint8_t *d_row_host, void *stream)
{
  return osm_b200_device_format_rows(d_rows, n_rows, K, delim, 0, d_text, slot_bytes, d_row_len, d_row_host, stream);
}

int32_t osm_b200_device_format_rows(const float *d_rows, int64_t n_rows, int32_t K, char delim, int32_t always_e, char *d_text, int64_t slot_bytes,
                                    int32_t *d_row_len, uint8_t *d_row_host, void *stream)
{
  if (n_rows <= 0) return 0;
  if (!d_rows || !d_text || !d_row_len || !d_row_host || K <= 0 || slot_bytes < osm_b200_device_csv_slot_bytes(K)) return 1;
  const long long blocks = (n_rows + kSinkWarps - 1) / kSinkWarps;
  csv_format_kernel<<<(unsigned)blocks, kSinkWarps * 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(d_rows, n_rows, K, delim, d_text, slot_bytes,
                                                                                                       d_row_len, d_row_host, always_e);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

int32_t osm_b200_device_pack_htk(const float *d_rows, int64_t n_values, uint32_t *d_out, void *stream)
{
  if (n_values <= 0) return 0;
  if (!d_rows || !d_out) return 1;
  const long long blocks = (n_values + 255) / 256;
  htk_pack_kernel<<<(unsigned)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(reinterpret_cast<const uint32_t *>(d_rows), d_out, n_values);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

int32_t osm_b200_device_gather_rows(const float *d_in, int32_t in_stride, const int64_t *d_meta, int32_t n_cols, int32_t n_utt,
                                    int64_t n_out_rows, float *d_out, void *stream)
{
  if (n_out_rows <= 0) return 0;
  if (!d_in || !d_meta || !d_out || n_cols <= 0 || n_utt <= 0) return 1;
  const long long *meta = reinterpret_cast<const long long *>(d_meta);
  const long long blocks = (n_out_rows + kSinkWarps - 1) / kSinkWarps;
  gather_rows_kernel<<<(unsigned)blocks, kSinkWarps * 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      d_in, in_stride, meta, n_cols, meta + n_cols, meta + n_cols + n_utt, n_utt, d_out);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

}  // extern "C"
