// chunk_schedule_host.cpp -- host build of the batch cut of the per-frame LLD kernels (opensmile_b200/csrc/chunk_schedule.hpp)
// (test infrastructure).
//   g++ -O2 -std=c++17 -shared -fPIC -I/usr/local/cuda/include -o chunk_schedule_host.so chunk_schedule_host.cpp
#include <cstring>

#include "../../opensmile_b200/csrc/chunk_schedule.hpp"

extern "C" {

// T[nUtt] -> the balanced chunk list for `ctas` CTAs, sentinel included, as rows of (utt, a, b, tile0, w0) in
// out[maxChunks][5]; returns the number of entries (or -1 when maxChunks is too small); *q = tiles per run
int csh_balanced(const int64_t *T, int nUtt, int F, int H, int KT, int ctas, int32_t *out, int maxChunks, int64_t *q)
{
  std::vector<osm::ChunkRef> chunks;
  std::vector<int32_t> c0(nUtt + 1), t0(nUtt + 1);
  *q = osm::balanced_chunks(T, nUtt, F, H, KT, ctas, chunks, c0.data(), t0.data());
  if ((int)chunks.size() > maxChunks) return -1;
  static_assert(sizeof(osm::ChunkRef) == 5 * sizeof(int32_t), "ChunkRef layout");
  memcpy(out, chunks.data(), chunks.size() * sizeof(osm::ChunkRef));
  return (int)chunks.size();
}

}
