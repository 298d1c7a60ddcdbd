// chunk_schedule.hpp -- host-side cut of a batch into the chunks of the per-frame LLD kernels and their CTA runs
// (LldParams::ctaTiles).  Host only; tests/native/chunk_schedule_host.cpp builds it for the CPU tests.
#pragma once
#include <algorithm>
#include <cstdint>
#include <vector>

#include "kernels.cuh"

namespace osm {

// Chunks: output rows [a,b) of one utterance whose static range [a-H, b+H) /\ [0,T) is a whole number of F-frame tiles
// (except at the utterance end), at most KT tiles each.  Q > 0 also ends a chunk where the schedule reaches a multiple of
// Q tiles, so that every CTA's run holds Q tiles; each such cut inside an utterance recomputes the halo, at most one tile.
// T[u] = static frames of utterance u.  Fills chunks (w0 = schedule position), uttChunk0 / uttTile0 [nUtt+1] and returns
// the schedule's length in tiles.
inline int64_t cut_chunks(const int64_t *T, int nUtt, int F, int H, int KT, int64_t Q, std::vector<ChunkRef> &chunks,
                          int32_t *uttChunk0, int32_t *uttTile0)
{
  chunks.clear();
  int64_t w = 0, tileCount = 0;
  for (int u = 0; u < nUtt; u++) {
    const int64_t Tu = T[u];
    uttChunk0[u] = (int32_t)chunks.size();
    uttTile0[u] = (int32_t)tileCount;
    for (int64_t a = 0; a < Tu;) {
      const int64_t s0 = std::max<int64_t>(a - H, 0);
      const auto end = [&](int64_t n) { return s0 + F * n >= Tu ? Tu : s0 + F * n - H; };   // b for a chunk of n tiles
      int64_t b = end(Q > 0 ? std::min<int64_t>(KT, Q - w % Q) : KT);
      if (b <= a) {
        // too few tiles for a row beside the halo: the rest of the current run stays idle; a whole run that short
        // (tiny batches) takes the chunk anyway
        if (Q > 0 && w % Q != 0) { w += Q - w % Q; continue; }
        b = end(KT);
      }
      chunks.push_back(ChunkRef{u, (int32_t)a, (int32_t)b, (int32_t)(tileCount + s0 / F), (int32_t)w});
      w += (std::min<int64_t>(b + H, Tu) - s0 + F - 1) / F;
      a = b;
    }
    tileCount += (Tu + F - 1) / F;
  }
  uttChunk0[nUtt] = (int32_t)chunks.size();
  uttTile0[nUtt] = (int32_t)tileCount;
  return w;
}

// The balanced cut for `ctas` resident CTAs: the smallest Q >= W / ctas whose cut fits ctas runs.  The chunk list ends
// with one entry whose w0 is the schedule's length (the launch reads a range's length from it).  Returns Q.
inline int64_t balanced_chunks(const int64_t *T, int nUtt, int F, int H, int KT, int ctas, std::vector<ChunkRef> &chunks,
                               int32_t *uttChunk0, int32_t *uttTile0)
{
  int64_t W = cut_chunks(T, nUtt, F, H, KT, 0, chunks, uttChunk0, uttTile0);
  int64_t Q = std::max<int64_t>((W + ctas - 1) / ctas, 1);
  while ((W = cut_chunks(T, nUtt, F, H, KT, Q, chunks, uttChunk0, uttTile0)) > Q * ctas) Q++;
  chunks.push_back(ChunkRef{nUtt, 0, 0, 0, (int32_t)W});
  return Q;
}

}  // namespace osm
