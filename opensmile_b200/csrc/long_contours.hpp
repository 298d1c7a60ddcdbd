// long_contours.hpp -- the work space plan of cFunctionals contours longer than the shared-memory path takes (functionals.cu;
// host-only C++17, also built by g++ for tests/native/long_contours_host.cpp).  Every contour (utterance, input element) of an
// utterance with more than kMaxShort rows gets a slice of one device work space: the segment-length / lag scratch, the filtered
// copy and the Peaks2 / Peaks extrema list (values, then positions), sized for the row count T (the filtered length N is at most T).
// The contours run in chunks of consecutive contours; the slices of a chunk all have the layout of its longest contour, and a
// chunk's slices together stay within a fixed cap, so the work space does not grow with batch size x length.  A contour whose
// slice alone exceeds the cap runs as a chunk of its own.
#pragma once
#include <algorithm>
#include <cstdint>
#include <vector>

namespace osm {

constexpr int kMaxShort = 8192;                      // longest contour the shared-memory path takes (32 KB copy per warp)
constexpr long long kMaxLongRows = 1LL << 30;        // Peaks2 packs (frame << 1) | type into an int
constexpr long long kLongWsCapFloats = 64LL << 20;   // 256 MB of work space per functionals object

struct LongContour {
  int u, e;                     // utterance, input element
  int n;                        // the filtered length, written by the per-warp kernel for the rank selection
};
struct LongChunk {
  int begin, end;               // contours [begin, end)
  int cap;                      // floats of every slice's contour copy: the chunk's longest T rounded up to 32
};

// listMul: 2 when Peaks2 / Peaks need the extrema list, else 0; lensFloats: floats of the segment-length / lag scratch
inline long long long_slice_floats(long long cap, int listMul, int lensFloats) { return lensFloats + cap * (1 + listMul); }

// contours: every long contour in (utterance, element) order.  Returns the work space floats the largest chunk needs.
inline long long plan_long_contours(const int64_t *nRows, int nUtt, int nIn, int listMul, int lensFloats, long long capFloats,
                                    std::vector<LongContour> &contours, std::vector<LongChunk> &chunks)
{
  contours.clear(); chunks.clear();
  long long need = 0;
  LongChunk ch{0, 0, 0};
  auto close = [&] {
    if (ch.end == ch.begin) return;
    need = std::max(need, (ch.end - ch.begin) * long_slice_floats(ch.cap, listMul, lensFloats));
    chunks.push_back(ch);
    ch = LongChunk{ch.end, ch.end, 0};
  };
  for (int u = 0; u < nUtt; u++) {
    if (nRows[u] <= kMaxShort) continue;
    const int cap = (int)((nRows[u] + 31) / 32 * 32);
    for (int e = 0; e < nIn; e++) {
      const int wider = std::max(ch.cap, cap);
      if ((ch.end - ch.begin + 1) * long_slice_floats(wider, listMul, lensFloats) > capFloats) close();
      contours.push_back(LongContour{u, e, 0});
      ch.cap = std::max(ch.cap, cap);
      ch.end++;
    }
  }
  close();
  return need;
}

}  // namespace osm
