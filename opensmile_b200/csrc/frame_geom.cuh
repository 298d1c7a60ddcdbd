// frame_geom.cuh -- where the frames of a cFramer level lie in their utterance, for the graph compiler (host) and every
// kernel that derives a frame count or reads the samples of a frame.
//
// core/winToVecProcessor.cpp:461-508 resolves the sampling centre c (frameCenterFrames, 0 for `left`) and starts reading at
// pre = -c (core/dataReader.cpp:618-633): frame t covers the source samples [t * step - c, t * step - c + size).  Positions
// before 0 hold sample 0 of the input (core/dataMemoryLevel.cpp:1651-1697 clamps the read index at 0).  With
// noPostEOIprocessing = 1 only complete frames are emitted (:868-877): frame t exists iff t * step - c + size <= L.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define OSM_HD __host__ __device__ __forceinline__
#else
#define OSM_HD inline
#endif

namespace osm {

// frames of an utterance of L samples
OSM_HD long long frame_count(long long L, int size, int step, int center)
{
  const long long Lc = L + center;
  return (size <= 0 || Lc < size) ? 0 : (Lc - size) / step + 1;
}

// first sample of frame t relative to the utterance start (negative for a frame that starts with padding)
OSM_HD long long frame_first_sample(long long t, int step, int center) { return t * step - center; }

// pad positions (copies of sample 0) at the start of frame t
OSM_HD int frame_pad(long long t, int step, int center)
{
  const long long s = frame_first_sample(t, step, center);
  return s < 0 ? (int)-s : 0;
}

}  // namespace osm
