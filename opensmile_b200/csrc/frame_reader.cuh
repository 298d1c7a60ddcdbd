// frame_reader.cuh -- sample n of frame t as the framer (or the windower) level holds it; shared by the
// time-domain kernels of ops.cu and formant.cu.  Every operation is an explicit round-to-nearest intrinsic, so the
// result does not depend on the FMA contraction setting of the including file.
#pragma once
#include "kernels.cuh"

namespace osm {

// ------------------------------------------------------------------------------------------
// time-domain frames: sample n of frame t, as the framer (or the windower) level holds it
// ------------------------------------------------------------------------------------------
// F32: the kernel instance for pre-converted mono float samples (TimeOpParams::pcmF32)
template <bool F32>
__device__ __forceinline__ float td_pcm(const TimeOpParams &p, const int16_t *s)
{
  if constexpr (F32) return *reinterpret_cast<const float *>(s);   // pre-converted mono float sample
  // smileutil/smileUtil.c:2520-2534 : ((sum_c (float)x_c) / nChan) / 32767
  float tmp = (float)s[0];
  for (int c = 1; c < p.nChan; c++) tmp = __fadd_rn(tmp, (float)s[c]);
  // x / 32767 through a reciprocal multiply + two FMAs: bit-identical to IEEE division for every
  // int16 and every half-integer mean of two (see kernels.cu div32767 / tests/test_host_cpu.py)
  if (p.nChan <= 2) {
    const float x = (p.nChan == 2) ? tmp * 0.5f : tmp;
    const float rc = 3.0518509447574615e-05f;
    const float q0 = __fmul_rn(x, rc);
    return __fmaf_rn(__fmaf_rn(-q0, 32767.0f, x), rc, q0);
  }
  return __fdiv_rn(__fdiv_rn(tmp, (float)p.nChan), 32767.0f);
}

template <bool F32>
struct FrameReader {
  const TimeOpParams &p;
  const int16_t *utt;      // first sample frame of the utterance
  long long s0;            // first sample of this frame within the utterance, frame_first_sample (< 0: a centred frame's padding)
  // positions before the utterance start read its sample 0 (frame_geom.cuh)
  __device__ __forceinline__ float raw(int n) const { return td_pcm<F32>(p, utt + max(s0 + n, 0LL) * p.nChan); }
  // the cVectorPreemphasis level (the framer level when p.preemph = 0)
  __device__ __forceinline__ float pre(int n) const
  {
    float x = raw(n);
    if (p.preemph) {                                  // vectorPreemphasis.cpp:89-108
      if (n == 0) x = __fmul_rn(p.oneMinusK, x);
      else {
        const float kx = __fmul_rn(p.preK, raw(n - 1));
        x = p.preDe ? __fadd_rn(x, kx) : __fsub_rn(x, kx);
      }
    }
    return x;
  }
  __device__ __forceinline__ float at(int n) const
  {
    if (!p.windowed) return raw(n);
    return __fadd_rn(__fmul_rn(pre(n), p.window[n]), p.winOffset);    // windower.cpp:226
  }
};

}  // namespace osm
