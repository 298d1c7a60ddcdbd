// lld_common.cuh -- helpers shared by the fused per-frame kernels (kernels.cu: the general lld_kernel;
// lld_fast.cu: the specialised 512-point MFCC instance): shared-memory layout, PCM conversion, mbarrier / bulk-copy
// wrappers, chunk / tile geometry, the in-place DIF stage, the cPlp back end and the fused delta emission.
#pragma once
#include <cstdio>

#include "fft_radix.cuh"
#include "kernels.cuh"

namespace osm {

// ------------------------------------------------------------------------------------------
// shared memory layout (identical computation on host and device)
// ------------------------------------------------------------------------------------------
struct SmemLayout {
  int zbuf, samp, raw, rawPcm, mbar, winLut, tw, splitTw, melCoef, melRange, dctCos, dctLift, eql, melS, ring;
  int total;
  int sampFloats, rawPcmBytes;
};

__host__ __device__ inline int align_up(int x, int a) { return (x + a - 1) / a * a; }

constexpr int kLeadFrames = 8;   // sample frames fetched ahead of a tile (x[n-1] for pre-emphasis)

__host__ __device__ inline SmemLayout make_layout(const LldParams &p, int M, int F)
{
  SmemLayout L;
  int o = 0;
  L.zbuf = o; o += M * F * 8;
  const int S = p.frameStep + p.sPad;
  L.sampFloats = align_up((F - 1) * S + p.frameSize + ((p.frameSize - 1) / p.frameStep) * p.sPad + 2, 4);
  L.samp = o; o += L.sampFloats * 4;
  L.raw = o; o += F * 4;
  o = align_up(o, 16);
  // raw PCM landing zone of the bulk (TMA) prefetch: <=15 bytes of alignment slack, the lead
  // frames, the tile's sample frames, rounded up to 16
  L.rawPcmBytes = align_up(16 + (kLeadFrames + (F - 1) * p.frameStep + p.frameSize) * p.nChan * 2, 16);
  L.rawPcm = o; o += L.rawPcmBytes;
  L.mbar = o; o += 16;
  L.winLut = o; o += M * 16;
  L.tw = o; o += p.twCount * 8;
  L.splitTw = o; o += (M / 2 + 1) * 8;
  o = align_up(o, 16);
  L.melCoef = o; o += (p.melVCount + 4) * 8;   // visit list: (w, 1-w) per visited bin, ranges padded to x4
  L.melRange = o; o += 2 * (p.nBands + 2) * 4;  // first bin / first visit entry of every range
  o = align_up(o, 16);
  // MFCC: the fast 512-point instance keeps the DCT table transposed, [nBands][16]
  L.dctCos = o; o += max(p.dctRows * p.dctStride, p.opKind == 0 ? p.nBands * 16 : 0) * 4;
  L.dctLift = o; o += p.nStat * 4;
  L.eql = o; o += (p.opKind == 1 ? p.nBands : 0) * 4;
  o = align_up(o, 16);
  // the band values live only between the mel phase and the DCT / PLP back end of the same tile: the
  // sample tile is dead then (it is rewritten by the next tile's staging), so they share its space
  if (L.sampFloats >= p.nBands * F) L.melS = L.samp;
  else { L.melS = o; o += p.nBands * F * 4; }
  L.ring = o; o += p.nStat * 2 * F * 4;     // static features of the last two tiles
  L.total = align_up(o, 16);
  return L;
}

// ------------------------------------------------------------------------------------------
// PCM conversion, smileutil/smileUtil.c:2520-2534 : ((sum_c (float)x_c) / nChan) / 32767
// ------------------------------------------------------------------------------------------
// x / 32767 with one reciprocal multiply and two FMAs (Markstein refinement).  Checked
// exhaustively against IEEE division for every int16 and every half-integer k/2 (stereo mix)
// |k| <= 65536: bit-identical (tests/test_host_cpu.py::test_div32767_trick).
__device__ __forceinline__ float div32767(float x)
{
  const float rc = 3.0518509447574615e-05f;   // fl(1/32767)
  const float q0 = __fmul_rn(x, rc);
  const float r = __fmaf_rn(-q0, 32767.0f, x);
  return __fmaf_rn(r, rc, q0);
}

#define OSM_COLD __noinline__     // rarely executed paths stay out of the hot instruction stream
template <bool F32>
__device__ __forceinline__ float pcm_to_float_generic(const int16_t *s, int nChan)
{
  if constexpr (F32) return *reinterpret_cast<const float *>(s);      // pre-converted mono float sample (LldParams::pcmF32)
  float tmp = (float)s[0];
  for (int c = 1; c < nChan; c++) tmp = __fadd_rn(tmp, (float)s[c]);
  if (nChan == 1) return div32767(tmp);
  if (nChan == 2) return div32767(tmp * 0.5f);          // tmp / 2.0f is exact
  return __fdiv_rn(__fdiv_rn(tmp, (float)nChan), 32767.0f);
}
// out-of-line copy for the rarely taken staging paths (unaligned / partial chunks, >2 channels)
template <bool F32>
static __device__ OSM_COLD float pcm_to_float_slow(const int16_t *s, int nChan) { return pcm_to_float_generic<F32>(s, nChan); }

// ------------------------------------------------------------------------------------------
// mbarrier + bulk async copy (TMA unit, SASS UBLKCP) wrappers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, int count)
{
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar)
{
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra LAB_DONE;\n"
      "bra LAB_WAIT;\n"
      "LAB_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}

// A chunk = output rows [a, b) of one utterance, processed by ONE CTA as consecutive tiles of F
// frames.  With a temporal halo H (fused delta stages) the chunk computes the static features of
// frames [max(a-H,0), min(b+H,T)); the host picks b so that this range is a whole number of
// tiles, i.e. the halo costs no extra tile.
struct ChunkCtx {
  int utt, a, b;     // output rows [a,b) of utterance utt
  int T;             // static frames of the utterance
  int s0;            // first static frame computed by this chunk
  int sEnd;          // one past the last static frame computed
  int nT;            // tiles in this chunk
  int tile0;         // global index of the chunk's first tile
  long long uo;      // sample-frame offset of the utterance
  long long row0;    // output row of frame 0 of the utterance
};

// CENTRED: frames start at t * frameStep - LldParams::frameCenter (lld_kernel).  Without it the left-framed geometry alone
// (frame_geom.cuh with centre 0) is compiled, in the form lld512_kernel's instruction stream was tuned on; lld512_kernel never
// serves a centred stream (lld_fast_applies).
template <int F, bool CENTRED = false>
__device__ __forceinline__ ChunkCtx load_chunk(const LldParams &p, int chunk)
{
  ChunkCtx c;
  const ChunkRef cr = p.chunks[chunk];
  c.utt = cr.utt; c.a = cr.a; c.b = cr.b; c.tile0 = cr.tile0;
  c.uo = p.uttOff[cr.utt];
  const long long Ls = p.uttOff[cr.utt + 1] - c.uo;
  if constexpr (CENTRED) c.T = (int)frame_count(Ls, p.frameSize, p.frameStep, p.frameCenter);
  else c.T = (int)((Ls - p.frameSize) / p.frameStep + 1);
  c.s0 = max(cr.a - p.halo, 0);
  c.sEnd = min(cr.b + p.halo, c.T);
  c.nT = (c.sEnd - c.s0 + F - 1) / F;
  c.row0 = p.rowOff[cr.utt];
  return c;
}

// first chunk of CTA g's run (LldParams::ctaTiles): the first chunk whose schedule position is at least g * ctaTiles
__device__ __forceinline__ int chunk_run_begin(const LldParams &p, int g)
{
  const long long w = (long long)p.chunks[0].w0 + (long long)g * p.ctaTiles;
  int lo = 0, hi = p.nChunks;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (p.chunks[mid].w0 < w) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// geometry of one tile (all warp-uniform)
struct TileGeom {
  int fs;            // first static frame of the tile
  int nf;            // frames in this tile
  int count;         // sample frames the tile covers
  int lead;          // sample frames fetched before the tile start (0 at the utterance start)
  int pad;           // centred frames: sample frames of the tile before the utterance start (copies of its sample 0, not fetched)
  int mis;           // bytes between the 16-byte aligned fetch address and the first wanted byte
  uint32_t bytes;    // bulk copy size
  const char *src;   // 16-byte aligned fetch address
};

// CENTRED (see load_chunk): the fetch stays inside the tile's utterance -- a tile whose first frames start before it fetches
// from its sample 0 on (pad > 0), and the lead frames stop at its start.
template <int F, bool CENTRED = false>
__device__ __forceinline__ TileGeom tile_geom(const LldParams &p, const ChunkCtx &c, int j)
{
  TileGeom g;
  g.fs = c.s0 + j * F;
  g.nf = min(F, c.sEnd - g.fs);
  g.count = (g.nf - 1) * p.frameStep + p.frameSize;
  const char *a;
  if constexpr (CENTRED) {
    const long long s0 = frame_first_sample(g.fs, p.frameStep, p.frameCenter);
    g.pad = s0 < 0 ? (int)-s0 : 0;
    g.lead = (int)min(max(s0, 0LL), (long long)kLeadFrames);
    a = reinterpret_cast<const char *>(p.pcm + (c.uo + s0 + g.pad - g.lead) * p.nChan);
  } else {
    const long long s0 = (long long)g.fs * p.frameStep;
    g.pad = 0;
    g.lead = (s0 > 0) ? kLeadFrames : 0;
    a = reinterpret_cast<const char *>(p.pcm + (c.uo + s0 - g.lead) * p.nChan);
  }
  g.mis = (int)(reinterpret_cast<uintptr_t>(a) & 15);
  g.src = a - g.mis;
  g.bytes = (uint32_t)align_up(g.mis + (g.lead + g.count - g.pad) * p.nChan * 2, 16);
  return g;
}

// Staging of a tile whose first frames start before the utterance (centred framing, first tile(s) of an utterance only):
// tile sample i is utterance sample max(i - pad, 0); rp = utterance sample 0 in the landing zone.  Same conversion,
// pre-emphasis and layout as the staging loop of lld_kernel; ks = the signed pre-emphasis coefficient, 0 without pre-emphasis.
// (Scalars, not the LldParams block: a reference to it would make the caller copy the block to its stack.)
template <int F, int NT, bool F32>
__device__ OSM_COLD void stage_padded_tile(const int16_t *rp, int pad, int count, int hop, int sPad, int nChan, float ks,
                                           float *samp, float *raw, int tid)
{
  for (int i = tid; i < count; i += NT) {
    const float x = pcm_to_float_slow<F32>(rp + max(i - pad, 0) * nChan, nChan);
    float y = x;
    if (ks != 0.f && i > 0) y = __fadd_rn(x, __fmul_rn(ks, pcm_to_float_slow<F32>(rp + max(i - 1 - pad, 0) * nChan, nChan)));
    const int q = i / hop, r = i - q * hop;
    if (r == 0 && q < F) raw[q] = x;
    samp[i + q * sPad] = y;
  }
}

// x / d.  rcp != 0 marks a divisor (2, 10, 28, 60 = the delta norms of windows 1..4) for which the
// reciprocal + two-FMA sequence was verified bit-identical to IEEE division for EVERY float x
// with 1e-30 < |x| < 1e30 (exhaustive 2^32 sweep on the CPU, DESIGN.md section 5); outside that
// range, and for any other divisor, the IEEE division is used.
__device__ __forceinline__ float div_exact(float x, float d, float rcp)
{
  const float ax = fabsf(x);
  if (rcp != 0.f && ax > 1e-30f && ax < 1e30f) {
    const float q0 = __fmul_rn(x, rcp);
    const float r = __fmaf_rn(-q0, d, x);
    return __fmaf_rn(r, rcp, q0);
  }
  return __fdiv_rn(x, d);
}

// reads of a window processor's input level under the tick-order model (see post_kernel)
__device__ __forceinline__ int win_navail(int t, int n0, int c0, int Tprev)
{
  return (t < c0) ? Tprev : min(n0 + (t - c0) + 1, Tprev);
}

// ------------------------------------------------------------------------------------------
// one in-place DIF stage.  Virtual warp vw (of NVW) handles butterflies t = vw, vw+NVW, ...
// ------------------------------------------------------------------------------------------
template <int M, int F, int NVW, int R, int MS, bool FIRST, bool LAST, bool VEC2>
__device__ __forceinline__ void fft_stage(float2 *__restrict__ Z, const float *__restrict__ sampF,
                                          const float *__restrict__ raw,
                                          const float4 *__restrict__ winLut,
                                          const float2 *__restrict__ tw,
                                          const LldParams &p, int vw, int f)
{
  constexpr int stride = MS / R;
  for (int t = vw; t < M / R; t += NVW) {
    const int blk = t / stride, j = t % stride;
    const int base = blk * MS + j;
    float2 v[R];
    if (FIRST) {
      // Elements beyond the frame (zero padding) have table weight 0 and offset 0: they load a
      // finite sample and multiply it by 0 -> no per-element branch (the sample tile only ever
      // holds finite floats, it is zero-filled at kernel start).
#pragma unroll
      for (int r = 0; r < R; r++) {
        const float4 wl = winLut[base + stride * r];   // (w[2e], w[2e+1], offset, #valid)
        const int off = __float_as_int(wl.z);
        float2 x;
        if (VEC2) {
          x = *reinterpret_cast<const float2 *>(sampF + off);
        } else {
          x.x = sampF[off];
          x.y = sampF[off + 1];
        }
        // windower.cpp:226 : src * (float)w (+ (float)offset below), separate roundings
        v[r] = make_float2(__fmul_rn(x.x, wl.x), __fmul_rn(x.y, wl.y));
      }
      if (base == 0 && p.preemph)      // first sample of the frame, vectorPreemphasis.cpp:94
        v[0].x = __fmul_rn(__fmul_rn(p.oneMinusK, raw[f]), winLut[0].x);
      if (p.hasWinOffset) {
#pragma unroll
        for (int r = 0; r < R; r++) {
          // #valid: 0 = padding, 1 = only the first sample of the pair exists, 2 = both
          const float nv = winLut[base + stride * r].w;
          if (nv >= 1.f) v[r].x = __fadd_rn(v[r].x, p.winOffset);
          if (nv >= 2.f) v[r].y = __fadd_rn(v[r].y, p.winOffset);
        }
      }
    } else {
#pragma unroll
      for (int r = 0; r < R; r++) v[r] = Z[(base + stride * r) * F + f];
    }
    Dft<R>::run(v);
    if (!LAST) {
      const float2 *twj = tw + j * R;
#pragma unroll
      for (int q = 1; q < R; q++) v[Dft<R>::out(q)] = cmul(v[Dft<R>::out(q)], twj[q]);
    }
#pragma unroll
    for (int q = 0; q < R; q++) Z[(base + stride * q) * F + f] = v[Dft<R>::out(q)];
  }
}

// ------------------------------------------------------------------------------------------
// cPlp back end for one tile, lane = frame (lldcore/plp.cpp:520-590):
//   IDFT of the compressed auditory spectrum -> autocorrelation (double accumulation, :522-532)
//   Durbin recursion (smileutil/smileUtil.c:1572-1627), lp -> cepstrum (HTK eq. 5.11, :1532-1556),
//   c0 = -log(1/gain), lifter.  melS holds the nBands processed band values per frame; acfS is
//   scratch [nAuto][F] (aliases the dead FFT tile); dst = ring slot base, row stride 2F.
// ------------------------------------------------------------------------------------------
constexpr int kMaxLp = 8;

template <int F, int NVW>
__device__ __forceinline__ void plp_backend(const LldParams &p, const float *melS, const float *sCos,
                                            const float *sLift, float *acfS, float *dst, int vw, int f)
{
  const int nB = p.nBands, nFreq = p.plpNFreq, nAuto = p.plpNAuto;
  if (!p.plpIDFT) {   // audSpec output: the processed bands themselves
    for (int i = vw; i < nB; i += NVW) dst[i * (2 * F) + f] = melS[i * F + f];
    return;
  }
  for (int i = vw; i < nAuto; i += NVW) {
    const float *ct = sCos + i * p.dctStride;
    double tmp = 0.0;
    if (p.plpHtk) tmp = (double)ct[0] * (double)melS[f];
    for (int m = 1; m < nFreq - 1; m++) tmp = __dadd_rn(tmp, (double)ct[m] * (double)melS[(m - 1) * F + f]);
    tmp = __dadd_rn(tmp, (double)ct[nFreq - 1] * (double)melS[(nFreq - 3) * F + f]);
    const float a = (float)(tmp / (2.0 * (double)(nFreq - 1)));
    if (!p.plpLP) dst[i * (2 * F) + f] = a;
    else acfS[i * F + f] = a;
  }
  if (!p.plpLP) return;
  __syncthreads();
  if (vw == 0) {
    const int P = p.plpOrder;
    float r[kMaxLp + 1], a[kMaxLp], cc[kMaxLp + 1];
#pragma unroll
    for (int i = 0; i <= kMaxLp; i++) r[i] = (i <= P) ? acfS[i * F + f] : 0.f;
#pragma unroll
    for (int i = 0; i < kMaxLp; i++) a[i] = 0.f;
    float gain = 0.f;
    if (r[0] != 0.f) {
      float e = r[0];
#pragma unroll
      for (int m = 1; m <= kMaxLp; m++) {
        if (m <= P && e != 0.f) {
          float sum = r[m];                                            // 1.0f * r[m]
#pragma unroll
          for (int i = 1; i < m; i++) sum = __fadd_rn(sum, __fmul_rn(a[i - 1], r[m - i]));
          const float km = __fmul_rn(__fdiv_rn(-1.0f, e), sum);
          a[m - 1] = km;
#pragma unroll
          for (int i = 1; i <= m / 2; i++) {
            const float x = a[i - 1];
            a[i - 1] = __fadd_rn(a[i - 1], __fmul_rn(km, a[m - i - 1]));
            if ((i < (m / 2)) || ((m & 1) == 1)) a[m - i - 1] = __fadd_rn(a[m - i - 1], __fmul_rn(km, x));
          }
          e = __fmul_rn(e, __fsub_rn(1.0f, __fmul_rn(km, km)));
        }
      }
      gain = e;
    }
    if (!p.plpCeps) {
#pragma unroll
      for (int i = 0; i < kMaxLp; i++) if (i < P) dst[i * (2 * F) + f] = a[i];
      return;
    }
    if (gain <= 0.f) gain = 1.0f;                                      // plp.cpp:541-544
    // lp -> cepstrum: ceps[n-1] = -(lp[n-1] + (float)(sum_{i<n} (n-i) lp[i-1] ceps[n-i-1] / n)),
    // products in float, sum in double (smileUtil.c:1545-1551)
    int first = p.plpFirstCC < 1 ? 1 : p.plpFirstCC;
    const int last = p.plpLastCC > P ? P : p.plpLastCC;
    // NOTE (reference indexing): ceps[] is written at n - firstCC but read at n - i - 1; the two
    // agree only for firstCC <= 1, which is what every shipped config uses (checked on the host)
#pragma unroll
    for (int n = 1; n <= kMaxLp; n++) {
      if (n >= first && n <= last) {
        double sum = 0.0;
#pragma unroll
        for (int i = 1; i < n; i++)
          sum = __dadd_rn(sum, (double)__fmul_rn(__fmul_rn((float)(n - i), a[i - 1]), cc[n - i - 1]));
        cc[n - first] = -__fadd_rn(a[n - first], (float)(sum / (double)n));
      }
    }
    const float zeroth = (float)(-log(1.0 / (double)gain));
    const int nC = p.nStat;
    // output order (plp.cpp:549-553): firstCC == 0 puts c0 first, or last when htkcompatible
#pragma unroll
    for (int i = 0; i <= kMaxLp; i++) {
      if (i < nC) {
        float v;
        if (p.plpFirstCC == 0) {
          if (p.plpHtk) v = (i == nC - 1) ? zeroth : cc[i];
          else v = (i == 0) ? zeroth : cc[i - 1];
        } else {
          v = cc[i];
        }
        if (p.plpLifter) v = __fmul_rn(v, sLift[i]);
        dst[i * (2 * F) + f] = v;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// cTonespec (lld/tonespec.cpp:403-434), per note after the band walk: the weighted bin sum over the note's bin count (IEEE
// division as the reference's dst[i] /= n), 0 for a note without bins, then sqrt under usePower (0 for a negative sum).
// The walk's products are fused into its sums (the mel phase's rounding, where the reference rounds product and sum
// separately): on the same magnitudes the rows stay within 2.4e-7 of the column scale of the reference's statement order.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float tone_mean(float sum, float nbins, int usePower)
{
  float v = nbins > 0.f ? __fdiv_rn(sum, nbins) : 0.f;
  if (usePower) v = v >= 0.f ? __fsqrt_rn(v) : 0.f;
  return v;
}

// The tone op's back end for one tile, lane = frame.  chromaOct == 0: the notes are the output.  Else cChroma
// (lld/chroma.cpp:86-117): chroma i = float sum over octaves j in ascending order of note j * octaveSize + i; one value below
// silThresh or a zero double total of the sums gives a zero vector, otherwise every value is divided by (float) total.
// dst = ring slot base, row stride 2F.
template <int F, int NVW>
__device__ __forceinline__ void tone_backend(const LldParams &p, const float *melS, float *dst, int vw, int f)
{
  const int K = p.chromaOct;
  if (K == 0) {
    for (int i = vw; i < p.nBands; i += NVW) dst[i * (2 * F) + f] = melS[i * F + f];
    return;
  }
  if (vw != 0) return;
  const int nOct = p.nBands / K;
  double sum = 0.0;
  bool sil = false;
  for (int i = 0; i < K; i++) {
    float s = 0.f;
    for (int j = 0; j < nOct; j++) s = __fadd_rn(s, melS[(j * K + i) * F + f]);
    if (s < p.chromaSilThresh) sil = true;
    sum = __dadd_rn(sum, (double)s);
    dst[i * (2 * F) + f] = s;
  }
  const bool norm = sum != 0.0 && !sil;
  const float fsum = (float)sum;
  for (int i = 0; i < K; i++) dst[i * (2 * F) + f] = norm ? __fdiv_rn(dst[i * (2 * F) + f], fsum) : 0.f;
}

// ------------------------------------------------------------------------------------------
// Fused delta / delta-delta emission of one interior tile (deltawin = 2 for both stages, no
// clamping, all rows before EOI): F output rows = statics | delta | delta-delta -> outS laid out
// like the global rows.  num = 1*(x[t+1]-x[t-1]) + 2*(x[t+2]-x[t-2]) in the reference's order:
// (0 + 1*d1) + 2*d2 == d1 + 2*d2 exactly (deltaRegression.cpp:139-146).
// ------------------------------------------------------------------------------------------
template <int F, int NT>
__device__ __forceinline__ void emit_interior(const float *__restrict__ ring, float *__restrict__ Dbuf,
                                              float *__restrict__ outS, int K, int dRows, int slot0, int rslot0,
                                              float norm1, float rcp1, float norm2, float rcp2, int tid)
{
  const int K3 = 3 * K;
  constexpr int DR = F + 4;                                    // delta rows of this tile
  for (int item = tid; item < K * DR; item += NT) {
    const int c = item / DR, tt = item - c * DR;
    const float *rc = ring + c * (2 * F);
    const int sl = slot0 + tt;
    const float dA = __fsub_rn(rc[(sl + 1) & (2 * F - 1)], rc[(sl - 1) & (2 * F - 1)]);
    const float dB = __fsub_rn(rc[(sl + 2) & (2 * F - 1)], rc[(sl - 2) & (2 * F - 1)]);
    const float dv = div_exact(__fadd_rn(dA, __fmul_rn(2.0f, dB)), norm1, rcp1);
    Dbuf[c * dRows + tt] = dv;
    const int rr = tt - 2;
    if (rr >= 0 && rr < F) outS[rr * K3 + K + c] = dv;
  }
  for (int item = tid; item < K * F; item += NT) {             // statics -> outS
    const int c = item / F, rr = item - c * F;
    outS[rr * K3 + c] = ring[c * (2 * F) + ((rslot0 + rr) & (2 * F - 1))];
  }
  __syncthreads();
  for (int item = tid; item < K * F; item += NT) {             // delta-delta rows
    const int c = item / F, rr = item - c * F;
    const float *dt = Dbuf + c * dRows + rr + 2;               // row t = r0 + rr sits at tt = rr + 2
    const float dA = __fsub_rn(dt[1], dt[-1]);
    const float dB = __fsub_rn(dt[2], dt[-2]);
    outS[rr * K3 + 2 * K + c] = div_exact(__fadd_rn(dA, __fmul_rn(2.0f, dB)), norm2, rcp2);
  }
  __syncthreads();
}

// Fused delta / delta-delta emission, general path (utterance edges, deltawin != 2): lane = row, warps
// take the coefficients; clamping and the tick-order model of post_kernel decide what a read past
// either end of a level returns.  Out of line: it runs on the first / last tiles of an utterance only.
// KC / WC != 0: the coefficients K and both windows W1 = W2 known at compile time (lld_fast.cu), the
// arguments K, W1, W2 are then not read.
template <int F, int NW, int KC = 0, int WC = 0>
__device__ OSM_COLD void emit_edge(const float *__restrict__ ring, float *__restrict__ Dbuf, float *__restrict__ outS,
                               int Kr, int W1r, int W2r, int T, int T1, int c01, int c02, int s0, int r0, int r1,
                               int d0, int d1, int dRows, float norm1, float rcp1, float norm2, float rcp2,
                               int warp, int lane)
{
  const int K = KC ? KC : Kr, W1 = WC ? WC : W1r, W2 = WC ? WC : W2r;
  const int K3 = 3 * K, nr = r1 - r0;
  for (int c = warp; c < K; c += NW) {
    const float *rc = ring + c * (2 * F);
    for (int tt = lane; tt < d1 - d0; tt += 32) {
      const int t = d0 + tt;
      // level-0 reads: navail = T (the static level is complete when EOI is raised)
      float num = 0.f;
      for (int i = 1; i <= W1; i++) {
        const int hi = t + i, lo = t - i;
        float later, prior;
        if (t - W1 < 0) {
          later = (hi >= T) ? 0.f : rc[(hi - s0) & (2 * F - 1)];
          prior = rc[(max(lo, 0) - s0) & (2 * F - 1)];
        } else {
          later = rc[(min(hi, T - 1) - s0) & (2 * F - 1)];
          prior = rc[(min(lo, T - 1) - s0) & (2 * F - 1)];
        }
        num = __fadd_rn(num, __fmul_rn((float)i, __fsub_rn(later, prior)));   // deltaRegression.cpp:139-146
      }
      const float dv = div_exact(num, norm1, rcp1);
      Dbuf[c * dRows + tt] = dv;
      if (t >= r0 && t < r1) outS[(t - r0) * K3 + K + c] = dv;
    }
    for (int rr = lane; rr < nr; rr += 32) outS[rr * K3 + c] = rc[(r0 + rr - s0) & (2 * F - 1)];
  }
  __syncthreads();
  // ---- delta-delta rows [r0, r1) -> outS ----
  for (int c = warp; c < K; c += NW) {
    const float *dc = Dbuf + c * dRows - d0;
    for (int rr = lane; rr < nr; rr += 32) {
      const int t = r0 + rr;
      const int navail2 = win_navail(t, c01, c02, T1);
      float num = 0.f;
      for (int i = 1; i <= W2; i++) {
        const int hi = t + i, lo = t - i;
        float later, prior;
        if (t - W2 < 0) {
          later = (hi >= navail2) ? 0.f : dc[hi];
          prior = dc[max(lo, 0)];
        } else {
          later = dc[min(hi, navail2 - 1)];
          prior = dc[min(lo, navail2 - 1)];
        }
        num = __fadd_rn(num, __fmul_rn((float)i, __fsub_rn(later, prior)));
      }
      outS[rr * K3 + 2 * K + c] = div_exact(num, norm2, rcp2);
    }
  }
  __syncthreads();
}

}  // namespace osm
