// lld_fast.cu -- the 512-point mono MFCC instance of the fused per-frame kernel (sm_90a).
//
// Same contract, shared-memory layout, tables, chunk / tile geometry and results as lld_kernel<256,32,256,2,VEC2,MFCC>
// (kernels.cu); launch_lld() selects it when the pass is: N = 512, one channel, cMfcc on the power spectrum, no
// magnitude dump, no window offset, frameStep and frameSize multiples of 8.  What differs is the instruction stream:
//
//   stage    one code path (mono, 8 samples per thread, 16-byte loads from the bulk-copy landing zone)
//   pass 1   radix-16 butterflies straight from the sample tile; rows of the butterfly that only ever see zero padding
//            (frameSize <= 416: rows 13..15) are not loaded and their additions are pruned
//   pass 2   the second radix-16 pass, the real-FFT split and re^2 + im^2 are ONE register-resident step: butterfly t
//            produces the bins k = t (mod 16) and the split pairs bin k with bin M - k = -t (mod 16), so a warp that owns
//            butterflies t and 16 - t holds both halves of 16 pairs in registers.  The transformed tile is never written
//            back and never re-read (one Z round trip and one barrier less than lld_kernel).  The two self-paired
//            butterflies (t = 0: k and 256 - k both = 0 mod 16; t = 8) go to warp 0, which reorders its registers into the
//            same (a_q, b_{15-q}) pairing so that every warp executes the same code.
//   mel      visit list read as float4 (two bins per load); the band level lives behind the power spectrum, not in the sample tile
//   DCT      table transposed, [band][16]: a warp evaluates two coefficients per band value read, in the reference's order
//   emit     with 13 static columns (lld512_kernel<NZR, 13>) every thread's Δ / ΔΔ items are fixed at compile time
//   store    the tile's rows leave 16 bytes at a time (staged at their global offset modulo 16 bytes)
//
// Reference rows as in kernels.cu (SURVEY.md 8a-1 ... a-8, a-13, a-15).
#include "lld_common.cuh"

namespace osm {

// Phase clocks (build with -DOSM_LLD_PHASE_CLOCKS, `make phase-clocks`; off in the default library): thread 0 of every CTA
// reads clock64() at each phase boundary of every tile and adds the cycles since the previous boundary into a per-CTA slot;
// the CTA's sums go to gLld512Phase at its exit.  Most boundaries follow a barrier, so a phase's count is the CTA's time
// from one barrier to the next.  Emit and store end without one: they count thread 0's own share, and the wait for the
// other threads lands in the next tile's stage.  scripts/lld512_phase_clocks.py prints the sums per frame.
enum { kPhStage, kPhPass1, kPhPass2, kPhMel, kPhDct, kPhEmit, kPhStore, kPhKernel, kPhKernelMax, kPhTiles, kPhSlots };
#ifdef OSM_LLD_PHASE_CLOCKS
__device__ unsigned long long gLld512Phase[kPhSlots];
#define OSM_PHASE(k)                                                    \
  do {                                                                  \
    if (tid == 0) {                                                     \
      const long long c_ = clock64();                                   \
      sPh[k] += (unsigned long long)(c_ - phT);                         \
      phT = c_;                                                         \
    }                                                                   \
  } while (0)
#else
#define OSM_PHASE(k) do {} while (0)
#endif

namespace {

constexpr int kM = 256, kF = 32, kNT = 256, kNW = 8;
constexpr int kKMax = 16;             // static outputs per frame (nStat <= 16): row length of the transposed DCT table
constexpr int kPartOff = 9216;        // float offset of the band level inside the FFT tile: behind P (257 x 32 floats)

// t1 -+ i t3 helper of the radix-4 butterfly whose fourth input is zero: d == 0 on entry
__device__ __forceinline__ void dft4_d0(float2 &a, float2 &b, float2 &c, float2 &d)
{
  const float2 t0 = cadd(a, c), t1 = csub(a, c), bb = b;
  a = cadd(t0, bb);
  c = csub(t0, bb);
  b = make_float2(t1.x + bb.y, t1.y - bb.x);   // t1 - i b
  d = make_float2(t1.x - bb.y, t1.y + bb.x);   // t1 + i b
}

// Dft<16>::run with rows NZR..15 known to be zero (NZR = 13 or 16)
template <int NZR>
__device__ __forceinline__ void dft16_first(float2 (&v)[16])
{
  dft4(v[0], v[4], v[8], v[12]);
  if (NZR <= 13) {
    dft4_d0(v[1], v[5], v[9], v[13]);
    dft4_d0(v[2], v[6], v[10], v[14]);
    dft4_d0(v[3], v[7], v[11], v[15]);
  } else {
    dft4(v[1], v[5], v[9], v[13]);
    dft4(v[2], v[6], v[10], v[14]);
    dft4(v[3], v[7], v[11], v[15]);
  }
  const float c1 = 0.92387953251128675613f, s1 = 0.38268343236508977173f;
  const float c2 = 0.70710678118654752440f;
  v[5] = cmul(v[5], make_float2(c1, -s1));
  { float2 a = v[6]; v[6] = make_float2(c2 * (a.x + a.y), c2 * (a.y - a.x)); }
  v[7] = cmul(v[7], make_float2(s1, -c1));
  { float2 a = v[9]; v[9] = make_float2(c2 * (a.x + a.y), c2 * (a.y - a.x)); }
  v[10] = cmul_mi(v[10]);
  { float2 a = v[11]; v[11] = make_float2(c2 * (a.y - a.x), -c2 * (a.x + a.y)); }
  v[13] = cmul(v[13], make_float2(s1, -c1));
  { float2 a = v[14]; v[14] = make_float2(c2 * (a.y - a.x), -c2 * (a.x + a.y)); }
  v[15] = cmul(v[15], make_float2(-c1, s1));
#pragma unroll
  for (int k1 = 0; k1 < 4; k1++) dft4(v[4 * k1], v[4 * k1 + 1], v[4 * k1 + 2], v[4 * k1 + 3]);
}

// real-FFT split of one pair: a = Z[k], b = Z[M-k], w = exp(-2 pi i k / N)  ->  4 |X[k]|^2, 4 |X[M-k]|^2
// (same statements as lld_kernel's split; the squares are accumulated with one FMA)
__device__ __forceinline__ void split_pair(float2 a, float2 b, float2 w, float &pk, float &pm)
{
  const float2 e2 = make_float2(a.x + b.x, a.y - b.y);
  const float2 o2 = make_float2(a.x - b.x, a.y + b.y);
  const float2 t2 = cmul(o2, w);
  const float xr = e2.x + t2.y, xi = e2.y - t2.x;
  const float yr = e2.x - t2.y, yi = e2.y + t2.x;
  pk = __fmaf_rn(xr, xr, __fmul_rn(xi, xi));
  pm = __fmaf_rn(yr, yr, __fmul_rn(yi, yi));
}

// eight samples of a landing zone whose fetch did not start 16-byte aligned (the PCM buffer is not): four 32-bit words
// from 16-bit loads, out of line -- a 16-byte aligned buffer never takes it
static __device__ OSM_COLD int4 load8_unaligned(const int16_t *s)
{
  const unsigned short *up = reinterpret_cast<const unsigned short *>(s);
  int w[4];
#pragma unroll
  for (int jj = 0; jj < 4; jj++) w[jj] = (int)((unsigned)up[2 * jj] | ((unsigned)up[2 * jj + 1] << 16));
  return make_int4(w[0], w[1], w[2], w[3]);
}

// one 8-byte shared-memory store (STS.64).  The sample tile's pairs are 8-byte aligned -- i is a multiple of 8, sPad is even
// (lld_fast_applies), the tile starts 16-byte aligned -- but the compiler cannot prove it and splits a float2 store in two.
__device__ __forceinline__ void sts_f2(float *dst, float a, float b)
{
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(smem_u32(dst)), "f"(a), "f"(b) : "memory");
}

// Fused Δ / ΔΔ emission of one interior tile (emit_interior of lld_common.cuh) with K static columns known at compile
// time: every thread's items are fixed -- the delta items tid and tid + NT, the static / delta-delta items of columns
// warp and warp + NW at row lane -- so the column / row split and the row offsets are constants of the thread, and only
// the ring slots move from tile to tile.  Same statements, same order, same results as emit_interior.
template <int K>
__device__ __forceinline__ void delta_item(const float *__restrict__ ring, float *__restrict__ Dbuf, float *__restrict__ outS,
                                           int slot0, float norm1, float rcp1, int item)
{
  constexpr int F = kF, DR = F + 4, dRows = F + 24, K3 = 3 * K, RM = 2 * F - 1;
  const int c = item / DR, tt = item - c * DR;
  const float *rc = ring + c * (2 * F);
  const int sl = slot0 + tt;
  const float dA = __fsub_rn(rc[(sl + 1) & RM], rc[(sl - 1) & RM]);
  const float dB = __fsub_rn(rc[(sl + 2) & RM], rc[(sl - 2) & RM]);
  const float dv = div_exact(__fadd_rn(dA, __fmul_rn(2.0f, dB)), norm1, rcp1);
  Dbuf[c * dRows + tt] = dv;
  const int rr = tt - 2;
  if (rr >= 0 && rr < F) outS[rr * K3 + K + c] = dv;
}

template <int K>
__device__ __forceinline__ void delta2_item(const float *__restrict__ Dbuf, float *__restrict__ outS, float norm2, float rcp2,
                                            int c, int lane)
{
  constexpr int dRows = kF + 24, K3 = 3 * K;
  const float *dt = Dbuf + c * dRows + lane + 2;                 // row t = r0 + lane sits at tt = lane + 2
  const float dA = __fsub_rn(dt[1], dt[-1]);
  const float dB = __fsub_rn(dt[2], dt[-2]);
  outS[lane * K3 + 2 * K + c] = div_exact(__fadd_rn(dA, __fmul_rn(2.0f, dB)), norm2, rcp2);
}

template <int K>
__device__ __forceinline__ void emit_interior_k(const float *__restrict__ ring, float *__restrict__ Dbuf,
                                                float *__restrict__ outS, int slot0, int rslot0,
                                                float norm1, float rcp1, float norm2, float rcp2, int tid)
{
  constexpr int F = kF, NT = kNT, NW = kNW, DR = F + 4, K3 = 3 * K, RM = 2 * F - 1;
  static_assert(K * DR > NT && K * DR <= 2 * NT && K > NW && K <= 2 * NW, "two delta items and two columns per thread");
  const int warp = tid >> 5, lane = tid & 31;
  delta_item<K>(ring, Dbuf, outS, slot0, norm1, rcp1, tid);
  if (tid < K * DR - NT) delta_item<K>(ring, Dbuf, outS, slot0, norm1, rcp1, tid + NT);
  const float *rs = ring + ((rslot0 + lane) & RM);               // statics -> outS
  outS[lane * K3 + warp] = rs[warp * (2 * F)];
  if (warp + NW < K) outS[lane * K3 + warp + NW] = rs[(warp + NW) * (2 * F)];
  __syncthreads();
  delta2_item<K>(Dbuf, outS, norm2, rcp2, warp, lane);          // delta-delta rows
  if (warp + NW < K) delta2_item<K>(Dbuf, outS, norm2, rcp2, warp + NW, lane);
  __syncthreads();
}

// KC: the static columns of the fused Δ / ΔΔ emission when known at compile time (13: MFCC 0..12), 0 = p.nStat
template <int NZR, int KC>
__global__ void __launch_bounds__(kNT, 2) lld512_kernel(const LldParams p)
{
  constexpr int M = kM, F = kF, NT = kNT, NW = kNW;
  using D16 = Dft<16>;

  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ ChunkCtx sCx[2];
  __shared__ int sTg[3];                // count, mis, lead of the tile in the landing zone (TileGeom), set with its fetch
  __shared__ int sRun[2];
  const SmemLayout L = make_layout(p, M, F);
  float2 *Z = reinterpret_cast<float2 *>(smem + L.zbuf);
  float *P = reinterpret_cast<float *>(smem + L.zbuf);
  float *samp = reinterpret_cast<float *>(smem + L.samp);
  float *raw = reinterpret_cast<float *>(smem + L.raw);
  unsigned char *rawPcm = smem + L.rawPcm;
  uint64_t *mbar = reinterpret_cast<uint64_t *>(smem + L.mbar);
  float4 *sWinLut = reinterpret_cast<float4 *>(smem + L.winLut);
  float2 *sTw = reinterpret_cast<float2 *>(smem + L.tw);
  float2 *sSplit = reinterpret_cast<float2 *>(smem + L.splitTw);
  float2 *sMelCoef = reinterpret_cast<float2 *>(smem + L.melCoef);
  int *sMelRange = reinterpret_cast<int *>(smem + L.melRange);
  float *sDct = reinterpret_cast<float *>(smem + L.dctCos);
  float *sLift = reinterpret_cast<float *>(smem + L.dctLift);
  float *ring = reinterpret_cast<float *>(smem + L.ring);
  float *Dbuf = reinterpret_cast<float *>(smem + L.zbuf);

  const int tid = threadIdx.x;
  const int warp = tid >> 5, f = tid & 31;

  if (tid == 0) mbar_init(mbar, 1);
  if (tid < 2) sRun[tid] = chunk_run_begin(p, blockIdx.x + tid);   // this CTA's chunks: [sRun[0], sRun[1])
  for (int i = tid; i < M; i += NT) sWinLut[i] = p.winLut[i];
  for (int i = tid; i < p.twCount; i += NT) sTw[i] = p.twiddles[i];
  for (int i = tid; i < M / 2 + 1; i += NT) sSplit[i] = p.splitTw[i];
  for (int i = tid; i < p.melVCount; i += NT) sMelCoef[i] = p.melVisit[i];
  for (int i = tid; i < p.nBands + 2; i += NT) { sMelRange[i] = p.melRange[i]; sMelRange[p.nBands + 2 + i] = p.melVB[i]; }
  for (int i = tid; i < p.nBands * kKMax; i += NT) {            // transposed, zero padded: sDct[band][kKMax]
    const int m = i / kKMax, c = i - m * kKMax;
    sDct[i] = (c < p.nStat) ? p.dctCos[c * p.dctStride + m] : 0.f;
  }
  for (int i = tid; i < p.nStat; i += NT) sLift[i] = p.dctLift[i];
  // lanes beyond a short tile read finite data (see lld_kernel): the sample tile and the first samples of its frames
  for (int i = tid; i < L.sampFloats; i += NT) samp[i] = 0.f;
  for (int i = tid; i < F; i += NT) raw[i] = 0.f;
  __syncthreads();

  const int hop = p.frameStep;
  const int S = hop + p.sPad;
  uint32_t phase = 0;
#ifdef OSM_LLD_PHASE_CLOCKS
  __shared__ unsigned long long sPh[kPhSlots];
  if (tid < kPhSlots) sPh[tid] = 0;
  const long long phT0 = clock64();
  long long phT = phT0;
#endif

  // The chunk context is CTA-uniform: it lives in shared memory (current / next chunk, alternating) instead of a dozen
  // registers per thread; thread 0 fills the next slot when it prefetches that chunk's first tile.
  int chunk = sRun[0];
  const int chunkEnd = sRun[1];
  if (chunk >= chunkEnd) return;
  int cpar = 0;
  if (tid == 0) {
    sCx[0] = load_chunk<F>(p, chunk);
    const TileGeom g0 = tile_geom<F>(p, sCx[0], 0);
    sTg[0] = g0.count; sTg[1] = g0.mis; sTg[2] = g0.lead;
    mbar_expect_tx(mbar, g0.bytes);
    bulk_g2s(rawPcm, g0.src, g0.bytes, mbar);
  }
  __syncthreads();
  int j = 0;
  int emitted = sCx[0].a;

  // pass 2: butterflies of this warp; bins of the pair slots (see the file header).  Slots 0..7 hold k = wl + 16 q
  // (and M - k = 256 - wl - 16 q), slots 8..15 hold k = 256 - wh - 16 q (and M - k = wh + 16 q): warps 1..7 have
  // wl = wh = warp; warp 0 has wl = 8 (butterfly 8) and wh = 0 (butterfly 0), so every address is base + constant
  const int tA = (warp == 0) ? 0 : warp, tB = (warp == 0) ? 8 : 16 - warp;
  const int wl = (warp == 0) ? 8 : warp, wh = (warp == 0) ? 0 : warp;
  const int melBs = p.melSplit[warp], melBe = p.melSplit[warp + 1];

  while (chunk < chunkEnd) {
    const ChunkCtx &cx = sCx[cpar];

    // ================= stage: PCM (landing zone) -> float -> pre-emphasis -> sample tile =================
    mbar_wait(mbar, phase);
    phase ^= 1;
    {
      // the tile's geometry comes from the thread that issued its fetch (sTg), not from every thread's 64-bit arithmetic
      const int count = sTg[0], mis = sTg[1], lead = sTg[2];
      const int16_t *rp = reinterpret_cast<const int16_t *>(rawPcm + mis) + lead;
      const bool aligned = (mis == 0);
      const bool hasLead = lead > 0;
      const float ks = p.preDe ? p.preK : -p.preK;
#pragma unroll 1
      for (int i = tid * 8; i < count; i += NT * 8) {
        int4 w4;
        if (aligned) w4 = *reinterpret_cast<const int4 *>(rp + i);
        else w4 = load8_unaligned(rp + i);
        const int wds[4] = {w4.x, w4.y, w4.z, w4.w};
        float x[8], y[8];
#pragma unroll
        for (int jj = 0; jj < 4; jj++) {
          x[2 * jj] = div32767((float)(short)(wds[jj] & 0xffff));
          x[2 * jj + 1] = div32767((float)(wds[jj] >> 16));
        }
        if (p.preemph) {
          // vectorPreemphasis.cpp:96-104 : x[n] -/+ k * x[n-1], two roundings
          float xprev = 0.f;
          if (i > 0 || hasLead) xprev = div32767((float)rp[i - 1]);
#pragma unroll
          for (int jj = 0; jj < 8; jj++) y[jj] = __fadd_rn(x[jj], __fmul_rn(ks, (jj == 0) ? xprev : x[jj - 1]));
        } else {
#pragma unroll
          for (int jj = 0; jj < 8; jj++) y[jj] = x[jj];
        }
        const int q = (int)__umulhi((unsigned)i, p.hopMagic);      // i / hop
        float *dst = samp + i + q * p.sPad;
        if (i == q * hop && q < F) raw[q] = x[0];                  // first sample of frame q, not pre-emphasised
#pragma unroll
        for (int jj = 0; jj < 8; jj += 2) sts_f2(dst + jj, y[jj], y[jj + 1]);
      }
    }
    __syncthreads();
    if (tid == 0) {
      if (j + 1 < cx.nT) {
        const TileGeom gn = tile_geom<F>(p, cx, j + 1);
        sTg[0] = gn.count; sTg[1] = gn.mis; sTg[2] = gn.lead;     // read after this tile's barriers
        mbar_expect_tx(mbar, gn.bytes);
        bulk_g2s(rawPcm, gn.src, gn.bytes, mbar);
      } else if (chunk + 1 < chunkEnd) {
        const ChunkCtx cn = load_chunk<F>(p, chunk + 1);
        sCx[cpar ^ 1] = cn;                           // read by everyone after the barriers of this tile
        const TileGeom gn = tile_geom<F>(p, cn, 0);
        sTg[0] = gn.count; sTg[1] = gn.mis; sTg[2] = gn.lead;
        mbar_expect_tx(mbar, gn.bytes);
        bulk_g2s(rawPcm, gn.src, gn.bytes, mbar);
      }
    }
    OSM_PHASE(kPhStage);

    // ================= FFT pass 1: window, radix 16, twiddles -> Z =================
    {
      const float *sampF = samp + f * S;
      const float2 *tw0 = sTw + p.twOff[0];
#pragma unroll 1
      for (int t = warp; t < 16; t += NW) {
        float2 v[16];
#pragma unroll
        for (int r = 0; r < 16; r++) {
          if (r < NZR) {
            const float4 wl = sWinLut[t + 16 * r];   // (w[2e], w[2e+1], offset, #valid); padding: weight 0, offset 0
            const float2 x = *reinterpret_cast<const float2 *>(sampF + __float_as_int(wl.z));
            v[r] = make_float2(__fmul_rn(x.x, wl.x), __fmul_rn(x.y, wl.y));   // windower.cpp:226
          } else {
            v[r] = make_float2(0.f, 0.f);
          }
        }
        if (t == 0 && p.preemph)      // first sample of the frame, vectorPreemphasis.cpp:94
          v[0].x = __fmul_rn(__fmul_rn(p.oneMinusK, raw[f]), sWinLut[0].x);
        dft16_first<NZR>(v);
        const float2 *twj = tw0 + t * 16;
#pragma unroll
        for (int q = 1; q < 16; q++) v[D16::out(q)] = cmul(v[D16::out(q)], twj[q]);
        float2 *zp = Z + t * F + f;
#pragma unroll
        for (int q = 0; q < 16; q++) zp[(16 * q) * F] = v[D16::out(q)];
      }
    }
    __syncthreads();
    OSM_PHASE(kPhPass1);

    // ================= FFT pass 2 + real-FFT split + power, in registers =================
    {
      float2 A[16], v[16];
#pragma unroll 2
      for (int h = 0; h < 2; h++) {
        const float2 *zp = Z + ((h ? tB : tA) * 16) * F + f;
#pragma unroll
        for (int r = 0; r < 16; r++) v[r] = zp[r * F];
        D16::run(v);
        if (h == 0) {
#pragma unroll
          for (int r = 0; r < 16; r++) A[r] = v[r];
        }
      }
      // X[tA + 16 q] = A[out(q)] =: a_q ; X[tB + 16 q] = v[out(q)] =: b_q ; slot q pairs a_q with b_{15-q}
      const float2 x0 = A[D16::out(0)];
      if (warp == 0) {
        // a = butterfly 0 (X[16 q]), b = butterfly 8 (X[8 + 16 q]):
        //   slots 0..7 : k = 8 + 16 q   -> (b_q, b_{15-q})                         : a'_q = b_q
        //   slots 8..15: k = 256 - 16 q -> Z[k] = a_{16-q} = b'_{15-q}, Z[M-k] = a_q : b'_j = a_{j+1}, j = 0..7
        float2 na[8], nb[8];
#pragma unroll
        for (int q = 0; q < 8; q++) { na[q] = v[D16::out(q)]; nb[q] = A[D16::out(q + 1)]; }
#pragma unroll
        for (int q = 0; q < 8; q++) { A[D16::out(q)] = na[q]; v[D16::out(q)] = nb[q]; }
      }
      float pk[16], pm[16];
      {
        const float2 *swl = sSplit + wl, *swh = sSplit + (256 - wh);
#pragma unroll
        for (int q = 0; q < 16; q++) {
          const float2 aq = A[D16::out(q)], bq = v[D16::out(15 - q)];
          if (q < 8) split_pair(aq, bq, swl[16 * q], pk[q], pm[q]);        // aq = Z[k], bq = Z[M-k], k = wl + 16 q
          else       split_pair(bq, aq, swh[-16 * q], pk[q], pm[q]);       // bq = Z[k], aq = Z[M-k], k = 256 - wh - 16 q
        }
      }
      __syncthreads();   // every warp has read its part of Z before P (aliasing Z) is written
      {
        float *Plo = P + wl * F + f, *Plm = P + (256 - wl) * F + f;
        float *Phi = P + (256 - wh) * F + f, *Phm = P + wh * F + f;
#pragma unroll
        for (int q = 0; q < 8; q++) { Plo[(16 * q) * F] = pk[q]; Plm[(-16 * q) * F] = pm[q]; }
#pragma unroll
        for (int q = 8; q < 16; q++) {
          Phi[(-16 * q) * F] = pk[q];
          if (q > 8 || warp != 0) Phm[(16 * q) * F] = pm[q];               // warp 0, slot 8: k = 128 = M - k
        }
      }
      if (warp == 0) {
        // k = 0: a = b = Z[0], w = 1 -> 2 X[0] = 2 (re + im), 2 X[M] = 2 (re - im), both real
        const float xr = 2.0f * (x0.x + x0.y), yr = 2.0f * (x0.x - x0.y);
        P[f] = __fmul_rn(xr, xr);
        P[M * F + f] = __fmul_rn(yr, yr);
      }
    }
    __syncthreads();
    OSM_PHASE(kPhPass2);

    // ================= mel filterbank (melspec.cpp:543-569) + log (mfcc.cpp:239-243) =================
    // the band level lives behind the power spectrum (P + kPartOff), not in the sample tile
    float *melS = P + kPartOff;
    if (melBs < melBe) {
      const int *sVB = sMelRange + p.nBands + 2;
      float cur = 0.f;
      for (int r = melBs; r <= melBe; r++) {
        float nxt = 0.f;
        const float *pp = P + sMelRange[r] * F + f;
        const int v0 = sVB[r];
        const float4 *cp = reinterpret_cast<const float4 *>(sMelCoef + v0);
#pragma unroll 1
        for (int q = (sVB[r + 1] - v0) >> 2; q > 0; q--, pp += 4 * F, cp += 2) {
          const float p0 = pp[0], p1 = pp[F], p2 = pp[2 * F], p3 = pp[3 * F];
          const float4 wa = cp[0], wb = cp[1];
          cur = __fmaf_rn(p0, wa.x, cur); nxt = __fmaf_rn(p0, wa.y, nxt);
          cur = __fmaf_rn(p1, wa.z, cur); nxt = __fmaf_rn(p1, wa.w, nxt);
          cur = __fmaf_rn(p2, wb.x, cur); nxt = __fmaf_rn(p2, wb.y, nxt);
          cur = __fmaf_rn(p3, wb.z, cur); nxt = __fmaf_rn(p3, wb.w, nxt);
        }
        if (r > melBs) {
          float mval = __fmul_rn(cur, p.melScale);
          if (p.doLog) mval = (mval < p.melfloor) ? p.logMelfloor : logf(mval);
          melS[(r - 1) * F + f] = mval;
        }
        cur = nxt;
      }
    }
    __syncthreads();
    OSM_PHASE(kPhMel);

    // ================= DCT-II + lifter (mfcc.cpp:251-272), the reference's m = 0 .. nBands-1 accumulation order =================
    // table transposed and zero padded, sDct[band][kKMax]: warp w evaluates coefficients 2w and 2w+1 together (one 8-byte
    // table read and one band value feed two dot products); the padding columns are zero
    const int ringBase = (j & 1) * F;
    {
      const int i = 2 * warp;
      if (i < p.nStat) {
        const float2 *cc = reinterpret_cast<const float2 *>(sDct + i);
        const float *lp = melS + f;
        float a0 = 0.f, a1 = 0.f;
#pragma unroll 4
        for (int m = 0; m < p.nBands; m++, lp += F, cc += kKMax / 2) {
          const float l0 = lp[0];
          const float2 c = cc[0];
          a0 = __fmaf_rn(l0, c.x, a0); a1 = __fmaf_rn(l0, c.y, a1);
        }
        ring[i * (2 * F) + ringBase + f] = __fmul_rn(a0, sLift[i]);
        if (i + 1 < p.nStat) ring[(i + 1) * (2 * F) + ringBase + f] = __fmul_rn(a1, sLift[i + 1]);
      }
    }
    __syncthreads();
    OSM_PHASE(kPhDct);

    // ================= store (same statements as lld_kernel) =================
    const int tfs = cx.s0 + j * F;                    // first static frame of this tile
    if (!p.fused) {
      const int tot = min(F, cx.sEnd - tfs) * p.nStat;
      for (int idx = tid; idx < tot; idx += NT) {
        const int ff = idx / p.nStat, c = idx - ff * p.nStat;
        p.out[(cx.row0 + tfs + ff) * p.outStride + p.outCol + c] = ring[c * (2 * F) + ringBase + ff];
      }
    } else {
      const int K = KC ? KC : p.nStat, W1 = p.fW1, W2 = p.fW2, H = W1 + W2;
      const int T = cx.T;
      const int r0 = emitted;
      const int r1 = (j + 1 == cx.nT) ? cx.b : min(tfs + F - H, cx.b);
      const int T1 = T + W1, c01 = max(T - W1, 0), c02 = max(c01 - W2, 0);
      const float norm1 = p.fNorm1, norm2 = p.fNorm2;
      const int d0 = max(r0 - W2, 0), d1 = min(r1 + W2, T1);
      const int dRows = F + 24;
      const int K3 = 3 * K;
      const int nr = r1 - r0;
      float *o = p.out + (cx.row0 + r0) * (long long)K3;
      // the rows are staged at the global rows' offset modulo 16 bytes (the 3 floats of slack are behind Dbuf in the
      // dead FFT tile), so that the store below moves them 16 bytes at a time
      const int oMis = (int)((reinterpret_cast<uintptr_t>(o) >> 2) & 3);
      float *outS = Dbuf + ((K * dRows + 3) & ~3) + oMis;
      const bool interior1 = (d0 >= W1) && (d1 + W1 <= T);
      const bool interior2 = (r0 >= W2) && (r1 <= c02);
      if (interior1 && interior2 && W1 == 2 && W2 == 2 && nr == F) {
        if constexpr (KC != 0)
          emit_interior_k<KC>(ring, Dbuf, outS, d0 - cx.s0, r0 - cx.s0, norm1, p.fRcp1, norm2, p.fRcp2, tid);
        else
          emit_interior<F, NT>(ring, Dbuf, outS, K, dRows, d0 - cx.s0, r0 - cx.s0, norm1, p.fRcp1, norm2, p.fRcp2, tid);
      } else if (KC != 0 && W1 == 2 && W2 == 2) {
        if constexpr (KC != 0)    // K and the windows at compile time: the window sums are straight-line code
          emit_edge<F, NW, KC, 2>(ring, Dbuf, outS, K, W1, W2, T, T1, c01, c02, cx.s0, r0, r1, d0, d1, dRows, norm1, p.fRcp1, norm2, p.fRcp2, warp, f);
      } else {
        emit_edge<F, NW>(ring, Dbuf, outS, K, W1, W2, T, T1, c01, c02, cx.s0, r0, r1, d0, d1, dRows, norm1, p.fRcp1, norm2, p.fRcp2, warp, f);
      }
      OSM_PHASE(kPhEmit);
      {
        // rows [r0, r1) are contiguous in p.out: up to 3 leading floats, 16-byte groups, up to 3 trailing floats
        const int n = nr * K3;
        const int head = min((4 - oMis) & 3, n);
        const int nv = (n - head) >> 2, tail = head + 4 * nv;
        if (tid < head) o[tid] = outS[tid];
        const float4 *sv = reinterpret_cast<const float4 *>(outS + head);
        float4 *gv = reinterpret_cast<float4 *>(o + head);
#pragma unroll 1
        for (int i = tid; i < nv; i += NT) gv[i] = sv[i];
        if (tid < n - tail) o[tail + tid] = outS[tail + tid];
      }
      emitted = r1;
    }
    OSM_PHASE(kPhStore);
#ifdef OSM_LLD_PHASE_CLOCKS
    if (tid == 0) sPh[kPhTiles]++;
#endif

    j++;
    if (j == cx.nT) {
      chunk++;
      j = 0;
      cpar ^= 1;
      if (chunk < chunkEnd) emitted = sCx[cpar].a;
    }
  }
#ifdef OSM_LLD_PHASE_CLOCKS
  if (tid == 0) {
    sPh[kPhKernel] = (unsigned long long)(clock64() - phT0);
    for (int k = 0; k < kPhSlots; k++)
      if (k != kPhKernelMax) atomicAdd(&gLld512Phase[k], sPh[k]);
    atomicMax(&gLld512Phase[kPhKernelMax], sPh[kPhKernel]);
  }
#endif
}

template <int NZR, int KC>
cudaError_t launch_fast_t(const LldParams &p, int numSMs, cudaStream_t st, LldLaunchInfo *info, bool launch)
{
  const size_t smem = (size_t)make_layout(p, kM, kF).total;
  auto kern = lld512_kernel<NZR, KC>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  int occ = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, kNT, smem);
  if (e != cudaSuccess) return e;
  if (occ < 1) return cudaErrorLaunchOutOfResources;
  const int grid = launch ? p.nRuns : numSMs * occ;
  if (info) {
    info->grid = grid; info->block = kNT; info->smem = smem; info->nChunks = p.nChunks;
    info->kernel = NZR == 13 ? "lld512_kernel<13>" : "lld512_kernel<16>";
  }
  if (!launch) return cudaSuccess;
  kern<<<grid, kNT, smem, st>>>(p);
  return cudaGetLastError();
}

}  // namespace

bool lld_fast_applies(const LldParams &p, int nfft)
{
  return nfft == 512 && !p.narrow && p.opKind == 0 && p.magOut == nullptr && p.melUsePower && p.nChan == 1 &&
         p.frameCenter == 0 && p.frameStep % 8 == 0 && p.frameSize % 8 == 0 && p.frameSize <= 512 && !p.hasWinOffset && p.nStat <= kKMax &&
         ((p.frameStep + p.sPad) % 2) == 0;
}

cudaError_t launch_lld_fast(const LldParams &p, int numSMs, cudaStream_t st, LldLaunchInfo *info, bool launch)
{
  // 13 static columns (MFCC 0..12, the shipped MFCC12 sets) take the compile-time emission
  if (p.frameSize <= 416) {
    if (p.nStat == 13) return launch_fast_t<13, 13>(p, numSMs, st, info, launch);
    return launch_fast_t<13, 0>(p, numSMs, st, info, launch);
  }
  if (p.nStat == 13) return launch_fast_t<16, 13>(p, numSMs, st, info, launch);
  return launch_fast_t<16, 0>(p, numSMs, st, info, launch);
}

#ifdef OSM_LLD_PHASE_CLOCKS
// copies the phase sums of every launch since the previous call into out[kPhSlots] and clears them
extern "C" __attribute__((visibility("default"))) int osm_b200_lld512_phase_clocks(unsigned long long *out)
{
  cudaError_t e = cudaMemcpyFromSymbol(out, gLld512Phase, sizeof(gLld512Phase));
  if (e == cudaSuccess) {
    static const unsigned long long zero[kPhSlots] = {};
    e = cudaMemcpyToSymbol(gLld512Phase, zero, sizeof(zero));
  }
  return (int)e;
}
#endif

}  // namespace osm
