// lld_kernel.cuh -- the general fused per-frame LLD kernel (lld_kernel) and launch_lld_kernel, which picks its instance (sm_90a).
//
// Design (see DESIGN.md): one persistent CTA processes "tiles" of F consecutive frames of one
// utterance.  Inside a tile every thread keeps the mapping  lane -> frame  for ALL phases:
//
//   stage   PCM (int16, HBM, coalesced 16-byte loads) -> float -> pre-emphasis -> smem
//   FFT     real FFT as an M = N/2 point complex FFT, in-place decimation-in-frequency with
//           register radix-8/16 butterflies; the data tile lives in shared memory as
//           Z[element][frame], so every warp-wide access is conflict free and every table
//           (window, twiddles, mel weights, DCT) is warp-uniform (broadcast)
//   split   real-FFT post-processing + |X|^2  -> P[bin][frame]
//   mel     two-tap triangular filterbank, sequential in the bin index exactly like the
//           reference's loop (lldcore/melspec.cpp:543-553) -> bit-faithful summation order
//   dct     log, DCT-II, lifter (lldcore/mfcc.cpp:238-273), again in the reference's order
//   store   rows of the output level
//
// The temporal regression stages (cDeltaRegression / cContourSmoother) run in a second,
// memory-bound kernel (post_kernel) with the reference's edge / phantom-frame semantics.
//
// Arithmetic that the reference performs in a fixed float order (conversion, pre-emphasis,
// window, power, mel, log, DCT, lifter, delta) uses explicit non-fused __fmul_rn/__fadd_rn so
// that, given identical inputs, results are bit-identical to the x86-64 reference build
// (which has no FMA contraction).  Only the FFT itself uses FMA freely.
#pragma once
#include <string>

#include "fft_radix.cuh"
#include "kernels.cuh"
#include "lld_common.cuh"

namespace osm {

// ------------------------------------------------------------------------------------------
// the fused kernel
// ------------------------------------------------------------------------------------------
// GEN = false: the MFCC-only instance (band op = cMfcc, no magnitude level dump); the PLP back end and
// the magnitude dump compile away.  GEN = true: band op and dump selected at run time.
// F32: the instance for pre-converted mono float samples (LldParams::pcmF32).
// CENTRED: the GEN instance for a centred framer (LldParams::frameCenter != 0), whose first tiles start before the utterance.
template <int M, int F, int NT, int MINB, bool VEC2, bool GEN, bool F32, bool CENTRED = false>
__global__ void __launch_bounds__(NT, MINB) lld_kernel(const LldParams p)
{
  const int opKind = GEN ? p.opKind : 0;
  float *const magOut = GEN ? p.magOut : nullptr;
  constexpr int NW = NT / 32, G = 32 / F, NVW = NW * G;
  constexpr int NBINS = M + 1;
  constexpr int NPAIR = M / 2 + 1;                 // pairs (k, M-k), k = 0..M/2
  constexpr int PAIRS_PER_VW = (NPAIR + NVW - 1) / NVW;
  using Fc = Fact<M>;

  extern __shared__ __align__(16) unsigned char smem[];
  const SmemLayout L = make_layout(p, M, F);
  float2 *Z = reinterpret_cast<float2 *>(smem + L.zbuf);
  float *P = reinterpret_cast<float *>(smem + L.zbuf);   // aliases Z (used after the split)
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
  float *sEql = reinterpret_cast<float *>(smem + L.eql);
  float *melS = reinterpret_cast<float *>(smem + L.melS);
  float *ring = reinterpret_cast<float *>(smem + L.ring);   // [nMfcc][2F], slot = (frame - chunk.s0) & (2F-1)
  float *Dbuf = reinterpret_cast<float *>(smem + L.zbuf);  // delta level rows (aliases Z, dead after mel)

  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int f = lane & (F - 1);
  const int vw = warp * G + lane / F;

  // ---- one-time setup: barrier, this CTA's chunks [sRun[0], sRun[1]), constant tables -> smem, zero the sample tile ----
  __shared__ int sRun[2];
  if (tid == 0) mbar_init(mbar, 1);
  if (tid < 2) sRun[tid] = chunk_run_begin(p, blockIdx.x + tid);
  for (int i = tid; i < M; i += NT) sWinLut[i] = p.winLut[i];
  for (int i = tid; i < p.twCount; i += NT) sTw[i] = p.twiddles[i];
  for (int i = tid; i < NPAIR; i += NT) sSplit[i] = p.splitTw[i];
  if (opKind >= 0) {
    for (int i = tid; i < p.melVCount; i += NT) sMelCoef[i] = p.melVisit[i];
    for (int i = tid; i < p.nBands + 2; i += NT) { sMelRange[i] = p.melRange[i]; sMelRange[p.nBands + 2 + i] = p.melVB[i]; }
    for (int i = tid; i < p.dctRows * p.dctStride; i += NT) sDct[i] = p.dctCos[i];
    if (opKind == 1) for (int i = tid; i < p.nBands; i += NT) sEql[i] = p.plpEql[i];
    for (int i = tid; i < p.nStat; i += NT) sLift[i] = p.dctLift[i];
  }
  // Lanes beyond a short tile compute frames that are never stored, from the sample tile and from raw[] (the frames' first
  // samples, written by the staging only for frames that start inside the tile).  Both start finite: the mel phase's
  // zero-weight padding entries read up to three bins past the spectrum, which in P's storage (aliasing Z) hold FFT
  // values of other lanes, and 0 * NaN would turn a valid frame's band into NaN.
  for (int i = tid; i < L.sampFloats; i += NT) samp[i] = 0.f;
  for (int i = tid; i < F; i += NT) raw[i] = 0.f;
  __syncthreads();

  const int hop = p.frameStep, nChan = p.nChan;
  const int S = hop + p.sPad;
  uint32_t phase = 0;

  int chunk = sRun[0];
  const int chunkEnd = sRun[1];
  if (chunk >= chunkEnd) return;
  ChunkCtx cx = load_chunk<F, CENTRED>(p, chunk);
  int j = 0;
  int emitted = cx.a;                 // next output row of the current chunk to be written
  if (tid == 0) {
    const TileGeom g0 = tile_geom<F, CENTRED>(p, cx, 0);
    mbar_expect_tx(mbar, g0.bytes);
    bulk_g2s(rawPcm, g0.src, g0.bytes, mbar);
  }

  while (chunk < chunkEnd) {
    const TileGeom tg = tile_geom<F, CENTRED>(p, cx, j);
    const int nf = tg.nf, count = tg.count;

    // ================= stage: PCM (smem, prefetched by the bulk copy) -> float -> pre-emphasis -> smem =================
    mbar_wait(mbar, phase);
    phase ^= 1;
    {
      const int16_t *rp = reinterpret_cast<const int16_t *>(rawPcm + tg.mis) + tg.lead * nChan;   // sample frame 0 of the tile
      const bool fastLoad = (tg.mis == 0) && (nChan <= 2) && !F32;
      const bool fastStore = (p.sPad == 0) || (hop % 8 == 0);
      if (CENTRED && tg.pad > 0) stage_padded_tile<F, NT, F32>(rp, tg.pad, count, hop, p.sPad, nChan, p.preemph ? (p.preDe ? p.preK : -p.preK) : 0.f, samp, raw, tid);
      else for (int c = tid; c * 8 < count; c += NT) {
        const int i = c * 8;
        const int nvalid = min(8, count - i);
        float x[8];
        if (fastLoad && nvalid == 8) {
          if (nChan == 1) {
            const int4 w4 = *reinterpret_cast<const int4 *>(rp + i);
            const int wds[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
            for (int jj = 0; jj < 4; jj++) {
              x[2 * jj] = div32767((float)(short)(wds[jj] & 0xffff));
              x[2 * jj + 1] = div32767((float)(wds[jj] >> 16));
            }
          } else {
            const int4 a4 = *reinterpret_cast<const int4 *>(rp + 2 * i);
            const int4 b4 = *reinterpret_cast<const int4 *>(rp + 2 * i + 8);
            const int wds[8] = {a4.x, a4.y, a4.z, a4.w, b4.x, b4.y, b4.z, b4.w};
#pragma unroll
            for (int jj = 0; jj < 8; jj++) {
              const float l = (float)(short)(wds[jj] & 0xffff), r = (float)(wds[jj] >> 16);
              x[jj] = div32767(__fadd_rn(l, r) * 0.5f);
            }
          }
        } else {
#pragma unroll
          for (int jj = 0; jj < 8; jj++) x[jj] = (jj < nvalid) ? pcm_to_float_slow<F32>(rp + (i + jj) * nChan, nChan) : 0.f;
        }
        float y[8];
        if (p.preemph) {
          // vectorPreemphasis.cpp:96-104 : x[n] -/+ k * x[n-1], two roundings
          float xprev = 0.f;
          if (i > 0 || tg.lead > 0) {
            if (nChan == 1) xprev = div32767((float)rp[i - 1]);
            else xprev = pcm_to_float_slow<F32>(rp + (i - 1) * nChan, nChan);
          }
          // x - k*xp == x + (-k)*xp exactly: one signed coefficient instead of a per-sample select
          const float ks = p.preDe ? p.preK : -p.preK;
#pragma unroll
          for (int jj = 0; jj < 8; jj++) y[jj] = __fadd_rn(x[jj], __fmul_rn(ks, (jj == 0) ? xprev : x[jj - 1]));
        } else {
#pragma unroll
          for (int jj = 0; jj < 8; jj++) y[jj] = x[jj];
        }
        // i / hop; the magic number of hop 1 (2^32) does not fit 32 bits
        const int q = (hop == 1) ? i : (int)__umulhi((unsigned)i, p.hopMagic);
        const int r = i - q * hop;
        float *dst = samp + i + q * p.sPad;
        if (fastStore && nvalid == 8 && r + 8 <= hop) {
          // the 8 samples lie inside one frame step: no pad crossing, at most one frame start
          if (r == 0 && q < F) raw[q] = x[0];
#pragma unroll
          for (int jj = 0; jj < 8; jj += 2) *reinterpret_cast<float2 *>(dst + jj) = make_float2(y[jj], y[jj + 1]);
        } else {
          int qq = q, rr = r;
#pragma unroll
          for (int jj = 0; jj < 8; jj++) {
            if (jj < nvalid) {
              if (rr == 0 && qq < F) raw[qq] = x[jj];
              dst[jj] = y[jj];
              rr++;
              if (rr == hop) { rr = 0; qq++; dst += p.sPad; }
            }
          }
        }
      }
    }
    __syncthreads();
    // the landing zone is free again: fetch the next tile's PCM while this one is processed
    if (tid == 0) {
      if (j + 1 < cx.nT) {
        const TileGeom gn = tile_geom<F, CENTRED>(p, cx, j + 1);
        mbar_expect_tx(mbar, gn.bytes);
        bulk_g2s(rawPcm, gn.src, gn.bytes, mbar);
      } else if (chunk + 1 < chunkEnd) {
        const ChunkCtx cn = load_chunk<F, CENTRED>(p, chunk + 1);
        const TileGeom gn = tile_geom<F, CENTRED>(p, cn, 0);
        mbar_expect_tx(mbar, gn.bytes);
        bulk_g2s(rawPcm, gn.src, gn.bytes, mbar);
      }
    }

    // ================= FFT =================
    {
      const float *sampF = samp + f * S;
      fft_stage<M, F, NVW, Fc::R0, M, true, false, VEC2>(Z, sampF, raw, sWinLut, sTw + p.twOff[0], p, vw, f);
      __syncthreads();
      if constexpr (Fc::NS == 2) {
        fft_stage<M, F, NVW, Fc::R1, M / Fc::R0, false, true, VEC2>(Z, nullptr, nullptr, nullptr, nullptr, p, vw, f);
      } else {
        fft_stage<M, F, NVW, Fc::R1, M / Fc::R0, false, false, VEC2>(Z, nullptr, nullptr, nullptr, sTw + p.twOff[1], p, vw, f);
        __syncthreads();
        fft_stage<M, F, NVW, Fc::R2, M / (Fc::R0 * Fc::R1), false, true, VEC2>(Z, nullptr, nullptr, nullptr, nullptr, p, vw, f);
      }
      __syncthreads();
    }

    // ================= real-FFT split + power spectrum =================
    // X[k] = E - i W^k O,  X[M-k] = conj(E + i W^k O),  E = (Z[k]+conj(Z[M-k]))/2, O = (Z[k]-conj(Z[M-k]))/2
    {
      float pk[PAIRS_PER_VW], pm[PAIRS_PER_VW];
#pragma unroll
      for (int i = 0; i < PAIRS_PER_VW; i++) {
        const int k = vw + i * NVW;
        pk[i] = 0.f; pm[i] = 0.f;
        if (k < NPAIR) {
          const float2 a = Z[fft_pos<M>(k) * F + f];
          const float2 b = Z[fft_pos<M>((M - k) & (M - 1)) * F + f];   // Z[M] == Z[0]
          const float2 w = sSplit[k];
          const float2 e2 = make_float2(a.x + b.x, a.y - b.y);         // 2E
          const float2 o2 = make_float2(a.x - b.x, a.y + b.y);         // 2O
          const float2 t2 = cmul(o2, w);                               // 2 W^k O
          // 2 X[k] = e2 - i t2 ; 2 conj(X[M-k]) = e2 + i t2
          const float xr = e2.x + t2.y, xi = e2.y - t2.x;
          const float yr = e2.x - t2.y, yi = e2.y + t2.x;
          // 4 |X|^2: fftmagphase.cpp:215-221 computes sqrt(re*re+im*im), melspec.cpp:524 squares it
          // again; the power path keeps re*re+im*im (<= 1.5 ulp apart, below the FFT's own noise
          // floor).  The factor 1/2 of X (1/4 of the power) is an exact power-of-two scaling that
          // commutes with every rounding downstream; it is folded into melScale on the host.
          pk[i] = __fadd_rn(__fmul_rn(xr, xr), __fmul_rn(xi, xi));
          pm[i] = __fadd_rn(__fmul_rn(yr, yr), __fmul_rn(yi, yi));
        }
      }
      if (magOut != nullptr || !p.melUsePower) {
        // magnitude needed (kept out of the loop above: this is the rarely used variant).  A
        // non-fused consumer reads the magnitude level |X| = 0.5 * sqrt(a^2+b^2) (exact scaling,
        // fftmagphase.cpp:215-221); the band op then squares it like melspec.cpp:524 does (melScale
        // carries no 1/4 in this mode)
        float *mo = (magOut != nullptr) ? magOut + ((size_t)(cx.tile0 + j) * NBINS) * F + f : nullptr;
#pragma unroll
        for (int i = 0; i < PAIRS_PER_VW; i++) {
          const int k = vw + i * NVW;
          if (k < NPAIR) {
            const float mk = 0.5f * __fsqrt_rn(pk[i]);
            const float mm = 0.5f * __fsqrt_rn(pm[i]);
            if (mo != nullptr) {
              mo[(size_t)k * F] = mk;
              if (k != M - k) mo[(size_t)(M - k) * F] = mm;
            }
            const bool sq = (mo != nullptr) && p.melUsePower;
            pk[i] = sq ? __fmul_rn(mk, mk) : mk;
            pm[i] = sq ? __fmul_rn(mm, mm) : mm;
          }
        }
      }
      __syncthreads();   // all Z reads done before P (aliasing Z) is written
#pragma unroll
      for (int i = 0; i < PAIRS_PER_VW; i++) {
        const int k = vw + i * NVW;
        if (k < NPAIR) {
          P[k * F + f] = pk[i];
          if (k != M - k) P[(M - k) * F + f] = pm[i];
        }
      }
    }
    __syncthreads();

    if (opKind >= 0) {
    // ================= mel filterbank (melspec.cpp:543-569) + log (mfcc.cpp:239-243) =================
    // range r holds the bins whose lower band is r-1: band[r-1] += p*w ; band[r] += p*(1-w), visited
    // in ascending bin order like the reference loop (same summation order per band; the products
    // are fused into the sums, which only removes roundings).
    {
      const int bs = p.melSplit[vw], be = p.melSplit[vw + 1];
      if (bs < be) {
        const int *sVB = sMelRange + p.nBands + 2;
        float cur = 0.f;
        // One loop for all ranges: every range is walked in groups of 4 visit entries (zero-weight
        // padding at its end multiplies the following bins by 0), so there is no remainder code and the
        // addresses inside a group are immediates.  Range bs only feeds band bs: its "current band"
        // sum is a throw-away and no value is stored after it.
        for (int r = bs; r <= be; r++) {
          float nxt = 0.f;
          const float *pp = P + sMelRange[r] * F + f;
          const float2 *cp = sMelCoef + sVB[r];
#pragma unroll 1
          for (int q = (sVB[r + 1] - sVB[r]) >> 2; q > 0; q--, pp += 4 * F, cp += 4) {
            const float p0 = pp[0], p1 = pp[F], p2 = pp[2 * F], p3 = pp[3 * F];
            const float2 w0 = cp[0], w1 = cp[1], w2 = cp[2], w3 = cp[3];
            cur = __fmaf_rn(p0, w0.x, cur); nxt = __fmaf_rn(p0, w0.y, nxt);
            cur = __fmaf_rn(p1, w1.x, cur); nxt = __fmaf_rn(p1, w1.y, nxt);
            cur = __fmaf_rn(p2, w2.x, cur); nxt = __fmaf_rn(p2, w2.y, nxt);
            cur = __fmaf_rn(p3, w3.x, cur); nxt = __fmaf_rn(p3, w3.y, nxt);
          }
          if (r == bs) { cur = nxt; continue; }
          float mval = __fmul_rn(cur, p.melScale);
          if (opKind == 2) mval = tone_mean(mval, sDct[r - 1], p.toneSqrt);       // tonespec.cpp:424-434 (doLog = 0)
          if (p.doLog) mval = (mval < p.melfloor) ? p.logMelfloor : logf(mval);   // mfcc.cpp:239-243 / plp.cpp:434-440
          if (opKind == 1 && p.plpAud) {
            // auditory weighting + loudness compression (plp.cpp:488-510)
            if (p.doLog) {
              mval = __fmul_rn(__fadd_rn(mval, sEql[r - 1]), p.plpCompression);
            } else {
              if (mval < p.melfloor) mval = p.melfloor;
              mval = __fmul_rn(mval, sEql[r - 1]);
              mval = (float)pow((double)mval, (double)p.plpCompression);
            }
          }
          if (opKind == 1 && p.plpInvLog) mval = expf(mval);                    // plp.cpp:513-518
          melS[(r - 1) * F + f] = mval;
          cur = nxt;
        }
      }
    }
    __syncthreads();

    // ================= DCT-II + lifter (mfcc.cpp:251-272) / PLP back end (plp.cpp:520-590) =================
    const int ringBase = (j & 1) * F;   // tiles of a chunk alternate between the two ring halves
    if (opKind == 0) {
    // each virtual warp owns coefficients i, i+NVW, ... and evaluates them two at a time so
    // that one read of the log-mel column feeds two dot products; the cosine rows are read as
    // float4 (row stride padded to 4).  Each dot product keeps the reference's m = 0..nBands-1
    // accumulation order.
    for (int i = vw; i < p.nStat; i += 2 * NVW) {
      const int i1 = i + NVW;
      const bool two = i1 < p.nStat;
      const float4 *c0 = reinterpret_cast<const float4 *>(sDct + i * p.dctStride);
      const float4 *c1 = reinterpret_cast<const float4 *>(sDct + (two ? i1 : i) * p.dctStride);
      const float *lp = melS + f;
      float a0 = 0.f, a1 = 0.f;
      int m = 0;
#pragma unroll 2
      for (; m + 4 <= p.nBands; m += 4, lp += 4 * F) {
        const float4 w0 = *c0++, w1 = *c1++;
        const float l0 = lp[0], l1 = lp[F], l2 = lp[2 * F], l3 = lp[3 * F];
        a0 = __fmaf_rn(l0, w0.x, a0); a1 = __fmaf_rn(l0, w1.x, a1);
        a0 = __fmaf_rn(l1, w0.y, a0); a1 = __fmaf_rn(l1, w1.y, a1);
        a0 = __fmaf_rn(l2, w0.z, a0); a1 = __fmaf_rn(l2, w1.z, a1);
        a0 = __fmaf_rn(l3, w0.w, a0); a1 = __fmaf_rn(l3, w1.w, a1);
      }
      const float *r0 = reinterpret_cast<const float *>(c0), *r1 = reinterpret_cast<const float *>(c1);
      for (int k = 0; m < p.nBands; m++, k++, lp += F) {
        const float l0 = lp[0];
        a0 = __fmaf_rn(l0, r0[k], a0); a1 = __fmaf_rn(l0, r1[k], a1);
      }
      ring[i * (2 * F) + ringBase + f] = __fmul_rn(a0, sLift[i]);
      if (two) ring[i1 * (2 * F) + ringBase + f] = __fmul_rn(a1, sLift[i1]);
    }
    } else if (opKind == 1) {
      plp_backend<F, NVW>(p, melS, sDct, sLift, reinterpret_cast<float *>(smem + L.zbuf), ring + ringBase, vw, f);
    } else {
      tone_backend<F, NVW>(p, melS, ring + ringBase, vw, f);
    }
    __syncthreads();

    // ================= store =================
    if (!p.fused) {
      // static rows only (the temporal stages, if any, run in post_kernel)
      const int tot = nf * p.nStat;
      for (int idx = tid; idx < tot; idx += NT) {
        const int ff = idx / p.nStat, c = idx - ff * p.nStat;
        p.out[(cx.row0 + tg.fs + ff) * p.outStride + p.outCol + c] = ring[c * (2 * F) + ringBase + ff];
      }
    } else {
      // Fused delta / delta-delta (cDeltaRegression x2 + cVectorConcat): output row t needs the
      // statics of frames t-H..t+H.  After tile j all rows up to (tile end - H) are computable
      // (up to b on the chunk's last tile); their statics live in the two ring halves.
      const int K = p.nStat, W1 = p.fW1, W2 = p.fW2, H = W1 + W2;
      const int T = cx.T;
      const int r0 = emitted;
      const int r1 = (j + 1 == cx.nT) ? cx.b : min(tg.fs + F - H, cx.b);
      // tick-order model (see post_kernel): level 1 (delta) has T+W1 frames, c0_1 = max(T-W1,0) of
      // them before EOI; level 2 reads it with n0 = c0_1
      const int T1 = T + W1, c01 = max(T - W1, 0), c02 = max(c01 - W2, 0);
      const float norm1 = p.fNorm1, norm2 = p.fNorm2;
      // Both stages keep lane = frame (row): warps take the coefficients, so the ring / Dbuf
      // reads are unit-stride across lanes and the staging buffer outS, laid out exactly like the
      // global rows ([row][3K], row stride 3K = 39 floats = 7 mod 32 banks), is written without
      // bank conflicts and then copied to HBM as one contiguous, fully coalesced block.
      const int d0 = max(r0 - W2, 0), d1 = min(r1 + W2, T1);
      const int dRows = F + 24;             // row stride of Dbuf: >= (F + H) + 2 W2 rows, H <= 8
      float *outS = Dbuf + ((K * dRows + 3) & ~3);   // [(r1-r0)][3K], aliases Z like Dbuf; 16-byte aligned
      const int K3 = 3 * K;
      const int nr = r1 - r0;
      // ---- delta rows [r0-W2, r1+W2) /\ [0, T1) -> Dbuf[K][dRows] (+ outS), statics -> outS ----
      const bool interior1 = (d0 >= W1) && (d1 + W1 <= T);        // no clamping anywhere in this tile
      const bool interior2 = (r0 >= W2) && (r1 <= c02);           // all rows computed before EOI
      if (interior1 && interior2 && W1 == 2 && W2 == 2 && nr == F) {
        // ---- common case (deltawin = 2 twice, interior tile): straight-line code, work items
        // spread evenly over all threads
        emit_interior<F, NT>(ring, Dbuf, outS, K, dRows, d0 - cx.s0, r0 - cx.s0, norm1, p.fRcp1, norm2, p.fRcp2, tid);
      } else {
        emit_edge<F, NW>(ring, Dbuf, outS, K, W1, W2, T, T1, c01, c02, cx.s0, r0, r1, d0, d1, dRows, norm1, p.fRcp1, norm2, p.fRcp2, warp, lane);
      }
      // ---- rows [r0, r1) -> HBM, one contiguous block ----
      {
        float *o = p.out + (cx.row0 + r0) * (long long)K3;
        const int n = nr * K3;
        for (int i = tid; i < n; i += NT) o[i] = outS[i];
      }
      emitted = r1;
      // Dbuf aliases Z: the next tile's first FFT stage writes Z only after the barrier that
      // follows its staging phase, which every thread reaches after finishing this block.
    }

    }   // opKind >= 0

    // ---- advance to the next tile / chunk ----
    j++;
    if (j == cx.nT) {
      chunk++;
      j = 0;
      if (chunk < chunkEnd) { cx = load_chunk<F, CENTRED>(p, chunk); emitted = cx.a; }
    }
  }
}

// ------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------
// "lld_kernel<M,F,NT,MINB,VEC2|SCALAR,GEN|MFCC|CENTRED>" ("lld_kernel_f32<...>" for float input), built once per instance
template <int M, int F, int NT, int MINB, bool VEC2, bool GEN, bool F32, bool CENTRED>
static const char *lld_kernel_name()
{
  static const std::string name = std::string(F32 ? "lld_kernel_f32" : "lld_kernel") + "<" + std::to_string(M) + "," + std::to_string(F) + "," +
                                  std::to_string(NT) + "," + std::to_string(MINB) + (VEC2 ? ",VEC2" : ",SCALAR") +
                                  (CENTRED ? ",CENTRED>" : GEN ? ",GEN>" : ",MFCC>");
  return name.c_str();
}

template <int M, int F, int NT, int MINB, bool VEC2, bool GEN, bool F32, bool CENTRED = false>
static cudaError_t launch_g(const LldParams &p, int numSMs, cudaStream_t st, LldLaunchInfo *info, bool launch)
{
  const size_t smem = (size_t)make_layout(p, M, F).total;
  auto kern = lld_kernel<M, F, NT, MINB, VEC2, GEN, F32, CENTRED>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  int occ = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, NT, smem);
  if (e != cudaSuccess) return e;
  if (occ < 1) return cudaErrorLaunchOutOfResources;
  const int grid = launch ? p.nRuns : numSMs * occ;
  if (info) {
    info->grid = grid; info->block = NT; info->smem = smem; info->nChunks = p.nChunks;
    info->kernel = lld_kernel_name<M, F, NT, MINB, VEC2, GEN, F32, CENTRED>();
  }
  if (!launch) return cudaSuccess;
  kern<<<grid, NT, smem, st>>>(p);
  return cudaGetLastError();
}

template <int M, int F, int NT, int MINB, bool VEC2, bool F32>
static cudaError_t launch_t(const LldParams &p, int numSMs, cudaStream_t st, LldLaunchInfo *info, bool launch)
{
  if (p.frameCenter != 0) return launch_g<M, F, NT, MINB, VEC2, true, F32, true>(p, numSMs, st, info, launch);
  if (p.opKind == 0 && p.magOut == nullptr) return launch_g<M, F, NT, MINB, VEC2, false, F32>(p, numSMs, st, info, launch);
  return launch_g<M, F, NT, MINB, VEC2, true, F32>(p, numSMs, st, info, launch);
}

// the lld_kernel instance for the geometry of the pass (launch_lld: everything the 512-point fast instance does not take)
template <bool F32>
cudaError_t launch_lld_kernel(const LldParams &p, int nfft, int numSMs, cudaStream_t st, LldLaunchInfo *info, bool launch)
{
  // VEC2: 64-bit sample-pair loads need an even per-lane stride (frameStep + sPad)
  const bool vec2 = ((p.frameStep + p.sPad) % 2) == 0;
  // narrow tiles: half the frames per tile with half the threads (same number of virtual warps)
  if (p.narrow && nfft == 1024) return vec2 ? launch_t<512, 16, 256, 1, true, F32>(p, numSMs, st, info, launch) : launch_t<512, 16, 256, 1, false, F32>(p, numSMs, st, info, launch);
  if (p.narrow && nfft == 2048) return vec2 ? launch_t<1024, 8, 256, 1, true, F32>(p, numSMs, st, info, launch) : launch_t<1024, 8, 256, 1, false, F32>(p, numSMs, st, info, launch);
  if (p.narrow && nfft == 4096) return vec2 ? launch_t<2048, 4, 128, 1, true, F32>(p, numSMs, st, info, launch) : launch_t<2048, 4, 128, 1, false, F32>(p, numSMs, st, info, launch);
  switch (nfft) {
    case 512:  return vec2 ? launch_t<256, 32, 256, 2, true, F32>(p, numSMs, st, info, launch) : launch_t<256, 32, 256, 2, false, F32>(p, numSMs, st, info, launch);
    case 1024: return vec2 ? launch_t<512, 32, 512, 1, true, F32>(p, numSMs, st, info, launch) : launch_t<512, 32, 512, 1, false, F32>(p, numSMs, st, info, launch);
    case 2048: return vec2 ? launch_t<1024, 16, 512, 1, true, F32>(p, numSMs, st, info, launch) : launch_t<1024, 16, 512, 1, false, F32>(p, numSMs, st, info, launch);
    case 4096: return vec2 ? launch_t<2048, 8, 256, 1, true, F32>(p, numSMs, st, info, launch) : launch_t<2048, 8, 256, 1, false, F32>(p, numSMs, st, info, launch);
    default:   return cudaErrorInvalidValue;
  }
}

// compiled in two translation units that build in parallel: kernels.cu (int16 input) and lld_kernel_f32.cu (float input)
extern template cudaError_t launch_lld_kernel<false>(const LldParams &, int, int, cudaStream_t, LldLaunchInfo *, bool);
extern template cudaError_t launch_lld_kernel<true>(const LldParams &, int, int, cudaStream_t, LldLaunchInfo *, bool);

}  // namespace osm
