// kernels.cu -- fused per-frame LLD kernels for sm_90a.
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
#include <cstdio>
#include <cstdlib>
#include <string>

#include "fft_radix.cuh"
#include "kernels.cuh"

#include "lld_common.cuh"

namespace osm {

constexpr int kUnrollMel = OSM_UNROLL_MEL, kUnrollDct = OSM_UNROLL_DCT;

// ------------------------------------------------------------------------------------------
// the fused kernel
// ------------------------------------------------------------------------------------------
// GEN = false: the MFCC-only instance (band op = cMfcc, no magnitude level dump); the PLP back end and
// the magnitude dump compile away.  GEN = true: band op and dump selected at run time.
template <int M, int F, int NT, int MINB, bool VEC2, bool GEN>
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
  ChunkCtx cx = load_chunk<F>(p, chunk);
  int j = 0;
  int emitted = cx.a;                 // next output row of the current chunk to be written
  if (tid == 0) {
    const TileGeom g0 = tile_geom<F>(p, cx, 0);
    mbar_expect_tx(mbar, g0.bytes);
    bulk_g2s(rawPcm, g0.src, g0.bytes, mbar);
  }

  while (chunk < chunkEnd) {
    const TileGeom tg = tile_geom<F>(p, cx, j);
    const int nf = tg.nf, count = tg.count;

    // ================= stage: PCM (smem, prefetched by the bulk copy) -> float -> pre-emphasis -> smem =================
    mbar_wait(mbar, phase);
    phase ^= 1;
    {
      const int16_t *rp = reinterpret_cast<const int16_t *>(rawPcm + tg.mis) + tg.lead * nChan;   // sample frame 0 of the tile
      const bool fastLoad = (tg.mis == 0) && (nChan <= 2) && !(OSM_PCM_F32_SUPPORT && p.pcmF32);
      const bool fastStore = (p.sPad == 0) || (hop % 8 == 0);
      for (int c = tid; c * 8 < count; c += NT) {
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
          for (int jj = 0; jj < 8; jj++) x[jj] = (jj < nvalid) ? pcm_to_float_slow(rp + (i + jj) * nChan, nChan, p.pcmF32) : 0.f;
        }
        float y[8];
        if (p.preemph) {
          // vectorPreemphasis.cpp:96-104 : x[n] -/+ k * x[n-1], two roundings
          float xprev = 0.f;
          if (i > 0 || tg.lead > 0) {
            if (nChan == 1) xprev = div32767((float)rp[i - 1]);
            else xprev = pcm_to_float_slow(rp + (i - 1) * nChan, nChan, p.pcmF32);
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
        const TileGeom gn = tile_geom<F>(p, cx, j + 1);
        mbar_expect_tx(mbar, gn.bytes);
        bulk_g2s(rawPcm, gn.src, gn.bytes, mbar);
      } else if (chunk + 1 < chunkEnd) {
        const ChunkCtx cn = load_chunk<F>(p, chunk + 1);
        const TileGeom gn = tile_geom<F>(p, cn, 0);
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
#if OSM_MEL_COMPACT
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
#else
        int n = sMelRange[bs];
        const float *pp = P + n * F + f;
        const float2 *cp = sMelCoef + sVB[bs];
        {
          const int n1 = sMelRange[bs + 1];
#pragma unroll kUnrollMel
          for (; n < n1; n++, pp += F, cp++) cur = __fmaf_rn(*pp, cp->y, cur);
        }
        for (int r = bs + 1; r <= be; r++) {
          float nxt = 0.f;
          const int n1 = sMelRange[r + 1];
          cp = sMelCoef + sVB[r];
#pragma unroll kUnrollMel
          for (; n < n1; n++, pp += F, cp++) {
            const float pw = *pp;
            const float2 w = *cp;
            cur = __fmaf_rn(pw, w.x, cur);
            nxt = __fmaf_rn(pw, w.y, nxt);
          }
#endif
          float mval = __fmul_rn(cur, p.melScale);
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
#pragma unroll kUnrollDct
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
    } else {
      plp_backend<F, NVW>(p, melS, sDct, sLift, reinterpret_cast<float *>(smem + L.zbuf), ring + ringBase, vw, f);
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
        emit_interior<F, NT, 0>(ring, Dbuf, outS, K, dRows, d0 - cx.s0, r0 - cx.s0, norm1, p.fRcp1, norm2, p.fRcp2, tid);
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
      if (chunk < chunkEnd) { cx = load_chunk<F>(p, chunk); emitted = cx.a; }
    }
  }
}

// ------------------------------------------------------------------------------------------
// temporal post-processing
// ------------------------------------------------------------------------------------------
// Tick-order model of chained window processors (cWindowProcessor with blocksize=1, components
// ticking in data-flow order; core/windowProcessor.cpp:85-119,167-230, core/componentManager.cpp:
// 1233-1262).  For the level produced by stage s:  final_s = final_{s-1} + W_s frames in total,
// c0_s = max(c0_{s-1} - W_s, 0) of them produced before EOI is raised (c0_0 = final_0 = T).
// When the consumer computes frame t >= c0_s its input level holds
//     navail = min(c0_{s-1} + (t - c0_s) + 1, final_{s-1})
// frames.  Matrix reads (core/dataMemoryLevel.cpp:1651-1738): window start >= 0: rows >= navail
// replicate row navail-1; window start < 0: rows < 0 replicate row 0 and rows >= navail come
// from the zero-initialised, not yet written level buffer (0.0).  For c0_{s-1} >= W_s this is the
// plain "clamp to [0, final-1]" rule; the rest only triggers for utterances shorter than the
// summed window lengths and is reproduced because the reference does it.
//
// post_kernel: one CTA per tile of kPostRows output rows of one utterance.  The static rows the
// tile depends on (halo = summed half windows) are staged in shared memory once, every stage of
// every group is then evaluated level by level in shared memory (O(window) per element) and
// the finished rows are written out.
constexpr int kPostRows = 64;      // at most; see post_tile_rows()
constexpr int kPostMaxHalo = 12;
constexpr int kPostThreads = 256;

__device__ __forceinline__ float post_read(const float *lvl, int n, int rowBase, int t, int W, int navail, int i, int c)
{
  // lvl: smem rows of the input level, row index (absolute frame - rowBase), n columns
  if (t - W < 0) {
    if (i < 0) i = 0;
    else if (i >= navail) return 0.f;
  } else if (i > navail - 1) {
    i = navail - 1;
  }
  return lvl[(i - rowBase) * n + c];
}

__global__ void __launch_bounds__(kPostThreads) post_kernel(const PostParams p)
{
  extern __shared__ float psm[];
  const TileRef tr = p.tiles[blockIdx.x];
  const int u = tr.utt, r0 = tr.f0;
  const long long Ls = p.uttOff[u + 1] - p.uttOff[u];
  const int Tout = (int)(p.rowOff[u + 1] - p.rowOff[u]);
  const int r1 = min(r0 + p.rows, Tout);
  const int H = p.halo;
  const int rowBase = r0 - H;                       // absolute frame of smem row 0 (may be < 0)
  const int nRowsBuf = p.rows + 2 * H;
  float *S0 = psm;                                  // [nRowsBuf][nStat]
  float *A = S0 + nRowsBuf * p.nStat;               // [nRowsBuf][maxN]
  float *B = A + nRowsBuf * p.maxN;
  const int tid = threadIdx.x;

  // ---- static rows [r0-H, r1+H) /\ [0, Tmax) -> smem (Tmax = rows of the static buffer) ----
  {
    const int Tmax = (int)(p.statOff[u + 1] - p.statOff[u]);
    const int lo = max(rowBase, 0), hi = min(r1 + H, Tmax);
    const float *src = p.stat + p.statOff[u] * (long long)p.statStride;
    const int tot = (hi - lo) * p.nStat;
    for (int idx = tid; idx < tot; idx += kPostThreads) {
      const int rr = idx / p.nStat, c = idx - rr * p.nStat;
      S0[(lo + rr - rowBase) * p.nStat + c] = src[(long long)(lo + rr) * p.statStride + c];
    }
  }
  __syncthreads();

  for (int gi = 0; gi < p.nGroups; gi++) {
    const PostGroup &g = p.groups[gi];
    const int n = g.n;
    const int T = (Ls >= g.frameSize) ? (int)((Ls - g.frameSize) / g.frameStep + 1) : 0;   // frames of this group's source level
    // a multi-level reader delivers min over its levels: that bounds how many frames the first stage
    // produces (before EOI and in total), while reads of THIS level still clamp at its own end
    int Tlim = T;
    for (int k = 0; k < g.nLim; k++) Tlim = min(Tlim, (Ls >= g.limSize[k]) ? (int)((Ls - g.limSize[k]) / g.limStep[k] + 1) : 0);
    // level 0 view of this group: copy its columns so that every level has row stride n
    const float *cur;
    {
      const int lo = max(rowBase, 0), hi = min(r1 + H, T);
      const int tot = (hi - lo) * n;
      for (int idx = tid; idx < tot; idx += kPostThreads) {
        const int rr = idx / n, c = idx - rr * n;
        A[(lo + rr - rowBase) * n + c] = S0[(lo + rr - rowBase) * p.nStat + g.srcCol + c];
      }
      cur = A;
    }
    __syncthreads();
    int Tprev = T, n0 = T;                          // input level: total frames, frames before EOI
    int Tcnt = Tlim, n0cnt = Tlim;                  // the same as seen through the reader (min over its levels)
    int Hrem = 0;
    for (int s = 0; s < g.nStages; s++) Hrem += g.win[s];
    for (int s = 0; s < g.nStages; s++) {
      const int W = g.win[s];
      Hrem -= W;
      const int c0 = max(n0cnt - W, 0);
      const int Tcur = Tcnt + W;
      float *dst = (cur == A) ? B : A;
      const int lo = max(r0 - Hrem, 0), hi = min(r1 + Hrem, Tcur);   // rows of this level needed
      const int tot = (hi - lo) * n;
      float norm = 0.f;
      for (int i = 1; i <= W; i++) norm = __fadd_rn(norm, __fmul_rn((float)i, (float)i));
      norm = __fmul_rn(norm, 2.0f);                 // deltaRegression.cpp:77-80
      for (int idx = tid; idx < tot; idx += kPostThreads) {
        const int rr = idx / n, c = idx - rr * n;
        const int t = lo + rr;
        const int navail = (t < c0) ? Tprev : min(n0 + (t - c0) + 1, Tprev);
        float y;
        if (g.kind[s] == 2) {
          // fullinputMean.cpp:516-522 : vec->data[i] -= means[i]
          y = __fsub_rn(post_read(cur, n, rowBase, t, 0, navail, t, c), p.means[(long long)u * p.nStat + g.srcCol + c]);
        } else if (g.kind[s] == 0) {
          // deltaRegression.cpp:139-146 : num = sum_i i*(x[t+i]-x[t-i]) ; y = num / norm
          float num = 0.f;
          const int fl = g.flags[s];                 // bit 1 relativeDelta, bit 2 absOutput, bit 3 halfWaveRect (:100-108,157-165)
          for (int i = 1; i <= W; i++) {
            const float later = post_read(cur, n, rowBase, t, W, navail, t + i, c);
            const float prior = post_read(cur, n, rowBase, t, W, navail, t - i, c);
            float delta = __fsub_rn(later, prior);
            if (fl & 2) delta = prior != 0.0f ? __fdiv_rn(delta, fabsf(prior)) : 0.0f;
            num = __fadd_rn(num, __fmul_rn((float)i, delta));
          }
          y = __fdiv_rn(num, norm);
          if (fl & 8) { if (y < 0.0f) y = 0.0f; }
          else if (fl & 4) { if (y < 0.0f) y = -y; }
        } else {
          // contourSmoother.cpp:84-117 : y = x[n]; y += x[n-w]; y += x[n+w]; y /= smaWin
          const int noZero = g.flags[s];
          const float x0 = post_read(cur, n, rowBase, t, W, navail, t, c);
          if (noZero && x0 == 0.f) {
            y = 0.f;
          } else {
            y = x0;
            int cnt = 1;
            for (int w = 1; w <= W; w++) {
              const float a = post_read(cur, n, rowBase, t, W, navail, t - w, c);
              const float b = post_read(cur, n, rowBase, t, W, navail, t + w, c);
              if (!noZero || a != 0.f) { y = __fadd_rn(y, a); cnt++; }
              if (!noZero || b != 0.f) { y = __fadd_rn(y, b); cnt++; }
            }
            y = __fdiv_rn(y, noZero ? (float)cnt : (float)(2 * W + 1));
          }
        }
        dst[(t - rowBase) * n + c] = y;
      }
      __syncthreads();
      cur = dst;
      n0 = c0; n0cnt = c0;
      Tprev = Tcur; Tcnt = Tcur;
    }
    // ---- write rows [r0, r1) of this group ----
    {
      float *o = p.out + (p.rowOff[u] + r0) * (long long)p.outStride + g.outCol;
      const int tot = (r1 - r0) * n;
      for (int idx = tid; idx < tot; idx += kPostThreads) {
        const int rr = idx / n, c = idx - rr * n;
        o[(long long)rr * p.outStride + c] = cur[(r0 + rr - rowBase) * n + c];
      }
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------
// cAcf (ACF + cepstrum) + cPitchACF, per-frame part.
//   dspcore/acf.cpp:250-345: both levels are the inverse real FFT of a real, even spectrum
//   (power resp. log(1+x)), i.e. cosine transforms.  With z[n] = Pfull[n] + i*Cfull[n] over the
//   symmetric extension n = 0..N-1, ONE complex FFT of size N gives both at once:
//   Re Z[j] = 2*acf_ooura[j], Im Z[j] = 2*cep_ooura[j]  (real even input -> real even output).
//   lldcore/pitchACF.cpp:137-361 then scans the two arrays per frame.
// One CTA per tile, lane = frame, same batched in-place FFT as lld_kernel.
// ------------------------------------------------------------------------------------------
template <int N, int F, int NT>
__global__ void __launch_bounds__(NT, 1) acf_pitch_kernel(const AcfPitchParams p)
{
  constexpr int NW = NT / 32, G = 32 / F, NVW = NW * G;
  using Fc = Fact<N>;
  extern __shared__ __align__(16) unsigned char smem[];
  float2 *Z = reinterpret_cast<float2 *>(smem);
  float2 *sTw = reinterpret_cast<float2 *>(smem + (size_t)N * F * 8);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int f = lane & (F - 1);
  const int vw = warp * G + lane / F;
  // the magnitude level is stored in tiles of p.F frames; this CTA handles F of them (sub-tile)
  const int SUB = p.F / F;
  const int tileIdx = blockIdx.x / SUB, sub = blockIdx.x - tileIdx * SUB;
  OpTile tl = p.tiles[tileIdx];
  tl.f0 += sub * F;
  tl.nf = min(max(tl.nf - sub * F, 0), F);
  const int nSrc = p.nSrc;
  for (int i = tid; i < p.twCount; i += NT) sTw[i] = p.twiddles[i];
  // ---- spectrum -> symmetric complex input ----
  {
    const float *mg = p.mag + (size_t)tileIdx * nSrc * p.F + sub * F;
    for (int idx = tid; idx < nSrc * F; idx += NT) {
      const int k = idx / F, ff = idx - k * F;
      const float m = mg[(size_t)k * p.F + ff];
      const float pw = p.acfUsePower ? __fmul_rn(m, m) : m;                       // acf.cpp:253-261
      const float cs = p.cepUsePower ? __fmul_rn(m, m) : m;
      float cv;
      if (p.oldCompatCepstrum) cv = (k == 0 || k == nSrc - 1) ? cs : ((cs > 0.0f) ? logf(cs) : 0.0f);   // acf.cpp:276-286 (float log)
      else cv = (cs > 0.0f) ? (float)log((double)cs + 1.0) : 0.0f;                 // acf.cpp:289-305
      const float2 v = make_float2(pw, cv);
      Z[k * F + ff] = v;
      if (k > 0 && k < N / 2) Z[(N - k) * F + ff] = v;
    }
  }
  __syncthreads();
  // oldCompatCepstrum: the two transforms share one complex FFT, whose rounding is relative to the larger channel, and log(x) of
  // the tiny powers of a quiet frame (|log x| ~ 20) would swamp its ACF channel (x ~ 1e-9).  The cepstrum channel of each frame is
  // weighted by the power of two that brings both channels to the same magnitude (exact) and the weight is undone on output.
  __shared__ float sCepUnscale[32];
  if (p.oldCompatCepstrum) {
    for (int ff = tid; ff < F; ff += NT) {
      float mp = 0.0f, mc = 0.0f;
      for (int k = 0; k <= N / 2; k++) { const float2 v = Z[k * F + ff]; mp = fmaxf(mp, fabsf(v.x)); mc = fmaxf(mc, fabsf(v.y)); }
      const int e = (mp > 0.0f && mc > 0.0f) ? max(min(ilogbf(mp) - ilogbf(mc), 100), -100) : 0;
      sCepUnscale[ff] = ldexpf(1.0f, -e);
      const float w = ldexpf(1.0f, e);
      for (int k = 0; k < N; k++) Z[k * F + ff].y *= w;
    }
    __syncthreads();
  }
  {
    LldParams dummy;     // fft_stage only reads it in its FIRST (sample loading) specialisation
    fft_stage<N, F, NVW, Fc::R0, N, false, false, false>(Z, nullptr, nullptr, nullptr, sTw + p.twOff[0], dummy, vw, f);
    __syncthreads();
    fft_stage<N, F, NVW, Fc::R1, N / Fc::R0, false, false, false>(Z, nullptr, nullptr, nullptr, sTw + p.twOff[1], dummy, vw, f);
    __syncthreads();
    fft_stage<N, F, NVW, Fc::R2, N / (Fc::R0 * Fc::R1), false, true, false>(Z, nullptr, nullptr, nullptr, nullptr, dummy, vw, f);
  }
  __syncthreads();
  // ---- per-frame analysis (lldcore/pitchACF.cpp:137-183) ----
  // lane = frame as everywhere; the lag range [0, n) is cut into NVW slices, one per virtual warp.
  // Counts, maxima and the first-peak index combine exactly; the two double sums (mean of the ACF,
  // mean |cepstrum|) are added slice by slice instead of lag by lag (differences at the 1e-16 level).
  const int n = N / 2;                                     // length of each cAcf level (Ndst = Nsrc - 1)
  const float fNsrc = (float)nSrc;
  auto acf = [&](int j) {
    float d = 0.5f * Z[fft_pos<N>(j) * F + f].x;
    if (p.normOutput) d = __fdiv_rn(d, fNsrc);             // acf.cpp:321-325
    return fabsf(d);                                       // :342-344
  };
  auto cep = [&](int j) {
    float d = 0.5f * Z[fft_pos<N>(j) * F + f].y;
    if (p.oldCompatCepstrum) d *= sCepUnscale[f];
    if (p.normOutput) d = __fdiv_rn(d, fNsrc);
    return p.absCepstrum ? fabsf(d) : d;                   // :327-341
  };
  // per-slice partial results, [NVW][F] each, behind the twiddles
  double *sD = reinterpret_cast<double *>(smem + (((size_t)N * F * 8 + (size_t)p.twCount * 8 + 15) & ~(size_t)15));
  double *sMx = sD, *sMean = sD + NVW * F, *sCmax = sD + 2 * NVW * F, *sCsum = sD + 3 * NVW * F;
  int *sI = reinterpret_cast<int *>(sD + 4 * NVW * F);
  int *sZcr = sI, *sMcr = sI + NVW * F, *sIdx = sI + 2 * NVW * F;
  const double Nd = (double)(2 * n);
  const double Tsamp = (double)p.fsSec / Nd;
  const int preskip = (p.maxPitch <= 0.0) ? 0 : (int)(1.0 / (p.maxPitch * Tsamp));
  const int skip = preskip + 1;
  const int j0 = (int)(((long long)n * vw) / NVW), j1 = (int)(((long long)n * (vw + 1)) / NVW);
  {
    // voicingProb pass (:249-284): sign changes, rising maximum, sum; cepstrum maximum and |.| sum (:286-297)
    int zcr = 0;
    double mx = -1.0, mean = 0.0;                          // ACF values are >= 0
    const int i0 = max(j0, 1);
    float a0 = acf(i0 - 1);
    for (int i = i0; i < j1; i++) {
      const float a1 = acf(i);
      if (__fmul_rn(a0, a1) < 0.0f) zcr++;
      if (i >= preskip) {
        if (((double)a1 > mx) && (a0 < a1)) mx = a1;
        mean += (double)a1;
      }
      a0 = a1;
    }
    double cmax = -1e300, csum = 0.0;
    for (int i = j1 - 1; i >= j0; i--) {
      const double buf = cep(i);
      csum += fabs(buf);
      if (i >= skip && buf > cmax) cmax = buf;
    }
    sZcr[vw * F + f] = zcr; sMx[vw * F + f] = mx; sMean[vw * F + f] = mean;
    sCmax[vw * F + f] = cmax; sCsum[vw * F + f] = csum;
  }
  __syncthreads();
  double mean = acf(preskip), mx = acf(n - 1), cmax = cep(n - 1), csum = 0.0;
  int zcr = 0;
  for (int w = 0; w < NVW; w++) {
    zcr += sZcr[w * F + f];
    mean += sMean[w * F + f];
    if (sMx[w * F + f] > mx) mx = sMx[w * F + f];
    if (sCmax[w * F + f] > cmax) cmax = sCmax[w * F + f];
  }
  for (int w = NVW - 1; w >= 0; w--) csum += sCsum[w * F + f];     // the reference walks the lags downwards
  mean /= (double)(n - preskip + 1);
  csum /= (double)n;
  {
    // mean crossings (:266-273) and the first cepstral peak above the threshold (:299-310)
    int mcr = 0;
    const int i0 = max(j0, 1);
    float a0 = acf(i0 - 1);
    for (int i = i0; i < j1; i++) {
      const float a1 = acf(i);
      if (((double)a0 - mean) * ((double)a1 - mean) < 0.0) mcr++;
      a0 = a1;
    }
    int first = 0x7fffffff;
    const double thr = (cmax + csum) * 0.6;
    const int lo = max(j0, skip + 1), hi = min(j1, n - 1);
    if (lo < hi) {
      float cm = cep(lo - 1), c0 = cep(lo);
      for (int i = lo; i < hi; i++) {
        const float c1 = cep(i + 1);
        if ((double)c0 > thr && (cm < c0) && (c0 > c1)) { first = i; break; }
        cm = c0; c0 = c1;
      }
    }
    sMcr[vw * F + f] = mcr; sIdx[vw * F + f] = first;
  }
  __syncthreads();
  if (vw == 0 && f < tl.nf) {
    int mcr = 0, maxIdx = 0x7fffffff;
    for (int w = 0; w < NVW; w++) { mcr += sMcr[w * F + f]; maxIdx = min(maxIdx, sIdx[w * F + f]); }
    if (maxIdx == 0x7fffffff) maxIdx = 0;
    const double acfZcr = (mcr > zcr) ? (double)mcr / (double)n : (double)zcr / (double)n;
    const float acf0 = acf(0);
    const double voicing = (acf0 > 0.0f) ? mx / (double)acf0 : 0.0;
    PitchRaw r;
    r.voicing = voicing; r.acfZcr = acfZcr; r.maxIdx = maxIdx;
    const float aI = acf(maxIdx);
    r.hnr = 0.f; r.hnrDB = 0.f; r.hnrLin = 0.f;
    if (p.HNR) {                                           // :312-326
      const float dd = __fsub_rn(acf0, aI);
      const double buf = (dd == 0.0f) ? 100000000000000000000.0 : (double)__fdiv_rn(aI, dd);
      r.hnr = (float)((buf > 0.00000000001) ? 10.0 * log(buf) : 10.0 * log(0.00000000001));
    }
    if (p.HNRdB) {                                         // :329-343
      double buf = (double)__fsub_rn(acf0, aI);
      buf = (buf == 0.0) ? 10e10 : (double)aI / buf;
      r.hnrDB = (float)((buf <= 10e-10) ? -100.0 : ((buf >= 10e10) ? +100.0 : 10.0 * log(buf) / log(10.0)));
    }
    if (p.linHNR) {                                        // :346-360
      double buf = (double)__fsub_rn(acf0, aI);
      buf = (buf == 0.0) ? 10e3 : (double)aI / buf;
      r.hnrLin = (float)((buf <= 10e-3) ? 10e-3 : ((buf >= 10e3) ? 10e3 : buf));
    }
    p.raw[p.statOff[tl.utt] + tl.f0 + f] = r;
  }
}

// per-utterance pitch contour smoothing state machine (lldcore/pitchACF.cpp:184-245): sequential in
// time, one thread per utterance
__global__ void pitch_smooth_kernel(const AcfPitchParams p, int u0, int u1)
{
  const int u = u0 + blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= u1) return;
  const long long Ls = p.uttOff[u + 1] - p.uttOff[u];
  const int T = (Ls >= p.frameSize) ? (int)((Ls - p.frameSize) / p.frameStep + 1) : 0;
  const int n = p.nfft / 2;
  const double Tsamp = (double)p.fsSec / (double)(2 * n);
  float lastPitch = 0.f, lastlastPitch = 0.f, glMeanPitch = 0.f, pitchEnv = 0.f;
  int onsFlag = 0;
  const double maxPitch = p.maxPitch;
  for (int t = 0; t < T; t++) {
    const PitchRaw r = p.raw[p.statOff[u] + t];
    float *dst = p.stat + (p.statOff[u] + t) * (long long)p.statStride + p.outCol;
    int k = 0;
    if (p.voiceProb) dst[k++] = (float)r.voicing;
    if (p.HNR) dst[k++] = r.hnr;
    if (p.HNRdB) dst[k++] = r.hnrDB;
    if (p.linHNR) dst[k++] = r.hnrLin;
    if (p.F0 || p.F0env || p.voiceQual || p.F0raw) {
      int maxIdx = r.maxIdx;
      const float invT = __fdiv_rn(1.0f, __fmul_rn((float)maxIdx, (float)Tsamp));
      float vq = __fmul_rn(__fsub_rn((float)maxPitch, (float)fabs((r.acfZcr * maxPitch) - (double)invT)), (float)r.voicing);
      if (maxIdx == 0) vq = 0.0f;
      if (p.voiceQual) dst[k++] = vq;
      float pitch = 0.0f, rawF0 = 0.0f;
      if (maxIdx > 0) { pitch = invT; rawF0 = pitch; }
      if (r.voicing < p.voicingCutoff) { maxIdx = 0; pitch = 0.0f; }
      if ((lastPitch == 0.0f) && (pitch > 0.0f)) onsFlag = 1;
      if ((lastPitch > 0.0f) && (pitch == 0.0f) && (onsFlag == 0)) onsFlag = -1;
      if ((lastPitch > 0.0f) && (pitch > 0.0f)) onsFlag = 0;
      if ((lastPitch == 0.0f) && (pitch == 0.0f)) onsFlag = 0;
      if ((pitch == 0.0f) && (onsFlag == 1)) lastPitch = 0.0f;
      const float oPitch = pitch;
      const float tol = 0.4f;
      float alpha = 0.3f;
      if (pitch > 0.0f) {
        if (glMeanPitch == 0.0f) glMeanPitch = pitch;
        if (!((pitch < __fmul_rn(__fadd_rn(1.0f, tol), glMeanPitch)) && (pitch > __fmul_rn(__fsub_rn(1.0f, tol), glMeanPitch)))) {
          pitch = glMeanPitch;
          alpha = __fdiv_rn(alpha, 3.0f);
        }
        if (onsFlag && (lastPitch > pitch)) lastPitch = __fmul_rn(lastPitch, 0.85f);
      }
      if ((pitch > 0.0f) && (onsFlag == -1)) lastPitch = pitch;
      if (oPitch > 0.0f) glMeanPitch = __fadd_rn(__fmul_rn(__fsub_rn(1.0f, alpha), glMeanPitch), __fmul_rn(alpha, oPitch));
      float out;
      if ((lastlastPitch != 0.0f) && (lastPitch != 0.0f)) out = __fmul_rn(0.5f, __fadd_rn(lastlastPitch, lastPitch));
      else out = lastPitch;
      if (p.F0) dst[k++] = out;
      if (p.F0raw) dst[k++] = rawF0;
      lastlastPitch = lastPitch;
      lastPitch = pitch;
      if (p.F0env) {
        if (out > 0.0f) pitchEnv = __fadd_rn(__fmul_rn(0.75f, pitchEnv), __fmul_rn(0.25f, out));
        dst[k++] = pitchEnv;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------
int lld_tile_frames(int nfft, bool narrow)
{
  const int F = nfft == 4096 ? 8 : (nfft == 2048 ? 16 : 32);
  return (narrow && nfft >= 1024) ? F / 2 : F;
}
int lld_virtual_warps(int nfft) { return nfft == 512 ? 8 : (nfft == 1024 ? 16 : 32); }
int lld_max_chunk_tiles() { return 16; }
bool lld_supported_fft(int nfft) { return nfft == 512 || nfft == 1024 || nfft == 2048 || nfft == 4096; }

size_t lld_smem_bytes(const LldParams &p, int nfft)
{
  return (size_t)make_layout(p, nfft / 2, lld_tile_frames(nfft, p.narrow != 0)).total;
}

#define OSM_STR2(x) #x
#define OSM_STR(x) OSM_STR2(x)
// "lld_kernel<M,F,NT,MINB,VEC2|SCALAR,GEN|MFCC>" (lld_kernel_f32 in the float-input build), built once per instance
template <int M, int F, int NT, int MINB, bool VEC2, bool GEN>
static const char *lld_kernel_name()
{
  static const std::string name = std::string(OSM_STR(lld_kernel)) + "<" + std::to_string(M) + "," + std::to_string(F) + "," +
                                  std::to_string(NT) + "," + std::to_string(MINB) + (VEC2 ? ",VEC2" : ",SCALAR") +
                                  (GEN ? ",GEN>" : ",MFCC>");
  return name.c_str();
}

template <int M, int F, int NT, int MINB, bool VEC2, bool GEN>
static cudaError_t launch_g(const LldParams &p, int numSMs, cudaStream_t st, LldLaunchInfo *info, bool launch)
{
  const size_t smem = (size_t)make_layout(p, M, F).total;
  auto kern = lld_kernel<M, F, NT, MINB, VEC2, GEN>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  int occ = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, NT, smem);
  if (e != cudaSuccess) return e;
  if (occ < 1) return cudaErrorLaunchOutOfResources;
  const int grid = launch ? p.nRuns : numSMs * occ;
  if (info) {
    info->grid = grid; info->block = NT; info->smem = smem; info->nChunks = p.nChunks;
    info->kernel = lld_kernel_name<M, F, NT, MINB, VEC2, GEN>();
  }
  if (!launch) return cudaSuccess;
  kern<<<grid, NT, smem, st>>>(p);
  return cudaGetLastError();
}

template <int M, int F, int NT, int MINB, bool VEC2>
static cudaError_t launch_t(const LldParams &p, int numSMs, cudaStream_t st, LldLaunchInfo *info, bool launch)
{
  if (p.opKind == 0 && p.magOut == nullptr) return launch_g<M, F, NT, MINB, VEC2, false>(p, numSMs, st, info, launch);
  return launch_g<M, F, NT, MINB, VEC2, true>(p, numSMs, st, info, launch);
}

cudaError_t launch_lld(const LldParams &p, int nfft, int numSMs, cudaStream_t st, LldLaunchInfo *info, bool launch)
{
  {
    static const bool fastOn = [] { const char *e = getenv("OSM_B200_LLD_FAST"); return !(e && e[0] == '0'); }();
    if (fastOn && lld_fast_applies(p, nfft)) return launch_lld_fast(p, numSMs, st, info, launch);
  }
  // VEC2: 64-bit sample-pair loads need an even per-lane stride (frameStep + sPad)
  const bool vec2 = ((p.frameStep + p.sPad) % 2) == 0;
  // narrow tiles: half the frames per tile with half the threads (same number of virtual warps)
  if (p.narrow && nfft == 1024) return vec2 ? launch_t<512, 16, 256, 1, true>(p, numSMs, st, info, launch) : launch_t<512, 16, 256, 1, false>(p, numSMs, st, info, launch);
  if (p.narrow && nfft == 2048) return vec2 ? launch_t<1024, 8, 256, 1, true>(p, numSMs, st, info, launch) : launch_t<1024, 8, 256, 1, false>(p, numSMs, st, info, launch);
  if (p.narrow && nfft == 4096) return vec2 ? launch_t<2048, 4, 128, 1, true>(p, numSMs, st, info, launch) : launch_t<2048, 4, 128, 1, false>(p, numSMs, st, info, launch);
  switch (nfft) {
    case 512:  return vec2 ? launch_t<256, 32, 256, 2, true>(p, numSMs, st, info, launch) : launch_t<256, 32, 256, 2, false>(p, numSMs, st, info, launch);
    case 1024: return vec2 ? launch_t<512, 32, 512, 1, true>(p, numSMs, st, info, launch) : launch_t<512, 32, 512, 1, false>(p, numSMs, st, info, launch);
    case 2048: return vec2 ? launch_t<1024, 16, 512, 1, true>(p, numSMs, st, info, launch) : launch_t<1024, 16, 512, 1, false>(p, numSMs, st, info, launch);
    case 4096: return vec2 ? launch_t<2048, 8, 256, 1, true>(p, numSMs, st, info, launch) : launch_t<2048, 8, 256, 1, false>(p, numSMs, st, info, launch);
    default:   return cudaErrorInvalidValue;
  }
}

int post_tile_rows(int nStat, int maxN, int halo)
{
  int rows = kPostRows;
  while (rows > 4 && (size_t)(rows + 2 * halo) * (nStat + 2 * maxN) * sizeof(float) > 160 * 1024) rows /= 2;
  return rows;
}

cudaError_t launch_post(const PostParams &p, cudaStream_t st)
{
  if (p.nTiles <= 0 || p.nGroups <= 0) return cudaSuccess;
  if (p.halo > kPostMaxHalo) return cudaErrorInvalidValue;
  const size_t smem = (size_t)(p.rows + 2 * p.halo) * (p.nStat + 2 * p.maxN) * sizeof(float);
  cudaError_t e = cudaFuncSetAttribute(post_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  post_kernel<<<p.nTiles, kPostThreads, smem, st>>>(p);
  return cudaGetLastError();
}

bool acf_pitch_supported_fft(int nfft) { return nfft == 512 || nfft == 1024 || nfft == 2048; }

template <int N, int F, int NT>
static cudaError_t launch_acf_t(const AcfPitchParams &p, cudaStream_t st)
{
  constexpr int NVW = (NT / 32) * (32 / F);
  // FFT tile | twiddles | per-slice partials of the analysis (4 doubles + 3 ints per slice and frame)
  const size_t smem = (((size_t)N * F * 8 + (size_t)p.twCount * 8 + 15) & ~(size_t)15) + (size_t)NVW * F * (4 * 8 + 3 * 4) + 16;
  auto kern = acf_pitch_kernel<N, F, NT>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  kern<<<p.nTiles * (p.F / F), NT, smem, st>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_acf_pitch(const AcfPitchParams &p, cudaStream_t st)
{
  if (p.nTiles <= 0) return cudaSuccess;
  switch (p.nfft) {
    case 512:  return launch_acf_t<512, 32, 512>(p, st);
    case 1024: return launch_acf_t<1024, 16, 512>(p, st);
    case 2048: return launch_acf_t<2048, 8, 256>(p, st);
    default:   return cudaErrorInvalidValue;
  }
}

// ------------------------------------------------------------------------------------------
// cPlp RASTA filter (lldcore/plp.cpp:446-483): a 5-tap FIR + one-pole IIR along time on every band,
// state reset per utterance; the first 5 outputs are forced to 0.  Sequential in time by
// construction -> one thread per (utterance, band); float operations in the reference's order.
// ------------------------------------------------------------------------------------------
__global__ void rasta_kernel(const RastaParams p, int u0, int u1)
{
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int nB = p.nBands;
  const int u = u0 + (int)(idx / nB), b = (int)(idx % nB);
  if (u >= u1) return;
  const long long L = p.uttOff[u + 1] - p.uttOff[u];
  const long long T = (L < p.frameSize) ? 0 : (L - p.frameSize) / p.frameStep + 1;
  float *x = p.band + p.statOff[u] * nB + b;
  if (p.mode == 1) {
    float fir[5] = {0.f, 0.f, 0.f, 0.f, 0.f};   // circular input history, slot ptr = newest
    float iir = 0.f;
    int ptr = 0;
    for (long long t = 0; t < T; t++) {
      const float s = x[t * nB];
      fir[ptr] = s;
      float sum = __fmul_rn(p.fir[0], s);
#pragma unroll
      for (int m = 1; m < 5; m++) sum = __fadd_rn(sum, __fmul_rn(p.fir[m], fir[(5 - m + ptr) % 5]));
      sum = __fadd_rn(sum, __fmul_rn(p.iir, iir));
      iir = sum;
      x[t * nB] = (t >= 5) ? sum : 0.f;
      ptr = (ptr + 1) % 5;
    }
  } else {
    float b0 = 0.f, b1 = 0.f, b2 = 0.f, b3 = 0.f;
    for (long long t = 0; t < T; t++) {
      const float s = x[t * nB];
      const float out = __fadd_rn(__fmul_rn(p.fir[0], s), b0);
      const float fb = (t >= 5) ? __fmul_rn(p.iir, out) : __fmul_rn(__fmul_rn(0.f, p.iir), out);   // (init>=5) * iir * out
      b0 = __fadd_rn(__fadd_rn(__fmul_rn(p.fir[1], s), b1), fb);
      b1 = __fadd_rn(__fmul_rn(p.fir[2], s), b2);
      b2 = __fadd_rn(__fmul_rn(p.fir[3], s), b3);
      b3 = __fmul_rn(p.fir[4], s);
      x[t * nB] = (t >= 5) ? out : 0.f;
    }
  }
}

cudaError_t launch_rasta(const RastaParams &p, int u0, int u1, cudaStream_t st)
{
  const long long n = (long long)(u1 - u0) * p.nBands;
  if (n <= 0) return cudaSuccess;
  const int bs = 128;
  rasta_kernel<<<(unsigned)((n + bs - 1) / bs), bs, 0, st>>>(p, u0, u1);
  return cudaGetLastError();
}

// rest of cPlp after the RASTA filter (plp.cpp:486-590) for 32 static rows per CTA, lane = frame
constexpr int kTailF = 32, kTailWarps = 4;
__global__ void __launch_bounds__(kTailF * kTailWarps) plp_tail_kernel(const LldParams p, const float *band, float *stat,
                                                                       int statStride, int outCol, long long row0, long long row1)
{
  extern __shared__ __align__(16) unsigned char smem[];
  const int nB = p.nBands;
  float *melS = reinterpret_cast<float *>(smem);                    // [nB][F]
  float *acfS = melS + nB * kTailF;                                 // [nAuto][F]
  float *outS = acfS + (kMaxLp + 1) * kTailF;                       // [nStat][2F]
  const int tid = threadIdx.x, f = tid & 31, vw = tid >> 5;
  const long long r0 = row0 + (long long)blockIdx.x * kTailF;
  const int nf = (int)min((long long)kTailF, row1 - r0);
  for (int idx = tid; idx < nB * kTailF; idx += blockDim.x) {
    const int ff = idx / nB, b = idx - ff * nB;
    float v = 0.f;
    if (ff < nf) {
      v = band[(r0 + ff) * nB + b];
      if (p.plpAud) {                                               // plp.cpp:488-510
        if (p.doLog) {
          v = __fmul_rn(__fadd_rn(v, p.plpEql[b]), p.plpCompression);
        } else {
          if (v < p.melfloor) v = p.melfloor;
          v = __fmul_rn(v, p.plpEql[b]);
          v = (float)pow((double)v, (double)p.plpCompression);
        }
      }
      if (p.plpInvLog) v = expf(v);                                 // :513-518
    }
    melS[b * kTailF + ff] = v;
  }
  __syncthreads();
  plp_backend<kTailF, kTailWarps>(p, melS, p.dctCos, p.dctLift, acfS, outS, vw, f);
  __syncthreads();
  for (int idx = tid; idx < nf * p.nStat; idx += blockDim.x) {
    const int ff = idx / p.nStat, c = idx - ff * p.nStat;
    stat[(r0 + ff) * statStride + outCol + c] = outS[c * (2 * kTailF) + ff];
  }
}

cudaError_t launch_plp_tail(const LldParams &op, const float *band, float *stat, int statStride, int outCol,
                            long long row0, long long row1, cudaStream_t st)
{
  if (row1 <= row0) return cudaSuccess;
  const size_t smem = (size_t)(op.nBands + kMaxLp + 1 + 2 * op.nStat) * kTailF * sizeof(float);
  cudaError_t e = cudaFuncSetAttribute(plp_tail_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  const long long nb = (row1 - row0 + kTailF - 1) / kTailF;
  plp_tail_kernel<<<(unsigned)nb, kTailF * kTailWarps, smem, st>>>(op, band, stat, statStride, outCol, row0, row1);
  return cudaGetLastError();
}

// cFullinputMean, single-loop mode (dspcore/fullinputMean.cpp:526-546): means = first frame, += every
// further frame (float, frame order), /= (float)n at EOI.  One thread per (utterance, column of a group
// that ends in a mean subtraction); T follows the group's reader (min over its levels' streams).
__global__ void cms_mean_kernel(const PostParams p, float *means, int u0, int u1)
{
  const int u = u0 + blockIdx.x;
  if (u >= u1) return;
  const long long Ls = p.uttOff[u + 1] - p.uttOff[u];
  const float *src = p.stat + p.statOff[u] * (long long)p.statStride;
  for (int gi = 0; gi < p.nGroups; gi++) {
    const PostGroup &g = p.groups[gi];
    if (g.nStages < 1 || g.kind[g.nStages - 1] != 2) continue;
    int T = (Ls >= g.frameSize) ? (int)((Ls - g.frameSize) / g.frameStep + 1) : 0;
    for (int k = 0; k < g.nLim; k++) T = min(T, (Ls >= g.limSize[k]) ? (int)((Ls - g.limSize[k]) / g.limStep[k] + 1) : 0);
    for (int c = threadIdx.x; c < g.n; c += blockDim.x) {
      float m = 0.f;
      if (T > 0) {
        m = src[g.srcCol + c];
        for (int t = 1; t < T; t++) m = __fadd_rn(m, src[(long long)t * p.statStride + g.srcCol + c]);
        m = __fdiv_rn(m, (float)T);
      }
      means[(long long)u * p.nStat + g.srcCol + c] = m;
    }
  }
}

cudaError_t launch_cms_means(const PostParams &p, float *means, int u0, int u1, cudaStream_t st)
{
  if (u1 <= u0) return cudaSuccess;
  cms_mean_kernel<<<u1 - u0, 64, 0, st>>>(p, means, u0, u1);
  return cudaGetLastError();
}

__global__ void vecop_ll1_kernel(float *stat, int statStride, int srcCol, int n, int outCol, long long row0, long long row1)
{
  const long long r = row0 + (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= row1) return;
  const float *x = stat + r * statStride + srcCol;
  float d = 0.f;
  for (int i = 0; i < n; i++) d = __fadd_rn(d, x[i]);               // vectorOperation.cpp:475-481
  if (n > 0) d = __fdiv_rn(d, (float)n);
  stat[r * statStride + outCol] = d;
}

cudaError_t launch_vecop_ll1(float *stat, int statStride, int srcCol, int n, int outCol, long long row0, long long row1,
                             cudaStream_t st)
{
  if (row1 <= row0) return cudaSuccess;
  const int bs = 128;
  vecop_ll1_kernel<<<(unsigned)((row1 - row0 + bs - 1) / bs), bs, 0, st>>>(stat, statStride, srcCol, n, outCol, row0, row1);
  return cudaGetLastError();
}

cudaError_t launch_pitch_smooth(const AcfPitchParams &p, int u0, int u1, cudaStream_t st)
{
  if (u1 <= u0) return cudaSuccess;
  const int bs = 64;
  pitch_smooth_kernel<<<(u1 - u0 + bs - 1) / bs, bs, 0, st>>>(p, u0, u1);
  return cudaGetLastError();
}

}  // namespace osm
