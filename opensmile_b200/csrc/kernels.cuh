// kernels.cuh -- parameter blocks and launchers of the fused LLD kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

#include "frame_geom.cuh"

namespace osm {

constexpr int kMaxVW = 32;   // virtual warps (F-lane groups) per CTA

struct TileRef { int32_t utt; int32_t f0; };   // (utterance, first row) of a post_kernel tile
// output rows [a,b) of one utterance = one CTA work unit; tile0 = global index of its first tile; w0 = tiles the chunks
// before it in the list compute (the position of its first tile in the launch's schedule, see LldParams::ctaTiles)
struct ChunkRef { int32_t utt; int32_t a; int32_t b; int32_t tile0; int32_t w0; };

// Everything the fused per-frame kernel needs.  Pointers are device pointers; the table
// pointers reference one packed constant blob uploaded at plan creation.
struct LldParams {
  // ---- input ----
  const int16_t *pcm;
  const long long *uttOff;       // [nUtt+1] sample-frame offsets
  const long long *rowOff;       // [nUtt+1] first output row of each utterance
  const ChunkRef *chunks;
  int nChunks;
  // schedule: CTA g runs, in order, the chunks c with g * ctaTiles <= chunks[c].w0 - chunks[0].w0 < (g + 1) * ctaTiles,
  // a contiguous run of about ctaTiles tiles (the host cuts chunks at these boundaries); nRuns = grid size
  int ctaTiles, nRuns;
  int nChan;
  // 1: `pcm` holds pre-converted mono float samples (pcm_convert_kernel: every input format but 16-bit integer).  The sample
  // frame is 4 bytes wide, so nChan is 2 here -- all offset arithmetic stays in int16 units -- and only the conversion differs.
  // Every kernel that reads PCM has an instance per format (template flag F32); its launcher picks it from this field.  A
  // run-time "float samples?" test inside the sample accessors made the ComParE step measurably slower.
  int pcmF32;
  // fused temporal stages (static | delta(W1) | delta(W1,W2)); halo = W1 + W2, 0 when not fused
  unsigned hopMagic;             // ceil(2^32 / frameStep): i / frameStep == __umulhi(i, hopMagic) for i * frameStep < 2^32
                                 // (0 for frameStep 1: 2^32 does not fit)
  int narrow;                    // 1: half-width tiles (F/2 frames), used when the full tile does not fit shared memory
  int fused, halo, fW1, fW2;
  float fNorm1, fNorm2;
  float fRcp1, fRcp2;            // 1/norm when the reciprocal+FMA division is proven exact for it, else 0
  // ---- front end ----
  int frameSize, frameStep, sPad;
  int preemph, preDe;
  float preK, oneMinusK;
  int hasWinOffset;
  float winOffset;
  const float4 *winLut;          // [M] (w[2e], w[2e+1], smem offset of sample 2e as int bits, #valid samples of the pair)
  const float2 *twiddles;        // per-stage tables, concatenated
  int twOff[4];                  // offset (in float2) of each stage's table
  int twCount;                   // total float2 in twiddles
  const float2 *splitTw;         // [M/2+1] exp(-2 pi i k / N)
  // ---- mel + mfcc op ----
  const float *melCoef;          // [nBins]
  const int *melRange;           // [nBands+2]
  // visit list of the mel phase: per range r the (w, 1-w) pairs of its bins, zero-padded to a multiple
  // of 4 entries (the padding multiplies the next bins by 0): melVisit[melVB[r] .. melVB[r+1])
  const float2 *melVisit; const int *melVB; int melVCount;
  int nBands;
  float melScale;
  int melUsePower;
  int melSplit[kMaxVW + 1];      // virtual warp w computes bands [melSplit[w], melSplit[w+1])
  // ---- static LLD op on the mel bands: 0 = cMfcc (log, DCT-II, lifter), 1 = cPlp, 2 = cTonespec [-> cChroma], -1 = none ----
  int opKind;
  // magnitude level for non-fused consumers (cSpectral ...): tile-major [tile][bin][F] floats, or null
  float *magOut;
  int nStat;                     // static outputs per frame (nMfcc / nCeps / ...)
  const float *dctCos;           // MFCC: [nStat][dctStride] DCT rows (output order, zero padded)
                                 // PLP : [nAuto][dctStride = nFreq] IDFT table
  int dctRows, dctStride;
  const float *dctLift;          // [nStat] MFCC: lifter * sqrt(2/N) ; PLP: lifter per output slot
  float melfloor, logMelfloor;
  int doLog;
  // cPlp (lldcore/plp.cpp:416-593)
  const float *plpEql;           // [nBands]
  int plpAud, plpInvLog, plpIDFT, plpLP, plpCeps, plpHtk, plpLifter;
  int plpOrder, plpNAuto, plpNFreq, plpFirstCC, plpLastCC;
  float plpCompression;
  // ---- output ----
  float *out;
  int outStride, outCol;
  // cTonespec / cChroma (opKind 2, lld/tonespec.cpp:403-434, lld/chroma.cpp:86-117): band = note, dctCos = per-note bin counts,
  // toneSqrt = usePower; chromaOct > 0 folds the notes into that many chroma values, 0 outputs the notes
  int toneSqrt, chromaOct;
  float chromaSilThresh;
  // ---- front end (cont.) ----
  int frameCenter;               // frame t starts at sample t * frameStep - frameCenter of its utterance (frame_geom.cuh)
};

// temporal post-processing (cDeltaRegression / cContourSmoother chains)
struct PostGroup {
  int srcCol, n, outCol;
  int frameSize, frameStep, frameCenter;   // geometry of the stream the source level belongs to (defines its T)
  // the source sits in a multi-level reader / concat together with levels of other streams: the
  // reader only delivers min over them (core/dataReader.cpp:375-380) -> T = min(T, T of these)
  int nLim; int limSize[3], limStep[3], limCenter[3];
  int nStages;
  int kind[3];                   // 0 = delta, 1 = sma, 2 = utterance mean subtraction (cFullinputMean)
  int win[3];
  int flags[3];
};
constexpr int kMaxPostGroups = 24;   // emo_large.conf: 6 smoothed levels x (sma, Δ, ΔΔ) = 18
struct PostParams {
  const float *stat;             // static rows
  int statStride;
  const long long *statOff;      // [nUtt+1] static row offsets
  float *out;
  int outStride;
  const long long *rowOff;       // [nUtt+1] output row offsets
  const long long *uttOff;       // [nUtt+1] sample-frame offsets (to derive T)
  int nUtt;
  int nGroups;
  PostGroup groups[kMaxPostGroups];
  const TileRef *tiles;          // (utt, first output row) per CTA, `rows` output rows each
  int rows;                      // output rows per CTA: post_tile_rows(nStat, maxN, halo)
  int nTiles;
  int nStat;                     // static columns staged per row
  int maxN;                      // widest group
  int halo;                      // max over groups of the summed half windows
  const float *means;            // [nUtt][nStat] per-utterance column means (groups with a kind-2 stage), or null
};

// kernel: static name of the instance that ran, e.g. "lld512_kernel<16>" or "lld_kernel<1024,8,256,1,VEC2,GEN>"
struct LldLaunchInfo { int grid, block; size_t smem; const char *kernel; long long nChunks; };

// returns cudaSuccess or the launch error; fills `info`.  launch = false only fills `info`, with grid = the CTAs the
// selected instance keeps resident (numSMs x occupancy)
cudaError_t launch_lld(const LldParams &p, int nfft, int numSMs, cudaStream_t st, LldLaunchInfo *info, bool launch = true);
cudaError_t launch_post(const PostParams &p, cudaStream_t st);
// lld_fast.cu: the specialised 512-point mono MFCC instance (same contract and results as lld_kernel); launch_lld selects it
// unless OSM_B200_LLD_FAST=0
bool lld_fast_applies(const LldParams &p, int nfft);
cudaError_t launch_lld_fast(const LldParams &p, int numSMs, cudaStream_t st, LldLaunchInfo *info, bool launch);
// output rows per post_kernel CTA: 64, or fewer when a wide static level would not fit shared memory
int post_tile_rows(int nStat, int maxN, int halo);
// smem bytes the fused kernel needs for a given geometry (host helper, used for diagnostics)
size_t lld_smem_bytes(const LldParams &p, int nfft);
// frames per tile / virtual warps per CTA for a given FFT size
int lld_tile_frames(int nfft, bool narrow = false);
int lld_virtual_warps(int nfft);
int lld_max_chunk_tiles();
bool lld_supported_fft(int nfft);

// ------------------------------------------------------------------------------------------
// standalone per-frame ops (ops.cu): lane = frame kernels used when an op is not fused into
// lld_kernel.  One tile = up to F consecutive frames of one utterance.
// ------------------------------------------------------------------------------------------
struct OpTile { int32_t utt; int32_t f0; int32_t nf; int32_t prev; };   // prev = 1 if frame f0-1 exists in tile-1

struct SpectralParams {
  const float *mag;              // tile-major magnitude level [tile][nSrc][F]
  const OpTile *tiles; int nTiles; int F;
  const long long *statOff;      // static row offsets
  float *stat; int statStride, outCol;
  int nSrc, loBin, hiBin;
  double F0;
  int squareInput, useLog, normBand, buggyRollOff, oldSlopeScale, reqMag, reqPow, reqLog;
  float specFloor, logSpecFloor;
  int nBands; int bandIL[16], bandIR[16]; double bandWL[16], bandWR[16];
  int nSlopes; int slopeIL[16], slopeIR[16]; double slopeWL[16], slopeWR[16], slopeNind[16];
  int nRollOff; double rollOff[16];
  int alphaRatio, hammarberg, flux, centroid, maxPos, minPos, entropy, stddev, variance, skewness, kurtosis,
      slope, sharpness, harmonicity, flatness, logFlatness;
  const double *sharpW;          // [hiBin-loBin+1] (device)
  int stageMag;                  // set by the launcher: magnitude tile staged in shared memory
};

struct TimeOpParams {            // cEnergy / cMZcr on the framer or windower level
  const int16_t *pcm; int nChan; int pcmF32;   // pcmF32: see LldParams
  const long long *uttOff, *statOff;
  const OpTile *tiles; int nTiles; int F;
  float *stat; int statStride, outCol;
  int frameSize, frameStep, frameCenter;
  int windowed, preemph, preDe; float preK, oneMinusK, winOffset;
  const float *window;           // [frameSize] (device), only when windowed
  // cEnergy
  int eHtk, eRms, eEnergy2, eLog; float escaleLog, escaleRms, escaleSquare, ebiasLog, ebiasRms, ebiasSquare;
  // cMZcr
  int zZcr, zMcr, zAmax, zMaxmin, zDc;
  // cIntensity
  int iIntensity, iLoudness; double iW0, iW1, iWinSum;
};

// cAcf (ACF) + cAcf (cepstrum) + cPitchACF: per-frame part (one CTA per tile, batched complex FFT of
// size nfft over the symmetric power / log spectrum) and the per-utterance smoothing pass
struct PitchRaw { double voicing, acfZcr; int maxIdx; float hnr, hnrDB, hnrLin; };
struct AcfPitchParams {
  const float *mag;              // tile-major magnitude level [tile][nSrc][F]
  const OpTile *tiles; int nTiles; int F;
  int nfft, nSrc;
  const long long *statOff, *uttOff;
  PitchRaw *raw;                 // [static rows]
  const float2 *twiddles; int twOff[4]; int twCount;
  int acfUsePower, cepUsePower, absCepstrum, normOutput;
  int oldCompatCepstrum;         // cepstrum input: log(x) without +1, DC and Nyquist un-logged (dspcore/acf.cpp:276-286)
  double maxPitch, voicingCutoff;
  float fsSec;
  int voiceProb, voiceQual, HNR, HNRdB, linHNR, F0, F0raw, F0env;
  // smoothing pass
  float *stat; int statStride, outCol;
  int frameSize, frameStep, frameCenter, nUtt;
};
cudaError_t launch_acf_pitch(const AcfPitchParams &p, cudaStream_t st);     // per-frame analysis -> raw
cudaError_t launch_pitch_smooth(const AcfPitchParams &p, int u0, int u1, cudaStream_t st);   // raw -> static columns
bool acf_pitch_supported_fft(int nfft);

// cPlp with RASTA: lld_kernel leaves the (log) band level in `band`, rasta_kernel filters it in place
// along time (one thread per utterance x band, lldcore/plp.cpp:446-483), plp_tail_kernel applies the
// rest of cPlp (auditory weighting ... cepstrum, :486-590) and writes the op's static columns.
struct RastaParams {
  float *band; int nBands;       // [static rows][nBands]
  const long long *uttOff, *statOff;
  int frameSize, frameStep, frameCenter;
  int mode;                      // 1 RASTA, 2 newRASTA
  float fir[5], iir;
};
cudaError_t launch_rasta(const RastaParams &p, int u0, int u1, cudaStream_t st);
// op = the cPlp op's LldParams (tables + plp* switches); rows [row0, row1) of the static level
cudaError_t launch_plp_tail(const LldParams &op, const float *band, float *stat, int statStride, int outCol,
                            long long row0, long long row1, cudaStream_t st);
// cVectorOperation ll1: stat[row][outCol] = (sum_i stat[row][srcCol + i]) / n, float, in order
// cFullinputMean: means[u][srcCol + c] = (float sum over the utterance's T frames, in frame order) / (float)T
// for the columns of every output group that ends in a mean subtraction (dspcore/fullinputMean.cpp:526-546)
cudaError_t launch_cms_means(const PostParams &p, float *means, int u0, int u1, cudaStream_t st);
cudaError_t launch_vecop_ll1(float *stat, int statStride, int srcCol, int n, int outCol, long long row0, long long row1,
                             cudaStream_t st);

// *staged (optional): 1 when the magnitude tile was staged in shared memory; *smem (optional): dynamic shared memory of the launch
cudaError_t launch_spectral(const SpectralParams &p, cudaStream_t st, int *staged = nullptr, int *smemBytes = nullptr);
// cFFTmagphase as an output level: tile-major magnitude level [tile][nSrc][F] -> columns of the static rows
cudaError_t launch_mag_rows(const float *mag, const OpTile *tiles, int nTiles, int F, int nSrc, const long long *statOff,
                            float *stat, int statStride, int outCol, cudaStream_t st, int mode = 0, float fftN = 1.f, float dBpnorm = 0.f,
                            float mindBp = 0.f);
cudaError_t launch_energy(const TimeOpParams &p, cudaStream_t st);
cudaError_t launch_mzcr(const TimeOpParams &p, cudaStream_t st);
cudaError_t launch_intensity(const TimeOpParams &p, cudaStream_t st);

// ------------------------------------------------------------------------------------------
// formant chain (formant.cu): windower level -> [cTransformFFT -> cSpecResample] -> cLpc -> cFormantLpc, one CTA
// per tile of frames: dense resampling product, then one warp per frame (ACF, Durbin, polynomial roots)
// ------------------------------------------------------------------------------------------
struct FormantParams {
  TimeOpParams tp;               // frame geometry, tiles, static rows (windowed = 1)
  const float *D;                // [frameSize][nResPad] composition of zero padding, FFT and the resampling inverse DFT
  int nRes, nResPad;             // samples of the resampled frame, row pitch of D
  int refOrder, kHalf, padLeft;  // reference-order path: D = [wc | cos | sin] (plan.hpp FormantOp)
  float halfK;
  int p;                         // predictor order
  int nFormants;
  double T, minF, maxF;          // sample period of the cLpc level, search range
  int saveFormants, saveBandwidths, saveNValid;
};
cudaError_t launch_formant(const FormantParams &p, cudaStream_t st);
size_t formant_smem_bytes(const FormantParams &p);

// ------------------------------------------------------------------------------------------
// stand-alone cLpc (method acf) [-> cLsp] on a time-domain frame level (lsp.cu): one CTA per tile, one warp per frame for
// the autocorrelation (lane = lag), then one lane per frame for Levinson-Durbin and the LSP root search
// ------------------------------------------------------------------------------------------
struct LpcParams {
  TimeOpParams tp;               // frame geometry, tiles, static rows; windowed / preemph describe the level cLpc reads
  int p;                         // predictor order
  int outLpc, outGain, outLsp;   // columns written: lpcCoeff[p] | lpGain  (a cLpc level)  or  lspFreq[p]  (a cLsp level)
};
cudaError_t launch_lpc(const LpcParams &p, cudaStream_t st);
size_t lpc_smem_bytes(const LpcParams &p);

// cHarmonics (harmonics.cu): one warp per frame on the magnitude level + F0 / formant columns of the static rows
struct HarmonicsParams {
  const float *mag;              // tile-major magnitude level [tile][nb][F]
  const OpTile *tiles; int nTiles; int F;
  int nb; double binHz;          // bins, bin spacing in Hz (frequency axis of the level, transformFft.cpp:111-115)
  const long long *statOff;
  float *stat; int statStride, outCol;
  int f0Col, fmtCol, nFmt;       // columns of the static rows: F0, formant frequencies
  const double *cosTab;          // [2 (nb - 1)] cos(2 pi m / N)
  int nHarm, doHnr, nDiffs;
  int diffs[16];                 // per difference: h1formant, h1idx, h2formant, h2idx
  int doFa, faStart, faEnd;
  float floorUnvoiced;
};
cudaError_t launch_harmonics(const HarmonicsParams &p, cudaStream_t st);
size_t harmonics_smem_bytes(const HarmonicsParams &p);

// ------------------------------------------------------------------------------------------
// cTonefilt [-> cChroma] on the wave level (tonefilt.cu, tonefilt_math.cuh): one CTA per segment of rows (blocks of P samples)
// of one utterance; the in-block sums are one FP64 tensor-core product with the table W, the blocks are chained per note
// ------------------------------------------------------------------------------------------
struct TonefiltParams {
  TimeOpParams tp;               // pcm, nChan, pcmF32, uttOff, statOff, stat, statStride, outCol (frame fields unused)
  const ChunkRef *segs; int nSegs;   // segments: rows [a, b) of utterance utt
  const double *W; int nc, kp;   // [kp][nc]: w_j of every note, re / im interleaved, zero-padded (tonefilt_math.cuh block_tables)
  const double *a, *freq;        // [nNotes] d^P, note frequency
  int P, nNotes; double T;       // samples per block, notes, period of the wave level
  double2 *agg, *cin;            // [nSegs][nNotes] end state of a segment from a zero state / state entering it
  int chromaK; float silThresh;  // chromaK > 0: cChroma behind the filter bank (octaveSize), 0: the tone values are the output
  size_t smemSums;               // byte offset of the chroma staging area in shared memory (tonefilt_smem_bytes)
};
// uttSeg0[u] = first segment of utterance u (absolute); p.segs / agg / cin start at segment uttSeg0[u0].  carry = some utterance of
// [u0, u1) has more than one segment: the aggregate pass and the carry kernel run first.
cudaError_t launch_tonefilt(const TonefiltParams &p, const int32_t *uttSeg0, int u0, int u1, bool carry, cudaStream_t st);
size_t tonefilt_smem_bytes(int nNotes, int chroma, size_t *sumsOffset);

// ------------------------------------------------------------------------------------------
// cCens on the N columns of a cChroma op (cens.cu): one CTA per tile of up to kCensRows rows of one utterance, the W - 1 rows in
// front of the tile staged with it; the CENS rows overwrite columns outCol .. outCol + N - 1 of the static level
// ------------------------------------------------------------------------------------------
constexpr int kCensRows = 128;
struct CensParams {
  float *stat; int statStride; const long long *statOff;
  const OpTile *tiles; int nTiles;   // rows [f0, f0 + nf) of utterance utt
  int srcCol, outCol, N, W;
  const float *win;                  // [W] (float)win[j]
  int l2norm; float unit;            // unit: every element of a zero-norm row
};
cudaError_t launch_cens(const CensParams &p, cudaStream_t st);
size_t cens_smem_bytes(int N, int W);
// once per plan, on its device: the shared-memory limit the shape (N, W) needs (optinBytes = sharedMemPerBlockOptin)
cudaError_t cens_configure(int N, int W, size_t optinBytes);

// ------------------------------------------------------------------------------------------
// SHS pitch chain (pitch.cu): cSpecScale + cPitchShs per frame (one warp per frame), cPitchSmootherViterbi
// [+ cValbasedSelector] per utterance (one thread), cPitchJitter per utterance (one warp), and the temporal
// stages of the levels behind them (one thread per utterance, seq_post_kernel).
// ------------------------------------------------------------------------------------------
struct ShsParams {
  const float *mag;              // tile-major magnitude level [tile][nMag][F]
  const OpTile *tiles; int nTiles; int F;
  const long long *statOff;      // static row offsets
  float *shs; int nShsCols;      // [static rows][nShsCols] cPitchShs level
  int nMag, nPts, blk;           // blk = ceil(nMag / 32)
  int enhance, smooth, hasAudW;
  const double *fwdA, *fwdP6, *r1, *r2, *bwdD;   // [nMag]
  const int *ik; const double *ia, *ic, *id;     // [nPts]
  const double *audW;                            // [nPts]
  int nCand, nHarm;
  int shift[32]; float hscale[32];               // [nHarm-1] per harmonic 2..nHarm: bin shift, compression^(h-1) (kernel parameters = constant bank)
  float Fmint, Fstept; double logBase, maxPitch, minPitch; float voicingCutoff;
  int lfCutBin, greedy, octaveCorr, scores, voicing, F0C1, voicingC1, F0raw, voicingClip;
};
cudaError_t launch_shs(const ShsParams &p, cudaStream_t st);

struct ViterbiParams {
  const float *shs; int nShsCols, nCand;
  const long long *uttOff, *statOff;
  int frameSize, frameStep, frameCenter;
  float *stat; int statStride, outCol;
  int *lag;                      // [nUtt] frames the level holds before the end-of-input flush
  int bufLen;
  int oF0final, oF0finalLog, oF0finalEnv, oF0finalEnvLog, oVClipped, oVUnclipped;
  double wLocal, wTvv, wTvvd, wTvuv, wThr, wRange, wTuu;
  float voiceThresh;
  int hasSel, selCol, selInvert, selAllowEqual; float selThreshold, selOutputVal;
};
cudaError_t launch_viterbi(const ViterbiParams &p, int u0, int u1, cudaStream_t st);

struct JitterParams {
  const int16_t *pcm; int nChan; int pcmF32;   // pcmF32: see LldParams
  const long long *uttOff, *statOff;
  int frameSize, frameStep, frameCenter;
  double Ts, pitchT;             // wave sample period, period of the F0 level
  float *stat; int statStride, f0Col, outCol;
  double searchRangeRel; float threshCC, lgHNRfloor; int minNumPeriods;
  int jitterLocal, jitterDDP, jitterLocalEnv, jitterDDPEnv, shimmerLocal, shimmerLocalDB, shimmerLocalEnv, shimmerLocalDBEnv,
      harmonicERMS, noiseERMS, linearHNR, logHNR, shimmerUseRms, refinedF0, srcQualRange, srcQualMean, peakToPeak, brokenThresh;
  int *errFlag;                  // set when a frame exceeds the kernel's workspace (reported by the host)
  // per-warp workspace (elements): staged wave window, cross correlations per candidate period length, averaged
  // period waveform, period starts -- sized from the frame geometry and the pitch range of the F0 level
  int capWav, capCC, capAvg, capPb;
};
cudaError_t launch_jitter(const JitterParams &p, int u0, int u1, cudaStream_t st);

// gateCol >= 0: cValbasedSelector (zeroVec) in front of the smoother -- the value of row i is the source value when the selector
// column passes the threshold (gateFlags bit 0 = invert, bit 1 = allowEqual), else gateOut (other/valbasedSelector.cpp:195-233)
struct SeqGroup { int srcCol, n, outCol, lagKind, nStages, deltaWin, noZero, segId, gateCol, gateFlags; float gateThr, gateOut; };
constexpr int kMaxSeqGroups = 56, kMaxSegIds = 16;
struct SeqPostParams {
  const float *stat; int statStride;
  const long long *statOff, *rowOff, *uttOff;
  float *out; int outStride;
  const int *lag;
  int frameSize, frameStep, frameCenter;
  int nGroups;
  SeqGroup groups[kMaxSeqGroups];
};
cudaError_t launch_seq_post(const SeqPostParams &p, int u0, int u1, cudaStream_t st);

}  // namespace osm
