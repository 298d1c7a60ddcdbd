// plan.hpp -- internal representation of a compiled LLD plan (host side) and the parameter
// blocks handed to the CUDA kernels.  Not part of the public ABI (include/osm_b200.h).
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "frame_geom.cuh"
#include "../../include/osm_b200.h"

namespace osm {

// ---------------------------------------------------------------------------------------
// Host-side tables.  Each builder restates the reference's table construction with the same
// float/double casting order (citations in tables.cpp).
// ---------------------------------------------------------------------------------------
struct MelBank {
  int nBands = 0;
  int nBins = 0;
  int nLo = 0, nHi = 0;            // bins [nLo, nHi) are visited (melspec.cpp:543)
  std::vector<float> coef;         // per bin weight of the lower band (melspec.cpp:441-447)
  std::vector<int> chanMap;        // per bin lower band index, -1, -3 (melspec.cpp:427-438)
  std::vector<double> bandHz;      // band centres in Hz (field info, melspec.cpp:408-411)
  // derived for the kernel: range r (0..nBands) = bins whose chanMap == r-1, as [begin,end)
  std::vector<int> rangeBegin;     // size nBands+2 ; rangeBegin[r+1] = end of range r
  float outScale = 1.f;            // htkcompatible scaling (melspec.cpp:559-569)
  bool usePower = false;
  bool oneTap = false;             // every bin feeds one band only (cTonespec): the (w, 1-w) pair becomes (w, 0)
};

// cTonespec (lld/tonespec.cpp:147-367): the reference's tables, and the same bank as a one-tap MelBank for the kernel's band walk
// (range r = the bins of note r, i.e. of output r-1; coef = filter map times the shifted dB(A) weight)
struct ToneTables {
  std::vector<float> pitchClassFreq;   // [nNotes + 2]
  std::vector<int> binKey;             // [nBins]
  std::vector<int> nbins;              // [nNotes + 2] bins per note over firstBin .. lastBin
  std::vector<float> filterMap;        // [nBins]
  int firstBin = 0, lastBin = 0;
};
struct ToneOp {
  int nNotes = 0;
  bool usePower = false;
  int octaveSize = 0;                  // > 0: cChroma behind the tonespec, 0: the tonespec level is the op's output
  float silThresh = 0.f;
  MelBank bank;
  std::vector<float> divisor;          // [nNotes] (float)pitchClassNbins[b + 1], 0 = output 0 (:424-434)
  int nOut = 0;
};

// cTonefilt (lld/tonefilt.cpp:65-189) after the reference's clamps, and an optional cChroma behind it
struct TonefiltOp {
  int nNotes = 0;
  int P = 1;                           // samples per output row (configureWriter, :101-134)
  double T = 0;                        // period of the wave level
  double period = 0;                   // outputPeriod: period and frame size of the level
  std::vector<double> freq, decay;     // [nNotes] (:180-189)
  int octaveSize = 0;                  // > 0: cChroma behind the filter bank
  float silThresh = 0.f;
};

// cCens (lld/cens.cpp:139-222) on the N columns of a cChroma op
constexpr int kCensMaxTaps = 512;      // winlength bound of the kernel (cens.cu)
struct CensOp {
  int N = 12, W = 41;
  bool l2norm = true;
  int ratio = 1;                       // downsampleRatio: the level's period is the input's times ratio
  std::vector<float> win;              // [W] (float)win[j]
  float unit = 0.f;                    // (float)(1.0 / sqrt((float)N)): every element of a zero-norm row
};

struct FrontEnd {
  double sampleRate = 0;
  int nChan = 1;
  int format = OSM_B200_PCM_S16;
  bool mixdown = true;
  int frameSize = 0, frameStep = 0, nfft = 0, nBins = 0;
  int frameCenter = 0;             // sampling centre in samples: frame t starts at t * frameStep - frameCenter (frame_geom.cuh)
  double frameSizeSec = 0;         // cFramer.frameSize (nominal)
  double frameStepSec = 0;
  double timeOffset = 0;           // seconds added to the time of a frame's first sample (cFramer.frameCenter)
  double fftFrameSizeSec = 0;      // after cTransformFFT's rescale (transformFft.cpp:78-85)
  bool preemph = false;
  float preK = 0.f;
  int preDe = 0;
  std::vector<float> window;       // (float)win[n], size frameSize (windower.cpp:226)
  float winOffset = 0.f;
  bool zeroPadSymmetric = false;   // phase only; magnitude consumers are unaffected
  // cTonefilt rows: the time of row r is that of its first sample, (double)(r * rowSampleStep) / fs (lld/tonefilt.cpp:252,
  // core/dataMemoryLevel.cpp:617-626, 1240); 0: a framer level, r * frameStepSec
  int rowSampleStep = 0;
};

enum StaticOpKind { SOP_MFCC = 0, SOP_PLP, SOP_MELSPEC, SOP_SPECTRAL, SOP_ENERGY, SOP_MZCR, SOP_PITCHACF, SOP_VECOP, SOP_MAG, SOP_INTENSITY, SOP_PITCH, SOP_JITTER, SOP_FORMANT, SOP_HARMONICS, SOP_LPC, SOP_TONE, SOP_TONEFILT, SOP_CENS };

struct MfccOp {
  int melIdx = 0;
  int first = 0, last = 0, nMfcc = 0;
  float melfloor = 0.f;            // value compared against
  float logMelfloor = 0.f;         // logf(melfloor)
  bool doLog = true;
  std::vector<float> cosT;         // [nMfcc][nBands] rows in OUTPUT order (htk c0-last swap applied)
  std::vector<float> liftFactor;   // [nMfcc] = sintable[i0] * factor, output order
};

struct PlpOp {
  int melIdx = 0;
  int lpOrder = 0, nAuto = 0, nFreq = 0, nCeps = 0, firstCC = 0, lastCC = 0;
  bool doLog = false, doAud = true, doInvLog = false, doIDFT = true, doLP = true, doLpToCeps = true;
  bool htk = true;
  float melfloor = 1.f, logMelfloor = 0.f, compression = 0.33f;
  bool lifter = false;
  std::vector<float> eql;          // [nBands] equal loudness weights (log of them when doLog)
  std::vector<float> cosT;         // [nAuto][nFreq] IDFT table (plp.cpp:298-306)
  std::vector<float> lift;         // [nCeps] lifter per OUTPUT slot (plp.cpp:560-573)
  int rasta = 0;                   // 0 none, 1 RASTA, 2 newRASTA: temporal band filter (plp.cpp:361-397,446-483)
  float rastaFir[5] = {0, 0, 0, 0, 0}, rastaIir = 0.f;
  int nOut = 0;
};

// cSpectral resolved against the bin-frequency axis of its input level (lldcore/spectral.cpp)
struct SpectralOp {
  int nSrc = 0;                    // input bins
  int loBin = 1, hiBin = 0;        // specRange (spectral.cpp:625-647)
  double F0 = 0;                   // bin spacing in Hz (field info, transformFft.cpp:111-115)
  bool squareInput = true, useLog = false, normBand = false, buggyRollOff = false, oldSlopeScale = true;
  bool reqMag = false, reqPow = false, reqLog = false;
  float specFloor = 0.f, logSpecFloor = 0.f;
  // bands / slopes: resolved edges
  std::vector<int> bandIL, bandIR; std::vector<double> bandWL, bandWR;
  std::vector<int> slopeIL, slopeIR; std::vector<double> slopeWL, slopeWR, slopeNind;
  std::vector<double> rollOff;
  bool alphaRatio = false, hammarberg = false, flux = false, centroid = false, maxPos = false, minPos = false,
       entropy = false, stddev = false, variance = false, skewness = false, kurtosis = false, slope = false,
       sharpness = false, harmonicity = false, flatness = false, logFlatness = false;
  std::vector<double> sharpW;      // [hiBin-loBin+1]
  int nOut = 0;
};

struct EnergyOp {
  bool htk = false, rms = true, energy2 = false, lg = true;
  float escaleLog = 1, escaleRms = 1, escaleSquare = 1, ebiasLog = 0, ebiasRms = 0, ebiasSquare = 0;
  int nOut = 0;
};

// cAcf (ACF) + cAcf (cepstrum) -> cPitchACF (dspcore/acf.cpp, lldcore/pitchACF.cpp)
struct PitchAcfOp {
  bool acfUsePower = true, cepUsePower = false, absCepstrum = false, normOutput = true;
  bool oldCompatCepstrum = false;  // cepstrum of log(x) (no +1) with DC / Nyquist un-logged (dspcore/acf.cpp:103-109,276-286)
  double maxPitch = 500, voicingCutoff = 0.55;
  float fsSec = 0.f;
  bool voiceProb = true, voiceQual = false, HNR = false, HNRdB = false, linHNR = false, F0 = false, F0raw = false, F0env = false;
  int nOut = 0;
};

// cIntensity (lldcore/intensity.cpp:86-146): Hamming-weighted mean square of the first min(N, nOut) samples
// (the reference bounds its loop by the OUTPUT size, reproduced as is), loudness = (I / 1e-6)^0.3
struct IntensityOp { bool intensity = true, loudness = false; double w[2] = {0, 0}; double winSum = 1.0; int nOut = 0; };

struct MzcrOp { bool zcr = true, mcr = true, amax = true, maxmin = true, dc = false; int nOut = 0; };

// cSpecScale -> cPitchShs -> cPitchSmootherViterbi [-> cValbasedSelector] (dsp/specScale.cpp, lld/pitchShs.cpp,
// lldcore/pitchBase.cpp, lld/pitchSmootherViterbi.cpp, other/valbasedSelector.cpp): one static producer
struct PitchChainOp {
  // --- cSpecScale: natural cubic spline from the linear bins onto an octave axis.  The abscissa terms are
  // constants, so the tridiagonal solve is two first-order recurrences with fixed coefficients:
  //   u[i]  = fwdA[i] * u[i-1] + fwdP6[i] * ((y[i+1]-y[i]) * r1[i] - (y[i]-y[i-1]) * r2[i])      (smileUtilSpline.c:159-165)
  //   y2[j] = bwdD[j] * y2[j+1] + u[j]                                                             (:178-180)
  int nMag = 0, nPts = 0;
  bool enhance = false, smooth = false;
  std::vector<double> fwdA, fwdP6, r1, r2, bwdD;
  std::vector<int> ik; std::vector<double> ia, ic, id;     // interpolation cache (smileUtilSpline.c:301-352)
  std::vector<double> audW;                                 // empty = no auditory weighting
  // --- cPitchShs
  int nCand = 3, nHarm = 15;
  std::vector<int> shift; std::vector<float> hscale;        // per harmonic 2..nHarm: bin shift, compression^(h-1) (float products)
  float Fmint = 0, Fstept = 0;
  double logBase = 0;                                        // log(base)
  double maxPitch = 620, minPitch = 52;
  float voicingCutoff = 0.7f;
  int lfCutBin = -1;
  bool greedy = false, octaveCorr = false, scores = true, voicing = true, F0C1 = false, voicingC1 = false, F0raw = false, voicingClip = false;
  int nShsCols = 0;
  bool shsOnly = false;                                      // the op is the cPitchShs level itself: no Viterbi stage, nOut = nShsCols
  // --- cPitchSmootherViterbi
  int bufLen = 30;
  bool oF0final = true, oF0finalLog = false, oF0finalEnv = false, oF0finalEnvLog = false, oVClipped = false, oVUnclipped = false;
  double wLocal = 2, wTvv = 10, wTvvd = 10, wTvuv = 10, wThr = 4, wRange = 1, wTuu = 0;
  // --- cValbasedSelector (optional)
  bool hasSel = false;
  int selOp = -1;                                            // static op whose first column is the selector value
  float selThreshold = 0, selOutputVal = 0;
  bool selInvert = false, selAllowEqual = false;
  int nOut = 0;
};

// cPitchJitter (lld/pitchJitter.cpp:591-1107): waveform matching around the F0 of a pitch chain op
struct JitterOp {
  int pitchOp = -1, f0Col = 0;         // F0 = column f0Col of static op pitchOp
  double searchRangeRel = 0.1, minCC = 0.5, lgHNRfloor = -100;
  int minNumPeriods = 2;
  bool jitterLocal = false, jitterDDP = false, jitterLocalEnv = false, jitterDDPEnv = false, shimmerLocal = false, shimmerLocalDB = false,
       shimmerLocalEnv = false, shimmerLocalDBEnv = false, harmonicERMS = false, noiseERMS = false, linearHNR = false, logHNR = false,
       shimmerUseRms = false, refinedF0 = false, srcQualRange = false, srcQualMean = false, peakToPeak = false, brokenThresh = false;
  int nOut = 0;
};

// cTransformFFT -> cSpecResample -> cLpc -> cFormantLpc on a windower level (dsp/specResample.cpp, lld/lpc.cpp,
// lld/formantLpc.cpp): one static producer
struct FormantOp {
  int nIn = 0;                     // samples of the windowed frame
  int nRes = 0, nResPad = 0;       // samples of the resampled frame (cSpecResample output), row pitch of D
  std::vector<float> D;            // [nIn][nResPad]: res[i] = sum_m xw[m] * D[m][i]   (composition path)
  // reference-order path (FFT size 512, fft_ref_order.cuh): the frame is transformed with the reference's rounding sequence
  // and resampled by the reference's float inverse-DFT sum; D then holds [wc (256) | cos [kHalf][nResPad] | sin [kHalf][nResPad]]
  bool refOrder = false;
  int kHalf = 0;                   // kMax / 2 of smileDsp_initIrdft: harmonics 1 .. kHalf-1 enter the sum
  int padLeft = 0;                 // zeros in front of the frame (cTransformFFT.zeroPadSymmetric)
  float halfK = 256.0f;            // the sum is divided by K / 2
  int p = 8;                       // cLpc.p
  double T = 0;                    // base period of the cLpc level = 1 / targetFs
  int nFormants = 0;
  double minF = 50, maxF = 5500;
  bool saveFormants = true, saveBandwidths = false, saveNValid = false;
  int nOut = 0;
};

// cHarmonics (lld/harmonics.cpp) on [pitch level ; formant level ; magnitude level]
struct HarmonicsOp {
  int pitchOp = -1, f0Col = 0;        // F0 = column f0Col of the static rows (absolute)
  int formantOp = -1, fmtCol = 0, nFmt = 0;   // formant frequencies = columns fmtCol .. fmtCol + nFmt - 1 (absolute)
  int nb = 0; double binHz = 0;
  int nHarm = 100;
  bool hnr = false;
  std::vector<int> diffs;             // 4 ints per difference: h1formant, h1idx, h2formant, h2idx
  bool fa = false; int faStart = 1, faEnd = 0;
  float floorUnvoiced = -201.f;
  int nOut = 0;
};

// stand-alone cLpc (method acf) on a time-domain frame level, or cLsp on such a cLpc level (lld/lpc.cpp, lld/lsp.cpp)
struct LpcOp { int p = 8; bool lpc = true, gain = false, lsp = false; };

// one field of a level: `n` elements named name (n == 1) or name[i + arrNameOffset]
struct FieldName { std::string name; int n = 1; int arrNameOffset = 0; };

struct StaticOp {
  StaticOpKind kind;
  int stream = 0;                  // index into PlanDesc::streams
  bool windowed = false;           // time-domain ops: reads the windower level instead of the framer level
  int outCol = 0, nOut = 0;
  std::vector<FieldName> fields;   // names of the produced level
  int srcOp = -1;                  // SOP_VECOP: op whose columns of the static level are reduced (ll1); SOP_CENS: the cChroma op
  int magMode = 0;                 // SOP_MAG: 0 magnitude, 1 normalise, 2 power, 3 both, 4 dBpsd (dspcore/fftmagphase.cpp:215-255)
  float magDbNorm = 0.f, magMinDb = 0.f;
  MfccOp mfcc;
  PlpOp plp;
  SpectralOp spectral;
  EnergyOp energy;
  MzcrOp mzcr;
  IntensityOp intensity;
  PitchAcfOp pitch;
  PitchChainOp chain;
  JitterOp jitter;
  FormantOp formant;
  HarmonicsOp harmonics;
  LpcOp lpc;
  ToneOp tone;
  TonefiltOp tonefilt;
  CensOp cens;
};

// temporal stage applied to a static column range (cWindowProcessor family)
enum StageKind { ST_DELTA = 0, ST_SMA = 1, ST_CMS = 2 };   // ST_CMS: cFullinputMean, x - mean over the utterance (win 0)
// flags: ST_SMA bit0 = noZeroSma; ST_DELTA bit0 = onlyInSegments (the norm accumulates over the whole level, SURVEY.md H4)
struct Stage { StageKind kind; int win; int flags; };

// one contiguous block of output columns
struct OutGroup {
  int srcCol = 0, n = 0;           // columns of the static vector
  int stream = 0;                  // stream whose frame geometry defines T of the source level
  std::vector<Stage> stages;       // applied in order
  std::vector<int> limitStreams;   // truncating concat / multi-level reader: source length = min over these streams too
  int outCol = 0;
  // Groups behind a Viterbi-smoothed pitch level are evaluated by seq_post_kernel (one thread per utterance):
  // lagKind 1 = columns of the pitch chain op, 2 = columns of a cPitchJitter op (its level lags during the
  // reference's first end-of-input pass), lagOp = the pitch chain op that supplies the per-utterance lag,
  // segId >= 0 = groups sharing one onlyInSegments delta component (one running norm, in column order)
  int lagKind = 0, lagOp = -1, segId = -1;
  // cValbasedSelector in front of the stages (other/valbasedSelector.cpp:153-233, zeroVec = 1): the element of row i is the source
  // value when the selector value sel[i] (static column gateCol) passes the threshold, else gateOutVal
  int gateCol = -1;
  float gateThreshold = 0.f, gateOutVal = 0.f;
  bool gateInvert = false, gateAllowEqual = false;
};

// one framer -> [pre-emphasis] -> [window] -> [FFT -> magnitude] chain
struct Stream {
  FrontEnd fe;
  bool hasWindow = false, hasFft = false;
  bool dumpMag = false;            // a non-fused consumer reads the magnitude level from HBM
  int fusedOp = -1;                // first band op (MFCC / PLP) evaluated inside lld_kernel, -1 = none
  std::vector<int> bandOps;        // all band ops of this FFT chain, one lld_kernel pass each
  const void *keyFramer = nullptr, *keyPe = nullptr, *keyWin = nullptr;
};

struct PlanDesc {
  std::vector<Stream> streams;
  std::vector<MelBank> mels;
  std::vector<StaticOp> ops;
  int nStatic = 0;
  std::vector<OutGroup> groups;
  int nOut = 0;
  std::vector<std::string> names;  // output element names
  // The output level is the host layer's "_unionconcat" of the input levels of several cFunctionals instances: every level keeps
  // its own length (no min over the levels), the output has as many rows as the longest (rows past a level's end are not read)
  bool padRows = false;
  int periodScale = 1;             // the output level's period = frameStepSec of stream 0 times this (cCens.downsampleRatio)
  const FrontEnd &fe0() const { return streams[0].fe; }
};

// graph.cpp
osm_b200_status compile_graph(const osm_b200_component *comps, int n, const char *outputLevel,
                              PlanDesc &out, std::string &err);
int64_t desc_num_frames(const PlanDesc &d, int64_t nSampleFrames);
int64_t desc_num_frames_first_eoi(const PlanDesc &d, int64_t nSampleFrames, int64_t viterbiFrames = -1);
int64_t desc_num_static_frames(const PlanDesc &d, int stream, int64_t nSampleFrames);
int64_t desc_max_static_frames(const PlanDesc &d, int64_t nSampleFrames);

// tables.cpp
void build_window(int winFunc, int N, double sigma, double gain, std::vector<float> &w, const double *alpha = nullptr, int squareRoot = 0, double fade = 0.0);
void build_mel(const osm_b200_melspec &cfg, int nBins, double frameSizeSec, MelBank &mb);
void build_mfcc(const osm_b200_mfcc &cfg, int nBands, MfccOp &op);
bool build_plp(const osm_b200_plp &cfg, const MelBank &mb, double levelPeriod, PlpOp &op, std::string &err);
bool build_spectral(const osm_b200_spectral &cfg, int nSrc, double fftFrameSizeSec, SpectralOp &op, std::string &err);
void build_energy(const osm_b200_energy &cfg, EnergyOp &op);
// cTonespec on a magnitude level of nBins bins, frame length fftFrameSizeSec; false (err set) where the reference's table
// construction writes past its filter map
bool build_tone_tables(const osm_b200_tonespec &cfg, int nBins, double fftFrameSizeSec, ToneTables &t, std::string &err);
bool build_tone(const osm_b200_tonespec &cfg, int nBins, double fftFrameSizeSec, ToneOp &op, std::string &err);
void build_mzcr(const osm_b200_mzcr &cfg, MzcrOp &op);
// cTonefilt on a wave level of sampling rate fs: the reference's clamps, block length and tables; false (err set) where unsupported
bool build_tonefilt(const osm_b200_tonefilt &cfg, double fs, TonefiltOp &op, std::string &err);
// vc == nullptr: the op stops at the cPitchShs level (PitchChainOp::shsOnly)
bool build_pitch_chain(const osm_b200_specscale &sc, const osm_b200_pitchshs &ps, const osm_b200_pitchsmootherviterbi *vc,
                       int nMag, double fftFrameSizeSec, PitchChainOp &op, std::string &err);

// fe = front end of the windower level the chain's cTransformFFT reads; zeroPadSymmetric = that cTransformFFT's switch
void build_ref_fft_tables(std::vector<float> &wc);
osm_b200_status set_last_error(osm_b200_status st, const std::string &msg);   // api.cu
bool build_formant(const osm_b200_specresample &rs, const osm_b200_lpc &lp, const osm_b200_formantlpc &fl, const FrontEnd &fe,
                   bool zeroPadSymmetric, FormantOp &op, std::string &err);

}  // namespace osm
