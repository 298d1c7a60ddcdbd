/*
 * osm_b200.h -- C ABI of libosm_b200.so: the H100 (sm_90a) back end for openSMILE's
 * per-frame low-level-descriptor (LLD) extraction path.
 *
 * Boundary (SURVEY.md 8b).  In the reference every LLD component is a cSmileComponent
 * subclass whose per-frame hook is called once per tick by cComponentManager::tick
 * (src/core/componentManager.cpp:1233-1262):
 *     cWinToVecProcessor::doProcess        src/include/core/winToVecProcessor.hpp:124-126
 *     cVectorProcessor::processVector      src/include/core/vectorProcessor.hpp:98-129
 *     cWindowProcessor::processBuffer      src/core/windowProcessor.cpp:124-146
 * This library replaces the *numerics* of that sub-graph (wave level -> lld level) by block
 * execution: the host side describes the component chain exactly as the .conf file does
 * (one osm_b200_component per [instance:cType] section, same field names and defaults as
 * the reference's ConfigType, see SURVEY.md Appendix A), osm_b200_plan_create() resolves
 * the reader.dmLevel / writer.dmLevel wiring and compiles it into one fused CUDA plan, and
 * osm_b200_plan_run_*() pushes a whole batch of utterances through it.
 *
 * Conventions (same spirit as progsrc/include/smileapi/SMILEapi.h:16-26,82-153):
 *   - plain C, no exceptions cross the boundary, every call returns osm_b200_status;
 *     osm_b200_last_error() returns a message owned by the library (thread local);
 *   - plan handles are owned by the caller (create/destroy);
 *   - *_device entry points take device pointers and a cudaStream_t passed as void*
 *     (NULL = default stream) and are asynchronous; *_host entry points take host
 *     buffers, do H2D / D2H themselves and return when the result is in `out`;
 *   - there is NO CPU fallback: without a usable CUDA device every compute call fails
 *     with OSM_B200_ERR_CUDA.
 *
 * Data layout.  PCM: all utterances of a batch packed back to back in one buffer,
 * utterance u starting at sample-frame offset utt_offsets[u] (units: sample frames, i.e.
 * one sample of every channel) and ending at utt_offsets[u+1]; interleaved channels,
 * int16 little endian (cWaveSource, src/iocore/waveSource.cpp:217-345).  Offsets that are
 * multiples of 8 sample frames get 16-byte vector loads, anything else still works.
 * Output: float32 rows, row-major, one row per LLD frame (`lld` level layout,
 * src/include/core/dataMemoryLevel.hpp:178-179), utterance u's rows starting at
 * frame_offsets[u]; number of rows per utterance follows the reference's framer / EOI
 * rules and is returned by osm_b200_plan_num_frames().
 */
#ifndef OSM_B200_H
#define OSM_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* 2: component types cSpecScale .. cPitchJitter appended (existing values and struct layouts unchanged)
 * 3: cSpecResample, cLpc, cFormantLpc, cDataSelector, cHarmonics appended (same rule; sizeof(osm_b200_component) grows);
 *    later cLsp appended under the same number: a new enum value at the end, no struct layout or size changes;
 *    cTonespec and cChroma likewise (their parameter blocks are smaller than the union); cTonefilt and cCens likewise */
#define OSM_B200_ABI_VERSION 3
#if defined(__GNUC__)
#define OSM_B200_API __attribute__((visibility("default")))
#else
#define OSM_B200_API
#endif
#define OSM_B200_NAME_LEN 64
#define OSM_B200_MAX_INPUTS 8
#define OSM_B200_MAX_LIST 16
#define OSM_B200_MAX_SELECTED 32

typedef enum {
  OSM_B200_OK = 0,
  OSM_B200_ERR_INVALID = 1,      /* bad argument / malformed graph          (cf. SMILE_INVALID_ARG) */
  OSM_B200_ERR_UNSUPPORTED = 2,  /* valid openSMILE graph this back end does not fuse (yet)      */
  OSM_B200_ERR_CUDA = 3,         /* CUDA runtime / device error, no device  (cf. SMILE_FAIL)       */
  OSM_B200_ERR_NOMEM = 4
} osm_b200_status;

/* component types; names = the reference's registered component names
 * (src/include/core/componentList.hpp:172-390) */
typedef enum {
  OSM_B200_C_WAVESOURCE = 0,     /* cWaveSource / cExternalAudioSource: defines the `wave` level */
  OSM_B200_C_FRAMER,             /* cFramer             src/dspcore/framer.cpp:54-68               */
  OSM_B200_C_VECTORPREEMPHASIS,  /* cVectorPreemphasis  src/dspcore/vectorPreemphasis.cpp:89-108  */
  OSM_B200_C_WINDOWER,           /* cWindower           src/dspcore/windower.cpp:159-229          */
  OSM_B200_C_TRANSFORMFFT,       /* cTransformFFT       src/dspcore/transformFft.cpp:165-223      */
  OSM_B200_C_FFTMAGPHASE,        /* cFFTmagphase        src/dspcore/fftmagphase.cpp:179-292       */
  OSM_B200_C_MELSPEC,            /* cMelspec            src/lldcore/melspec.cpp:184-573           */
  OSM_B200_C_MFCC,               /* cMfcc               src/lldcore/mfcc.cpp:136-281              */
  OSM_B200_C_PLP,                /* cPlp                src/lldcore/plp.cpp:276-593               */
  OSM_B200_C_SPECTRAL,           /* cSpectral           src/lldcore/spectral.cpp:586-1555         */
  OSM_B200_C_ENERGY,             /* cEnergy             src/lldcore/energy.cpp:152-187            */
  OSM_B200_C_MZCR,               /* cMZcr               src/lldcore/mzcr.cpp:109-157              */
  OSM_B200_C_ACF,                /* cAcf                src/dspcore/acf.cpp:170-354               */
  OSM_B200_C_PITCHACF,           /* cPitchACF           src/lldcore/pitchACF.cpp:137-361          */
  OSM_B200_C_DELTAREGRESSION,    /* cDeltaRegression    src/dspcore/deltaRegression.cpp:113-175   */
  OSM_B200_C_CONTOURSMOOTHER,    /* cContourSmoother    src/dspcore/contourSmoother.cpp:84-117    */
  OSM_B200_C_VECTORCONCAT,       /* cVectorConcat       src/other/vectorConcat.cpp:48-53          */
  OSM_B200_C_VECTOROPERATION,    /* cVectorOperation    src/other/vectorOperation.cpp:130 (ll1)   */
  OSM_B200_C_FULLINPUTMEAN,      /* cFullinputMean      src/dspcore/fullinputMean.cpp:484-548     */
  OSM_B200_C_INTENSITY,          /* cIntensity          src/lldcore/intensity.cpp:124-146         */
  OSM_B200_C_SPECSCALE,          /* cSpecScale          src/dsp/specScale.cpp:318-371             */
  OSM_B200_C_PITCHSHS,           /* cPitchShs           src/lld/pitchShs.cpp:220-358, lldcore/pitchBase.cpp:173-300 */
  OSM_B200_C_PITCHSMOOTHERVITERBI, /* cPitchSmootherViterbi src/lld/pitchSmootherViterbi.cpp:79-545 */
  OSM_B200_C_VALBASEDSELECTOR,   /* cValbasedSelector   src/other/valbasedSelector.cpp:130-233    */
  OSM_B200_C_PITCHJITTER,        /* cPitchJitter        src/lld/pitchJitter.cpp:591-1107          */
  OSM_B200_C_SPECRESAMPLE,       /* cSpecResample       src/dsp/specResample.cpp:97-185           */
  OSM_B200_C_LPC,                /* cLpc                src/lld/lpc.cpp:156-215 (method acf)      */
  OSM_B200_C_FORMANTLPC,         /* cFormantLpc         src/lld/formantLpc.cpp:192-394 (root solving branch) */
  OSM_B200_C_DATASELECTOR,       /* cDataSelector       src/core/dataSelector.cpp:296-366 (elementMode=1)    */
  OSM_B200_C_HARMONICS,          /* cHarmonics          src/lld/harmonics.cpp:743-935 (GeMAPS switch set)    */
  OSM_B200_C_LSP,                /* cLsp                src/lld/lsp.cpp:113-313 (on a stand-alone cLpc level) */
  OSM_B200_C_TONESPEC,           /* cTonespec           src/lld/tonespec.cpp:89-441 (on a cFFTmagphase magnitude level) */
  OSM_B200_C_CHROMA,             /* cChroma             src/lld/chroma.cpp:46-117 (on a cTonespec or cTonefilt level) */
  OSM_B200_C_TONEFILT,           /* cTonefilt           src/lld/tonefilt.cpp:65-259 (on the cWaveSource level) */
  OSM_B200_C_CENS,               /* cCens               src/lld/cens.cpp:64-222 (on a cChroma level)      */
  OSM_B200_C_COUNT_
} osm_b200_component_type;

/* window functions, cWindower.winFunc (src/dspcore/windower.cpp:60-80) */
typedef enum {
  OSM_B200_WIN_RECTANGLE = 0, OSM_B200_WIN_HANNING, OSM_B200_WIN_HAMMING, OSM_B200_WIN_GAUSS,
  OSM_B200_WIN_SINE, OSM_B200_WIN_TRIANGLE, OSM_B200_WIN_BARTLETT,
  OSM_B200_WIN_BLACKMAN, OSM_B200_WIN_BLACKHARR, OSM_B200_WIN_BARTHANN, OSM_B200_WIN_LANCZOS
} osm_b200_winfunc;

/* sample formats of the PCM buffers handed to osm_b200_plan_run_*: what smilePcm_convertSamples / smilePcm_convertFloatSamples accept
 * (src/smileutil/smileUtil.c:2500-2680), interleaved channels, little endian.  A sample frame = nChannels samples.
 *   S16    int16                      x / 32767                       (read by the kernels directly)
 *   F32    IEEE float                 x
 *   S8     int8 (the reference reads 8-bit WAV data as SIGNED bytes)  x / 127
 *   S24    3 bytes per sample         x / (32767 * 256)
 *   S24_32 24 valid bits in 4 bytes   (x & 0xFFFFFF) / (32767 * 256)  -- no sign extension, as the reference (smileUtil.c:2559)
 *   S32    int32                      x / 2147483647
 * With several channels the reference sums the float samples in channel order and divides by the channel count first
 * (monoMixdown).  Every format but S16 is converted on the device by one pre-pass (pcm_convert_kernel) into mono floats. */
typedef enum { OSM_B200_PCM_S16 = 0, OSM_B200_PCM_F32 = 1, OSM_B200_PCM_S8 = 2, OSM_B200_PCM_S24 = 3, OSM_B200_PCM_S24_32 = 4,
               OSM_B200_PCM_S32 = 5 } osm_b200_pcm_format;

/* ---- per-type parameter blocks.  Field names and defaults = the reference's config
 * schema (SURVEY.md Appendix A); osm_b200_component_defaults() fills the defaults. ---- */

typedef struct {            /* cWaveSource (src/iocore/waveSource.cpp) */
  double  sampleRate;       /* Hz, from the WAV header                                   */
  int32_t nChannels;        /* channels in the PCM buffer                                */
  int32_t monoMixdown;      /* 1: average channels (config/shared/standard_wave_input.conf.inc:19) */
  int32_t format;           /* osm_b200_pcm_format                                       */
  char    outFieldName[OSM_B200_NAME_LEN]; /* "pcm" (standard_wave_input.conf.inc:20)     */
} osm_b200_wavesource;

typedef struct {            /* cFramer */
  double  frameSize;        /* 0.025 */
  double  frameStep;        /* 0 = frameSize */
  /* sampling centre (core/winToVecProcessor.cpp:461-508): frameCenterSpecial, when set, overrides the other two;
   * frameCenterFrames, when set, overrides frameCenter */
  int32_t frameCenterSpecial;     /* osm_b200_frame_center, OSM_B200_CENTER_UNSET */
  int32_t frameCenterFramesSet;   /* 0 */
  double  frameCenter;            /* 0 (seconds) */
  int32_t frameCenterFrames;      /* 0 (samples), read when frameCenterFramesSet */
  int32_t noPostEOIprocessing;    /* 1 */
} osm_b200_framer;

/* cFramer.frameCenterSpecial: the first two letters of the value, case-insensitive ("mi" / "ce" = frame centre,
 * "ri" = frame end, anything else = frame start) */
typedef enum { OSM_B200_CENTER_UNSET = 0, OSM_B200_CENTER_LEFT = 1, OSM_B200_CENTER_MID = 2, OSM_B200_CENTER_RIGHT = 3 } osm_b200_frame_center;

typedef struct { double k; int32_t de; } osm_b200_vectorpreemphasis;  /* 0.97, 0 */

typedef struct {            /* cWindower */
  int32_t winFunc;          /* osm_b200_winfunc, default Hanning */
  double  gain, offset, sigma;    /* 1, 0, 0.4 */
  /* Blackman / Blackman-Harris / Bartlett-Hann coefficients as the reference resolves them (dspcore/windower.cpp:83-113):
   * Blackman (1-alpha)/2, 1/2, alpha/2 with alpha = 0.16 unless alpha0..2 are all set; Blackman-Harris 0.35875, 0.48829, 0.14128,
   * 0.01168; Bartlett-Hann 0.62, 0.48, 0.38.  osm_b200_component_defaults() fills the Blackman values. */
  double  alpha0, alpha1, alpha2, alpha3;
  double  fade;             /* 0: fraction (<= 0.5) of the window faded in / out with a half raised cosine (:201-208) */
  int32_t squareRoot;       /* 0; 1 = square root of the window function (:178-188) */
} osm_b200_windower;

typedef struct { int32_t inverse; int32_t zeroPadSymmetric; } osm_b200_transformfft; /* 0, 1 */

typedef struct {            /* cFFTmagphase */
  int32_t magnitude, phase, normalise, power, dBpsd;  /* 1,0,0,0,0 */
  /* normalise / power / dBpsd (dspcore/fftmagphase.cpp:223-255) are served where the level is the OUTPUT level (spectrogram.conf);
   * the consumers on the path (cMelspec, cSpectral, cAcf, cSpecScale ...) read the plain magnitude */
  double  dBpnorm, mindBp;  /* 90.302, -102.0 (mindBp is raised to dBpnorm - 120, :95-98) */
} osm_b200_fftmagphase;

/* cMelspec.specScale (lldcore/melspec.cpp:100-135; smileutil/smileUtil.c:1097-1204): the frequency scale the band centres are
 * equidistant on.  Only read when htkcompatible = 0 (HTK compatibility forces mel). */
typedef enum { OSM_B200_SCALE_MEL = 0, OSM_B200_SCALE_BARK, OSM_B200_SCALE_BARK_SPEEX, OSM_B200_SCALE_BARK_SCHROED, OSM_B200_SCALE_SEMITONE,
               OSM_B200_SCALE_LINEAR, OSM_B200_SCALE_LOG } osm_b200_specscale_kind;

typedef struct {            /* cMelspec */
  int32_t nBands;           /* 26 */
  double  lofreq, hifreq;   /* 20, 8000 */
  int32_t usePower;         /* 0 */
  int32_t htkcompatible;    /* 1 */
  int32_t specScale;        /* OSM_B200_SCALE_MEL */
  double  scaleParam;       /* semitone: firstNote (27.5); log: logScaleBase (2.0, values <= 0 or == 1 become 2.0) */
} osm_b200_melspec;

typedef struct {            /* cMfcc */
  int32_t firstMfcc, lastMfcc;  /* 1, 12 */
  double  melfloor;         /* 1e-8 */
  int32_t doLog;            /* 1 */
  double  cepLifter;        /* 22 */
  int32_t htkcompatible;    /* 1 */
} osm_b200_mfcc;

typedef struct {            /* cPlp */
  int32_t lpOrder;          /* 5 */
  int32_t nCeps;            /* -1 */
  int32_t firstCC, lastCC;  /* 1, -1 */
  int32_t doLog, doAud, RASTA, newRASTA, doInvLog, doIDFT, doLP, doLpToCeps; /* 1,1,0,0,1,1,1,1 */
  double  rastaUpperCutoff, rastaLowerCutoff;  /* 29, 1 */
  double  cepLifter;        /* 0 */
  double  compression;      /* 0.33 */
  double  melfloor;         /* 9.3e-10 */
  int32_t htkcompatible;    /* 1 */
} osm_b200_plp;

typedef struct {            /* cSpectral (subset of switches used by eGeMAPS / ComParE) */
  int32_t squareInput;      /* 1 */
  int32_t nBands;  double bandLo[OSM_B200_MAX_LIST], bandHi[OSM_B200_MAX_LIST];   /* bands[] */
  int32_t nSlopes; double slopeLo[OSM_B200_MAX_LIST], slopeHi[OSM_B200_MAX_LIST]; /* slopes[] */
  int32_t nRollOff; double rollOff[OSM_B200_MAX_LIST];                            /* rollOff[] */
  int32_t flux, centroid, maxPos, minPos, entropy, standardDeviation, variance, skewness,
          kurtosis, slope, alphaRatio, hammarbergIndex, sharpness, harmonicity, flatness;
  int32_t normBandEnergies, buggyRollOff, oldSlopeScale, useLogSpectrum;
  double  freqRangeLo, freqRangeHi;  /* freqRange = lo-hi, 0-0 = full */
  double  specFloor;        /* 1e-7 */
  int32_t logFlatness;      /* 0 */
} osm_b200_spectral;

typedef struct {            /* cEnergy */
  int32_t htkcompatible, rms, energy2, log;  /* 0,1,0,1 */
  double  escaleLog, escaleRms, escaleSquare, ebiasLog, ebiasRms, ebiasSquare; /* 1,1,1,0,0,0 */
} osm_b200_energy;

typedef struct { int32_t zcr, mcr, amax, maxmin, dc; } osm_b200_mzcr; /* 1,1,1,1,0 */

typedef struct {            /* cAcf */
  int32_t usePower, cepstrum, inverse, cosLifterCepstrum, expBeforeAbs, symmetricData,
          acfCepsNormOutput, oldCompatCepstrum, absCepstrum; /* 1,0,0,0,1,1,1,0,0 */
} osm_b200_acf;

typedef struct {            /* cPitchACF */
  double  maxPitch;         /* 500 */
  int32_t voiceProb, voiceQual, HNR, HNRdB, linHNR, F0, F0raw, F0env; /* 1,0,0,0,0,0,0,0 */
  double  voicingCutoff;    /* 0.55 */
} osm_b200_pitchacf;

typedef struct {            /* cDeltaRegression */
  int32_t deltawin;         /* 2 */
  int32_t absOutput, halfWaveRect, onlyInSegments, zeroSegBound, relativeDelta; /* 0,0,0,1,0 */
} osm_b200_deltaregression;

typedef struct { int32_t smaWin; int32_t noZeroSma; } osm_b200_contoursmoother; /* 3, 0 */

typedef struct {            /* cVectorOperation, n -> 1 operations only (src/other/vectorOperation.cpp:475-481) */
  int32_t operation;        /* 0 = ll1: sum of the input vector / number of elements */
  char    nameBase[OSM_B200_NAME_LEN]; /* replaces the input field name when set (:246-248) */
} osm_b200_vectoroperation;

/* cVectorConcat: the cVectorProcessor field selection (src/core/vectorProcessor.cpp:37-39,196-243).
 * processArrayFields = 1 passes array fields only (single-element fields are dropped unless
 * includeSingleElementFields = 1); processArrayFields = 0 passes the whole frame, field names kept. */
typedef struct { int32_t processArrayFields, includeSingleElementFields; } osm_b200_vectorconcat; /* 1, 0 */

/* cFullinputMean: per-utterance mean subtraction (cepstral mean subtraction of the *_Z configurations).
 * Only the default mode is supported: arithmetic mean, single EOI loop (src/dspcore/fullinputMean.cpp:484-548) */
typedef struct { int32_t mvn, meanNorm /* 0 = amean */, symmSubtract, subtractClipToZero, specEnorm, htkLogEnorm, excludeZeros, multiLoopMode; } osm_b200_fullinputmean;

typedef struct { int32_t intensity, loudness; } osm_b200_intensity;   /* cIntensity: 1, 0 */

/* ---- sub-harmonic-summation pitch chain (SURVEY.md 8f-1) ---- */
typedef struct {            /* cSpecScale: scale=octave, sourceScale=lin, interpMethod=spline only */
  int32_t scaleOctave, sourceLin, splineInterp;  /* 1 when the section selects exactly these (else the plan is rejected) */
  double  minF, maxF;       /* 25, -1 */
  int32_t nPointsTarget;    /* 0 = number of magnitude bins */
  int32_t specSmooth, specEnhance, auditoryWeighting;  /* 0, 0, 0 */
} osm_b200_specscale;

typedef struct {            /* cPitchShs (cPitchBase options + its own) */
  double  maxPitch, minPitch;   /* 620, 52 */
  int32_t nCandidates;      /* 3 */
  int32_t scores, voicing, F0C1, voicingC1, F0raw, voicingClip;  /* 1,1,0,0,0,0 */
  double  voicingCutoff;    /* 0.70 */
  int32_t octaveCorrection; /* 0 */
  int32_t nHarmonics;       /* 15 */
  double  compressionFactor;/* 0.85 */
  int32_t greedyPeakAlgo;   /* 0 */
  double  lfCut;            /* 0 */
} osm_b200_pitchshs;

typedef struct {            /* cPitchSmootherViterbi */
  int32_t bufferLength;     /* 30 */
  int32_t F0final, F0finalLog, F0finalEnv, F0finalEnvLog, voicingFinalClipped, voicingFinalUnclipped; /* 1,0,0,0,0,0 */
  int32_t F0raw, voicingC1, voicingClip;  /* 0,0,0 (copies of input fields: not supported when set) */
  double  wLocal, wTvv, wTvvd, wTvuv, wThr, wRange, wTuu;  /* 2, 10, 5, 10, 4, 1, 0 */
} osm_b200_pitchsmootherviterbi;

typedef struct {            /* cValbasedSelector: reader.dmLevel = <selector level>;<data level> */
  double  threshold;        /* 1.0 */
  int32_t idx, invert, allowEqual, removeIdx, zeroVec, adaptiveThreshold;  /* 0,0,0,0,0,0 */
  double  outputVal;        /* 0 */
} osm_b200_valbasedselector;

typedef struct {            /* cPitchJitter: reader.dmLevel = wave level, F0reader.dmLevel = pitch level */
  char    F0reader_dmLevel[OSM_B200_NAME_LEN];
  char    F0field[OSM_B200_NAME_LEN];   /* "F0final" */
  double  searchRangeRel;   /* 0.10 */
  int32_t jitterLocal, jitterDDP, jitterLocalEnv, jitterDDPEnv;           /* 0,0,0,0 */
  int32_t shimmerLocal, shimmerLocalDB, shimmerLocalEnv, shimmerLocalDBEnv; /* 0,0,0,0 */
  int32_t harmonicERMS, noiseERMS, linearHNR, logHNR;                     /* 0,0,0,0 */
  double  lgHNRfloor;       /* -100 */
  int32_t shimmerUseRmsAmplitude, minNumPeriods;  /* 0, 2 */
  double  minCC;            /* 0.5 */
  int32_t refinedF0, sourceQualityRange, sourceQualityMean;  /* 0,0,0 */
  int32_t usePeakToPeakPeriodLength, useBrokenJitterThresh, onlyVoiced;  /* 0, 1, 0 */
} osm_b200_pitchjitter;

typedef struct {            /* cSpecResample: reads a cTransformFFT level (complex spectrum) */
  double  targetFs;         /* 16000 */
  double  resampleRatio;    /* <= 0: derive from targetFs (the reference's "not set") */
} osm_b200_specresample;

typedef struct {            /* cLpc */
  int32_t method;           /* 0 = acf (the only supported one), 1 = burg */
  int32_t p;                /* 8 */
  int32_t saveLPCoeff, lpGain, saveRefCoeff, residual, residualGainScale, forwardFilter, lpSpectrum;  /* 1,0,0,0,0,0,0 */
} osm_b200_lpc;

typedef struct {            /* cFormantLpc */
  int32_t nFormants;        /* -1 = p - 1 */
  int32_t saveFormants, saveIntensity, saveNumberOfValidFormants, saveBandwidths;  /* 1,0,0,0 */
  double  minF, maxF;       /* 50, 5500 */
  int32_t useLpSpec, medianFilter, octaveCorrection;   /* 0,0,0 (only these values are supported) */
} osm_b200_formantlpc;

typedef struct {            /* cDataSelector, elementMode = 1: exact element names, output in the order of `selected` */
  int32_t nSelected;
  int32_t elementMode;      /* 1 */
  char    selected[OSM_B200_MAX_SELECTED][OSM_B200_NAME_LEN];
  char    newNames[OSM_B200_MAX_SELECTED][OSM_B200_NAME_LEN];   /* "" = keep the name (+ "_" nameAppend) */
} osm_b200_dataselector;

typedef struct {            /* cHarmonics: reader.dmLevel = <pitch level>;<formant level>;<cFFTmagphase level> (any order) */
  char    f0ElementName[OSM_B200_NAME_LEN];             /* "F0final" */
  char    magSpecFieldName[OSM_B200_NAME_LEN];          /* "pcm_fftMag" */
  char    formantFrequencyFieldName[OSM_B200_NAME_LEN]; /* "" */
  char    formantBandwidthFieldName[OSM_B200_NAME_LEN]; /* "" */
  int32_t f0ElementNameIsFull, magSpecFieldNameIsFull, formantFrequencyFieldNameIsFull, formantBandwidthFieldNameIsFull; /* 1,0,1,1 */
  int32_t nHarmonics, firstHarmonicMagnitude, nHarmonicMagnitudes, outputLogRelMagnitudes, outputLinearMagnitudes;       /* 100,1,0,1,0 */
  int32_t nHarmonicDifferences;                          /* entries of harmonicDifferences */
  char    harmonicDifferences[4][16];                    /* "H1-H2", "H1-A3", ... */
  int32_t harmonicDifferencesLog, harmonicDifferencesRatioLinear;    /* 1, 0 */
  int32_t formantAmplitudes, formantAmplitudesLinear, formantAmplitudesLogRel, formantAmplitudesStart, formantAmplitudesEnd; /* 0,0,1,1,-1 */
  int32_t computeAcfHnrLogdB, computeAcfHnrLinear;       /* 0, 0 */
  double  logRelValueFloorUnvoiced;                      /* -201 */
} osm_b200_harmonics;

typedef struct {            /* cLsp: reads a cLpc level (its lpcCoeff field) */
  int32_t processArrayFields;   /* 1 (the cVectorProcessor default); only 0 is supported */
} osm_b200_lsp;

/* cTonespec.filterType (lld/tonespec.cpp:107-111) */
typedef enum { OSM_B200_TONE_GAU = 0, OSM_B200_TONE_TRI, OSM_B200_TONE_TRP, OSM_B200_TONE_REC } osm_b200_tone_filter;

typedef struct {            /* cTonespec (lld/tonespec.cpp:46-52) */
  int32_t nOctaves;         /* 6 */
  double  firstNote;        /* 55 Hz */
  int32_t filterType;       /* osm_b200_tone_filter, OSM_B200_TONE_GAU */
  int32_t usePower;         /* 0 */
  int32_t dbA;              /* 1 */
} osm_b200_tonespec;

typedef struct {            /* cChroma (lld/chroma.cpp:46-49) */
  int32_t octaveSize;       /* 12 */
  double  silThresh;        /* 0.001 */
} osm_b200_chroma;

typedef struct {            /* cTonefilt (lld/tonefilt.cpp:35-41) */
  int32_t nNotes;           /* 48 */
  double  firstNote;        /* 55 Hz */
  double  decayF0;          /* 0.9995 */
  double  decayFN;          /* 0.998 */
  double  outputPeriod;     /* 0.1 s */
} osm_b200_tonefilt;

typedef struct {            /* cCens (lld/cens.cpp:40-48) */
  int32_t window;           /* OSM_B200_WIN_HANNING; HAMMING or BARTLETT (a window name the reference does not know is Hanning) */
  int32_t winlength;        /* 41 taps; values < 1 become 1 */
  int32_t l2norm;           /* 1 */
  int32_t downsampleRatio;  /* 10; values < 1 become 1.  Scales the level's period only: every input row is an output row */
  double  winlength_sec;    /* 0.41; used only when winlength_secSet (not supported: the reference crashes when it is set) */
  int32_t winlength_secSet;
} osm_b200_cens;

/* one `[name:cType]` section */
typedef struct {
  int32_t type;                                  /* osm_b200_component_type */
  char    name[OSM_B200_NAME_LEN];               /* instance name (diagnostics only) */
  int32_t n_inputs;                              /* reader.dmLevel = a;b;c */
  char    reader_dmLevel[OSM_B200_MAX_INPUTS][OSM_B200_NAME_LEN];
  char    writer_dmLevel[OSM_B200_NAME_LEN];
  /* cDataProcessor naming fields (src/core/dataProcessor.cpp:41-48,249-325).  nameAppend ""
   * selects the type's default ("mfcc", "de", "sma", "fftMag", ...); copyInputName default 1. */
  char    nameAppend[OSM_B200_NAME_LEN];
  int32_t copyInputName;
  union {
    osm_b200_wavesource wavesource;
    osm_b200_framer framer;
    osm_b200_vectorpreemphasis vectorpreemphasis;
    osm_b200_windower windower;
    osm_b200_transformfft transformfft;
    osm_b200_fftmagphase fftmagphase;
    osm_b200_melspec melspec;
    osm_b200_mfcc mfcc;
    osm_b200_plp plp;
    osm_b200_spectral spectral;
    osm_b200_energy energy;
    osm_b200_mzcr mzcr;
    osm_b200_acf acf;
    osm_b200_pitchacf pitchacf;
    osm_b200_deltaregression deltaregression;
    osm_b200_contoursmoother contoursmoother;
    osm_b200_vectoroperation vectoroperation;
    osm_b200_vectorconcat vectorconcat;
    osm_b200_fullinputmean fullinputmean;
    osm_b200_intensity intensity;
    osm_b200_specscale specscale;
    osm_b200_pitchshs pitchshs;
    osm_b200_pitchsmootherviterbi pitchsmootherviterbi;
    osm_b200_valbasedselector valbasedselector;
    osm_b200_pitchjitter pitchjitter;
    osm_b200_specresample specresample;
    osm_b200_lpc lpc;
    osm_b200_formantlpc formantlpc;
    osm_b200_dataselector dataselector;
    osm_b200_harmonics harmonics;
    osm_b200_lsp lsp;
    osm_b200_tonespec tonespec;
    osm_b200_chroma chroma;
    osm_b200_tonefilt tonefilt;
    osm_b200_cens cens;
  } u;
} osm_b200_component;

typedef struct osm_b200_plan osm_b200_plan;

/* ---- library ---- */
OSM_B200_API int32_t     osm_b200_abi_version(void);
/* sizeof(osm_b200_component) as compiled into the library: bindings in other languages
 * (ctypes, cgo, JNI) assert it against their own mirror of the struct */
OSM_B200_API int32_t     osm_b200_sizeof_component(void);
OSM_B200_API const char *osm_b200_last_error(void);
/* number of usable CUDA devices (0 = none; compute entry points will then fail) */
OSM_B200_API int32_t     osm_b200_device_count(void);

/* fill `c` with the reference's defaults for `type` (everything else zeroed) */
OSM_B200_API osm_b200_status osm_b200_component_defaults(int32_t type, osm_b200_component *c);

/* ---- plan ---- */
/* Compile the component graph that produces `output_level` into a fused plan bound to CUDA
 * device `device`.  The graph must contain exactly one OSM_B200_C_WAVESOURCE.
 * device < 0 creates a description-only plan (element names, geometry, frame-count rules)
 * without touching CUDA; its run_* calls fail with OSM_B200_ERR_CUDA. */
OSM_B200_API osm_b200_status osm_b200_plan_create(const osm_b200_component *comps, int32_t n_comps,
                                     const char *output_level, int32_t device,
                                     osm_b200_plan **plan);
OSM_B200_API void            osm_b200_plan_destroy(osm_b200_plan *plan);

/* output row width (elements of the output level) and names of its elements, formed by the
 * reference's naming rules (src/core/dataProcessor.cpp:249-325), e.g. "pcm_fftMag_mfcc[1]" */
OSM_B200_API int32_t     osm_b200_plan_num_elements(const osm_b200_plan *plan);
OSM_B200_API const char *osm_b200_plan_element_name(const osm_b200_plan *plan, int32_t idx);
/* period of the output level in seconds: cFramer.frameStep, cTonefilt.outputPeriod, and for a cCens level (and the levels behind
 * it) its input's period times cCens.downsampleRatio (lld/cens.cpp:107-114).  It is the HTK sample period and the seconds unit of
 * cFunctionals; it is not the spacing of a cCens level's row time stamps (osm_b200_plan_row_time). */
OSM_B200_API double      osm_b200_plan_frame_period(const osm_b200_plan *plan);
/* time stamp of row r of the output level: r * cFramer.frameStep for framer levels; (double)(r * P) / fs, the time of the row's
 * first sample, for a cTonefilt level (blocks of P samples; its period outputPeriod need not be P / fs).  A cCens level keeps the
 * time stamps of its chroma rows (core/vectorProcessor.cpp:308): downsampleRatio scales the period only, not these times. */
OSM_B200_API double      osm_b200_plan_row_time(const osm_b200_plan *plan, int64_t row);
/* geometry resolved at plan time */
OSM_B200_API int32_t     osm_b200_plan_frame_size_samples(const osm_b200_plan *plan);
OSM_B200_API int32_t     osm_b200_plan_frame_step_samples(const osm_b200_plan *plan);
OSM_B200_API int32_t     osm_b200_plan_fft_size(const osm_b200_plan *plan);

/* rows the reference would emit on the output level for an utterance of n sample frames
 * (bit-exact integer rule: framer with noPostEOIprocessing, window processors' EOI padding,
 * concat = min over inputs; SURVEY.md 8a-2/13/15) */
OSM_B200_API int64_t     osm_b200_plan_num_frames(const osm_b200_plan *plan, int64_t n_sample_frames);

/* rows of the output level that exist when a full-input reader (cFunctionals, frameMode = full) ticks for the first time at
 * end of input: the window processors of the level have each appended one frame by then, not yet all of them
 * (blocksize 1, core/windowProcessor.cpp:167-230); that is the contour the reference's functionals summarise */
/* the window table cWindower multiplies a frame of n samples with (dspcore/windower.cpp:159-217: window function, squareRoot,
 * fade, gain), as float: what osm_b200_plan_create stages for the kernels (bindings, tests) */
OSM_B200_API osm_b200_status osm_b200_window_table(const osm_b200_windower *cfg, int32_t n, float *out);
/* the tables cTonespec builds for a magnitude level of n_bins bins and frame length frame_size_sec (after cTransformFFT's
 * rescale, so 1 / frame_size_sec = fs / N_fft): note frequencies pitch_class_freq[nNotes + 2], bin_key[n_bins] (nearest note of
 * every bin), bin_count[nNotes + 2] (bins per note over firstBin .. lastBin), filter_map[n_bins] (filter weight times the
 * shifted dB(A) weight, zero outside firstBin .. lastBin) and fl_bin[2] = firstBin, lastBin (lld/tonespec.cpp:147-367),
 * as osm_b200_plan_create stages them for the kernels (bindings, tests).  nNotes = 12 * cfg->nOctaves. */
OSM_B200_API osm_b200_status osm_b200_tone_tables(const osm_b200_tonespec *cfg, int32_t n_bins, double frame_size_sec,
                                                  float *pitch_class_freq, int32_t *bin_key, int32_t *bin_count,
                                                  float *filter_map, int32_t *fl_bin);
OSM_B200_API int64_t     osm_b200_plan_num_frames_first_eoi(const osm_b200_plan *plan, int64_t n_sample_frames);
/* the same for levels behind the SHS pitch chain, whose length at that moment depends on the data: viterbi_frames = frames the
 * cPitchSmootherViterbi level held when end of input was raised (osm_b200_plan_copy_seq_lag after a run; < 0: not known, the
 * static frame count is assumed) */
OSM_B200_API int64_t     osm_b200_plan_num_frames_first_eoi_v(const osm_b200_plan *plan, int64_t n_sample_frames, int64_t viterbi_frames);
/* per utterance of the last run: frames of the Viterbi level before the end-of-input flush (-1 when the plan has no SHS pitch chain);
 * synchronises the device */
OSM_B200_API osm_b200_status osm_b200_plan_copy_seq_lag(osm_b200_plan *plan, int32_t *out, int32_t n_utt);
/* the same values for a run enqueued on `stream` (cudaStream_t): waits for that stream only, never for the whole device */
OSM_B200_API osm_b200_status osm_b200_plan_copy_seq_lag_stream(osm_b200_plan *plan, int32_t *out, int32_t n_utt, void *stream);

/* number of distinct time stamps of those rows: frames of the level the first output field comes from, before its
 * window processors.  The rows a window processor appends at the end of input repeat the time stamp of the last
 * real frame (their tmeta is a copy, src/core/dataMemoryLevel.cpp:1698-1708), so row r of a sink's file carries the
 * time min(r, n - 1) * period */
OSM_B200_API int64_t     osm_b200_plan_num_time_frames(const osm_b200_plan *plan, int64_t n_sample_frames);

/* exclusive prefix sums over utterances: frame_offsets[0..n_utt] (host arrays) */
OSM_B200_API osm_b200_status osm_b200_plan_frame_offsets(const osm_b200_plan *plan,
                                            const int64_t *utt_offsets, int32_t n_utt,
                                            int64_t *frame_offsets);

/* ---- execution ---- */
/* Device-resident batch.  d_pcm / d_out are device pointers; utt_offsets / frame_offsets are
 * HOST arrays of n_utt+1 entries (frame_offsets as returned by osm_b200_plan_frame_offsets).
 * Asynchronous on `stream` (a cudaStream_t, NULL = default stream). */
OSM_B200_API osm_b200_status osm_b200_plan_run_device(osm_b200_plan *plan, const void *d_pcm,
                                         const int64_t *utt_offsets, int32_t n_utt,
                                         const int64_t *frame_offsets, float *d_out,
                                         void *stream);

/* Padded device batch, the layout a torch tensor [n_utt][n_channels][stride] has: channel-planar, utterance u's samples at
 * d_pcm + u * n_channels * stride, lengths[u] <= stride sample frames (HOST array of n_utt entries; the padding is never read).
 * Samples are int16 or float32 as the plan's cWaveSource.format says (OSM_B200_PCM_S16 / OSM_B200_PCM_F32; other formats are
 * refused), its channel count is the plan's.  One kernel (pcm_pack_kernel) re-lays the batch out, without arithmetic, into a
 * plan-owned buffer in the packed interleaved layout of osm_b200_plan_run_device, which then runs on it: rows are those of the
 * same samples packed.  frame_offsets as returned by osm_b200_plan_frame_offsets for the offsets the lengths add up to (may be
 * NULL).  Asynchronous on `stream`; like run_device, the plan's buffers are reused by its next run. */
OSM_B200_API osm_b200_status osm_b200_plan_run_device_padded(osm_b200_plan *plan, const void *d_pcm, int64_t stride,
                                                             const int64_t *lengths, int32_t n_utt,
                                                             const int64_t *frame_offsets, float *d_out, void *stream);

/* Host buffers: copies PCM to the device, runs, copies the rows back into `out`
 * (frame_offsets[n_utt] * num_elements floats) and synchronises. */
OSM_B200_API osm_b200_status osm_b200_plan_run_host(osm_b200_plan *plan, const void *pcm,
                                       const int64_t *utt_offsets, int32_t n_utt,
                                       const int64_t *frame_offsets, float *out);

/* like run_host, but the rows stay in HBM: *d_rows = the plan's own device row buffer [rows][num_elements], valid until
 * the plan's next run (hand-over to osm_b200_functionals_run_device, include/osm_b200_functionals.h) */
OSM_B200_API osm_b200_status osm_b200_plan_run_host_resident(osm_b200_plan *plan, const void *pcm,
                                            const int64_t *utt_offsets, int32_t n_utt,
                                            const int64_t *frame_offsets, const float **d_rows);
/* bytes of one sample frame of the plan's input (nChannels * bytes per sample of cWaveSource.format) */
OSM_B200_API int32_t     osm_b200_plan_sample_frame_bytes(const osm_b200_plan *plan);
/* number of CUDA kernels the last run_* call launched (for bench.py's gpu_launches) */
OSM_B200_API int32_t     osm_b200_plan_last_launch_count(const osm_b200_plan *plan);
/* Device-side condition flags of the runs since the last call (synchronises the device, then clears them).
 * bit 0: a cPitchJitter frame left the supported geometry (wave window past the end of the utterance or beyond the
 * kernel's workspace) and its row was zeroed.  osm_b200_plan_run_host checks this itself and fails with
 * OSM_B200_ERR_UNSUPPORTED; callers of the asynchronous osm_b200_plan_run_device ask here after their own sync. */
OSM_B200_API int32_t     osm_b200_plan_take_device_flags(osm_b200_plan *plan);
/* the same condition for a run enqueued on `stream`, as run_host reports it: OSM_B200_ERR_UNSUPPORTED (and the flag cleared)
 * when it was raised.  Waits for `stream` only, and only when the plan has a cPitchJitter op: otherwise returns at once. */
OSM_B200_API osm_b200_status osm_b200_plan_check_device_flags(osm_b200_plan *plan, void *stream);
/* device time in ms of the fused LLD kernel(s) of the last run_* call, measured with CUDA
 * events on the run's stream; blocks until the run has finished.  <0 if unavailable. */
OSM_B200_API float       osm_b200_plan_last_kernel_ms(osm_b200_plan *plan);
/* the same split per kernel: *lld_ms = the fused per-frame kernel, *post_ms = the temporal
 * (delta / smoothing) kernel, 0 if none was launched.  Either pointer may be NULL. */
OSM_B200_API osm_b200_status osm_b200_plan_last_kernel_times(osm_b200_plan *plan, float *lld_ms,
                                                             float *post_ms);

/* Per-kernel profiling of run_device (measurement aid, bench.py): when on, the auxiliary stream is not used and a CUDA
 * event follows every kernel launch; after a run, entry idx names the idx-th launch of the step and its device time in ms. */
OSM_B200_API void            osm_b200_plan_set_profiling(osm_b200_plan *plan, int32_t on);
OSM_B200_API int32_t         osm_b200_plan_profile_count(osm_b200_plan *plan);
OSM_B200_API osm_b200_status osm_b200_plan_profile_entry(osm_b200_plan *plan, int32_t idx, const char **name, float *ms);

/* The last per-frame (LLD) kernel launch of the last run_* call: *kernel = static name of the instance, e.g.
 * "lld512_kernel<13>" or "lld_kernel<1024,8,256,1,VEC2,GEN>" (NULL when the run launched none), *grid = CTAs,
 * *n_chunks = chunks (work units) of that launch.  run_host may launch once per pipeline piece: the last piece counts.
 * Any pointer may be NULL. */
OSM_B200_API osm_b200_status osm_b200_plan_last_lld_launch(const osm_b200_plan *plan, const char **kernel, int32_t *grid,
                                                           int64_t *n_chunks);

#ifdef __cplusplus
}
#endif
#endif /* OSM_B200_H */
