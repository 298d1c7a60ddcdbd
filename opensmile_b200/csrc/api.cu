// api.cu -- the C ABI of libosm_b200.so (include/osm_b200.h): plan objects, device tables,
// batch bookkeeping (tile lists, row offsets) and kernel launches.  No CPU fallback: every
// compute entry point fails with OSM_B200_ERR_CUDA when no device is usable.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "chunk_schedule.hpp"
#include "cuda_owned.hpp"
#include "kernels.cuh"
#include "plan.hpp"
#include "tonefilt_math.cuh"

using namespace osm;

namespace {
thread_local std::string g_err;
}
// shared with the other translation units of the library (functionals.cu): the message osm_b200_last_error() returns
namespace osm { osm_b200_status set_last_error(osm_b200_status st, const std::string &msg) { g_err = msg; return st; } }

namespace {

osm_b200_status fail(osm_b200_status st, const std::string &msg) { return osm::set_last_error(st, msg); }

// ---- input formats (cWaveSource.format) ----
int sample_bytes(int format)
{
  switch (format) {
    case OSM_B200_PCM_S8: return 1;
    case OSM_B200_PCM_S16: return 2;
    case OSM_B200_PCM_S24: return 3;
    default: return 4;                 // F32, S24_32, S32
  }
}
// channel count the kernels see: 16-bit input is read in place; every other format is pre-converted to mono floats, whose 4-byte
// sample frame the kernels address as "two int16 per frame" (LldParams::pcmF32)
int kernel_nchan(const FrontEnd &fe) { return fe.format == OSM_B200_PCM_S16 ? fe.nChan : 2; }

// smilePcm_convertSamples / smilePcm_convertFloatSamples with monoMixdown (smileutil/smileUtil.c:2518-2580, 2651-2661): the channel
// values are converted to float and summed in channel order starting from 0.0f, the sum is divided by the channel count, then by
// the format's full scale -- two IEEE divisions, exactly the reference's statement.  One thread per sample frame.
__global__ void __launch_bounds__(256) pcm_convert_kernel(const unsigned char *in, int format, int nChan, long long nFrames, float *out)
{
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nFrames) return;
  float tmp = 0.0f;
  float scale = 1.0f;
  switch (format) {
    case OSM_B200_PCM_S8: {
      const signed char *b = reinterpret_cast<const signed char *>(in) + i * nChan;
      for (int c = 0; c < nChan; c++) tmp = __fadd_rn(tmp, (float)b[c]);
      scale = 127.0f;
      break;
    }
    case OSM_B200_PCM_S24: {
      const unsigned char *b = in + i * nChan * 3;
      for (int c = 0; c < nChan; c++) {                                             // :2543-2552 (byte assembly, arithmetic shift)
        const unsigned int is = ((unsigned int)b[3 * c] << 8) | ((unsigned int)b[3 * c + 1] << 16) | ((unsigned int)b[3 * c + 2] << 24);
        tmp = __fadd_rn(tmp, (float)((int)is >> 8));
      }
      scale = 8388352.0f;                                                           // (float)(32767.0 * 256.0)
      break;
    }
    case OSM_B200_PCM_S24_32: {
      const int *b = reinterpret_cast<const int *>(in) + i * nChan;
      for (int c = 0; c < nChan; c++) tmp = __fadd_rn(tmp, (float)(b[c] & 0xFFFFFF));   // :2559 (no sign extension)
      scale = 8388352.0f;
      break;
    }
    case OSM_B200_PCM_S32: {
      const int *b = reinterpret_cast<const int *>(in) + i * nChan;
      for (int c = 0; c < nChan; c++) tmp = __fadd_rn(tmp, (float)b[c]);
      scale = 2147483648.0f;                                                        // (float)2147483647.0
      break;
    }
    default: {                                                                      // OSM_B200_PCM_F32: no full-scale division (:2658)
      const float *b = reinterpret_cast<const float *>(in) + i * nChan;
      for (int c = 0; c < nChan; c++) tmp = __fadd_rn(tmp, b[c]);
      out[i] = __fdiv_rn(tmp, (float)nChan);
      return;
    }
  }
  out[i] = __fdiv_rn(__fdiv_rn(tmp, (float)nChan), scale);
}

// A padded device batch -- [nUtt][nChan][stride] samples, channel-planar, the layout of a torch tensor -- re-laid out as the packed,
// channel-interleaved batch the plan reads: the first uttOff[u + 1] - uttOff[u] sample frames of utterance u land at sample frame
// uttOff[u].  Samples are moved as 2- or 4-byte words with no arithmetic, so the mixdown and conversion statements stay with the
// kernels behind (pcm_convert_kernel, the int16 sample readers).  Samples past an utterance's length are never read.
// Block (x, y): frames [x * tileF, (x + 1) * tileF) of utterances y, y + gridDim.y, ...  Mono is a straight copy; with several
// channels the tile passes through shared memory ([nChan][tileF]) so that the planar reads and the interleaved writes both coalesce.
constexpr int kPackThreads = 256;
constexpr int kPackMonoFrames = 4096;           // frames per block of a mono batch
constexpr int kPackTileBytes = 16 << 10;        // shared tile of a multi-channel batch
template <typename T>
__global__ void __launch_bounds__(kPackThreads) pcm_pack_kernel(const T *__restrict__ in, long long stride, int nChan, int tileF,
                                                               const long long *__restrict__ uttOff, int nUtt, T *__restrict__ out)
{
  extern __shared__ __align__(16) unsigned char packSmem[];
  T *tile = reinterpret_cast<T *>(packSmem);
  const long long f0 = (long long)blockIdx.x * tileF;
  for (int u = blockIdx.y; u < nUtt; u += gridDim.y) {
    const long long o = uttOff[u], len = uttOff[u + 1] - o;
    if (f0 >= len) continue;                                            // the same for every thread of the block
    const int nf = (int)min((long long)tileF, len - f0);
    const T *src = in + (size_t)u * nChan * stride + f0;
    T *dst = out + (size_t)(o + f0) * nChan;
    if (nChan == 1) {
#pragma unroll 4
      for (int t = threadIdx.x; t < nf; t += kPackThreads) dst[t] = src[t];
      continue;
    }
    for (int c = 0; c < nChan; c++)
      for (int t = threadIdx.x; t < nf; t += kPackThreads) tile[c * tileF + t] = src[(size_t)c * stride + t];
    __syncthreads();
    for (int k = threadIdx.x; k < nf * nChan; k += kPackThreads) {
      const int t = k / nChan;
      dst[k] = tile[(k - t * nChan) * tileF + t];
    }
    __syncthreads();                                                    // the tile is refilled for the next utterance
  }
}

}  // namespace


// per-stream runtime state (one framer / FFT chain)
// one lld_kernel launch of a stream: the FFT front end + one band op (or none: magnitude dump only)
struct PassRt {
  LldParams kp;
  DevBuf<unsigned char> dConst;  // constant tables of the pass; kp points into them
  int op = -1;                   // index into PlanDesc::ops, -1 = no band op
  bool rasta = false;            // cPlp with RASTA: kp stops at the band level, tail = the rest of cPlp
  LldParams tail;
  RastaParams rp;
  DevBuf<float> dBand;           // [static rows][nBands]
};

struct StreamRt {
  LldParams kp;                  // pass 0 (the only pass of fused plans)
  std::vector<PassRt> extra;     // passes 1.. (further band ops on the same FFT chain)
  PassRt pass0x;                 // constant tables and RASTA state of pass 0 (kp of pass 0 lives above)
  int tileF = 32;
  bool runLld = false;           // lld_kernel is launched for this stream
  bool forceNarrow = false;
  bool needTiles = false;        // standalone ops read this stream tile by tile
  const float *dWindow = nullptr;   // [frameSize] window floats (time-domain ops)
  std::vector<int32_t> uttChunk0, uttTile0;
  PinBuf<ChunkRef> hChunks; DevBuf<ChunkRef> dChunks; size_t nChunks = 0;   // + one entry whose w0 ends the schedule
  int lldCtas = 1;               // CTAs pass 0's lld instance keeps resident
  int ctaTiles = 1;              // tiles per CTA run of the whole batch (LldParams::ctaTiles)
  PinBuf<OpTile> hTiles; DevBuf<OpTile> dTiles; size_t nTiles = 0;
  DevBuf<float> dMag;
};

struct OpRt {
  int kind = 0, stream = 0;
  int vSrcCol = 0, vN = 0, vOutCol = 0;     // SOP_VECOP
  int magMode = 0; float magN = 1.f, magDbNorm = 0.f, magMinDb = 0.f;   // SOP_MAG: cFFTmagphase normalise / power / dBpsd
  SpectralParams sp;
  TimeOpParams tp;
  AcfPitchParams ap;
  DevBuf<double> dSharpW;
  DevBuf<float2> dTw;
  DevBuf<PitchRaw> dRaw;
  // SHS pitch chain (SOP_PITCH) / cPitchJitter (SOP_JITTER)
  ShsParams shs;
  ViterbiParams vit;
  JitterParams jit;
  HarmonicsParams hrm;                  // SOP_HARMONICS
  DevBuf<double> dCosTab;               // its cos(2 pi m / N) table
  FormantParams fmt;                    // SOP_FORMANT
  LpcParams lpc;                        // SOP_LPC
  DevBuf<float> dFmtD;                  // its resampling table
  DevBuf<unsigned char> dPitchTab;      // spline / interpolation / harmonic tables of the chain
  DevBuf<float> dShs;                   // [static rows][nShsCols] cPitchShs level
  DevBuf<int> dLag;                     // [nUtt] frames of the Viterbi level before the end-of-input flush
  // cTonefilt (SOP_TONEFILT): block tables, segments of the prepared batch and their states
  TonefiltParams tf;
  DevBuf<double> dTfTab;                // W | a | freq
  PinBuf<ChunkRef> hSegs; DevBuf<ChunkRef> dSegs;
  std::vector<int32_t> uttSeg0; DevBuf<int32_t> dUttSeg0;
  DevBuf<double2> dAgg, dCin;
  // cCens (SOP_CENS): its window, and tiles of the prepared batch (cut per utterance: rows do not depend on the batch)
  CensParams cens;
  DevBuf<float> dCensWin;
  std::vector<int32_t> uttTile0;
  PinBuf<OpTile> hCensTiles; DevBuf<OpTile> dCensTiles;
  int descOp = -1;                      // index into PlanDesc::ops
};

struct osm_b200_plan {
  PlanDesc d;
  int device = -1;               // -1 until a device has been validated: release then makes no CUDA call
  int numSMs = 0;
  std::vector<StreamRt> st;
  std::vector<OpRt> ops;         // standalone ops (not fused into lld_kernel)
  PostParams pp;
  SeqPostParams sp;              // groups behind a Viterbi-smoothed pitch level (seq_post_kernel)
  int seqLagOp = -1;             // index into `ops` of the pitch chain whose lag they follow
  DevBuf<int> dErr;              // device flag: a kernel left its supported geometry (checked after run_host)
  // the pitch chain (shs -> viterbi -> jitter: latency-bound, low occupancy) runs on its own stream next to the
  // other standalone ops of a step
  CudaStream auxStream;
  CudaEvent evFork, evJoin;
  bool staticDirect = false;     // static rows are written straight into the output rows
  int identityOutCol = 0;
  bool fused = false;            // delta / delta-delta evaluated inside lld_kernel
  // batch bookkeeping
  std::vector<int64_t> cachedUttOff;
  PinBuf<long long> hMeta;       // uttOff | rowOff | statOff
  DevBuf<long long> dMeta;
  PinBuf<TileRef> hPost; DevBuf<TileRef> dPost; size_t nPostTiles = 0;
  std::vector<int32_t> uttPost0;
  DevBuf<float> dStat;
  DevBuf<float> dMeans;          // [nUtt][nStatic] column means for cFullinputMean groups
  bool needMeans = false;
  long long totalRows = 0, totalStat = 0, totalSamples = 0;
  size_t totalWork = 0;
  CudaEvent evMetaDone, evK0, evKm, evK1;
  bool metaPending = false, timed = false;
  // run_host buffers
  DevBuf<int16_t> dPcm;
  DevBuf<float> dPcmF;             // mono float samples of the batch (inputs in another format than 16-bit integer)
  DevBuf<unsigned char> dPadPcm;   // packed copy of a padded device batch (osm_b200_plan_run_device_padded)
  DevBuf<float> dOut;
  CudaStream hostStream, h2dStream, d2hStream;
  std::vector<CudaEvent> evPiece;   // 2 per pipeline piece: PCM landed / rows computed
  int lastLaunches = 0;
  // per-kernel profiling mode (osm_b200_plan_set_profiling): one event after every launch, everything on one stream
  bool profile = false;
  std::vector<CudaEvent> profEv;
  std::vector<const char *> profName;
  int profN = 0;
  LldLaunchInfo lastInfo{};
  // osm_b200_plan_last_run_info: pipeline pieces of the last run, the last spectral_kernel launch's staging path and shared memory
  int lastPieces = 0, lastSpecStaged = -1, lastSpecSmem = 0;

  // work still in flight may use any member: drain the device before they release themselves
  ~osm_b200_plan()
  {
    if (device < 0) return;
    cudaSetDevice(device);
    if (hostStream) cudaStreamSynchronize(hostStream);
    cudaDeviceSynchronize();
  }
};
extern "C" {

int32_t osm_b200_abi_version(void) { return OSM_B200_ABI_VERSION; }
int32_t osm_b200_sizeof_component(void) { return (int32_t)sizeof(osm_b200_component); }

const char *osm_b200_last_error(void) { return g_err.c_str(); }

int32_t osm_b200_device_count(void)
{
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

// defaults = the reference's ConfigType defaults (SURVEY.md Appendix A)
osm_b200_status osm_b200_component_defaults(int32_t type, osm_b200_component *c)
{
  if (!c || type < 0 || type >= OSM_B200_C_COUNT_) return fail(OSM_B200_ERR_INVALID, "bad component type");
  memset(c, 0, sizeof *c);
  c->type = type;
  c->copyInputName = 1;
  switch (type) {
    case OSM_B200_C_WAVESOURCE:
      c->u.wavesource.sampleRate = 16000; c->u.wavesource.nChannels = 1; c->u.wavesource.monoMixdown = 1;
      c->u.wavesource.format = OSM_B200_PCM_S16; strcpy(c->u.wavesource.outFieldName, "pcm");
      break;
    case OSM_B200_C_FRAMER:
      c->u.framer.frameSize = 0.025; c->u.framer.frameStep = 0.0;
      c->u.framer.frameCenterSpecial = OSM_B200_CENTER_UNSET; c->u.framer.noPostEOIprocessing = 1;
      break;
    case OSM_B200_C_VECTORPREEMPHASIS: c->u.vectorpreemphasis.k = 0.97; c->u.vectorpreemphasis.de = 0; break;
    case OSM_B200_C_WINDOWER:
      c->u.windower.winFunc = OSM_B200_WIN_HANNING; c->u.windower.gain = 1.0; c->u.windower.offset = 0.0;
      c->u.windower.sigma = 0.4;
      c->u.windower.alpha0 = (1.0 - 0.16) * 0.5; c->u.windower.alpha1 = 0.5; c->u.windower.alpha2 = 0.16 * 0.5; c->u.windower.alpha3 = 0.0;
      c->u.windower.fade = 0.0; c->u.windower.squareRoot = 0;
      break;
    case OSM_B200_C_TRANSFORMFFT: c->u.transformfft.inverse = 0; c->u.transformfft.zeroPadSymmetric = 1; break;
    case OSM_B200_C_FFTMAGPHASE: c->u.fftmagphase.magnitude = 1; c->u.fftmagphase.dBpnorm = 90.302; c->u.fftmagphase.mindBp = -102.0; break;   // dspcore/fftmagphase.cpp:44-49
    case OSM_B200_C_MELSPEC:
      c->u.melspec.nBands = 26; c->u.melspec.lofreq = 20; c->u.melspec.hifreq = 8000;
      c->u.melspec.usePower = 0; c->u.melspec.htkcompatible = 1;
      break;
    case OSM_B200_C_MFCC:
      c->u.mfcc.firstMfcc = 1; c->u.mfcc.lastMfcc = 12; c->u.mfcc.melfloor = 1e-8; c->u.mfcc.doLog = 1;
      c->u.mfcc.cepLifter = 22; c->u.mfcc.htkcompatible = 1;
      break;
    case OSM_B200_C_PLP: {
      auto &p = c->u.plp;
      p.lpOrder = 5; p.nCeps = -1; p.firstCC = 1; p.lastCC = -1; p.doLog = 1; p.doAud = 1; p.RASTA = 0;
      p.newRASTA = 0; p.doInvLog = 1; p.doIDFT = 1; p.doLP = 1; p.doLpToCeps = 1; p.rastaUpperCutoff = 29;
      p.rastaLowerCutoff = 1; p.cepLifter = 0; p.compression = 0.33; p.melfloor = 9.3e-10; p.htkcompatible = 1;
      break;
    }
    case OSM_B200_C_SPECTRAL: {
      auto &s = c->u.spectral;
      s.squareInput = 1; s.flux = 1; s.centroid = 1; s.maxPos = 1; s.minPos = 1; s.oldSlopeScale = 1;
      s.specFloor = 1e-7;
      break;
    }
    case OSM_B200_C_ENERGY: {
      auto &e = c->u.energy;
      e.rms = 1; e.log = 1; e.escaleLog = e.escaleRms = e.escaleSquare = 1.0;
      break;
    }
    case OSM_B200_C_MZCR: c->u.mzcr.zcr = 1; c->u.mzcr.mcr = 1; c->u.mzcr.amax = 1; c->u.mzcr.maxmin = 1; break;
    case OSM_B200_C_ACF: {
      auto &a = c->u.acf;
      a.usePower = 1; a.expBeforeAbs = 1; a.symmetricData = 1; a.acfCepsNormOutput = 1;
      break;
    }
    case OSM_B200_C_PITCHACF: c->u.pitchacf.maxPitch = 500; c->u.pitchacf.voiceProb = 1; c->u.pitchacf.voicingCutoff = 0.55; break;
    case OSM_B200_C_DELTAREGRESSION: c->u.deltaregression.deltawin = 2; c->u.deltaregression.zeroSegBound = 1; break;
    case OSM_B200_C_CONTOURSMOOTHER: c->u.contoursmoother.smaWin = 3; break;
    case OSM_B200_C_INTENSITY: c->u.intensity.intensity = 1; c->u.intensity.loudness = 0; break;
    case OSM_B200_C_VECTORCONCAT: c->u.vectorconcat.processArrayFields = 1; c->u.vectorconcat.includeSingleElementFields = 0; break;
    case OSM_B200_C_SPECSCALE: {           // dsp/specScale.cpp:38-62 (scale "log" with logScaleBase 2 == octave)
      auto &q = c->u.specscale;
      q.scaleOctave = 1; q.sourceLin = 1; q.splineInterp = 1; q.minF = 25.0; q.maxF = -1.0;
      break;
    }
    case OSM_B200_C_PITCHSHS: {            // lldcore/pitchBase.cpp:41-62, lld/pitchShs.cpp:56-64
      auto &q = c->u.pitchshs;
      q.maxPitch = 620.0; q.minPitch = 52.0; q.nCandidates = 3; q.scores = 1; q.voicing = 1; q.voicingCutoff = 0.70;
      q.nHarmonics = 15; q.compressionFactor = 0.85;
      break;
    }
    case OSM_B200_C_PITCHSMOOTHERVITERBI: { // lld/pitchSmootherViterbi.cpp:45-68
      auto &q = c->u.pitchsmootherviterbi;
      q.bufferLength = 30; q.F0final = 1; q.wLocal = 2.0; q.wTvv = 10.0; q.wTvvd = 5.0; q.wTvuv = 10.0; q.wThr = 4.0;
      q.wRange = 1.0; q.wTuu = 0.0;
      break;
    }
    case OSM_B200_C_VALBASEDSELECTOR: c->u.valbasedselector.threshold = 1.0; break;   // other/valbasedSelector.cpp:35-49
    case OSM_B200_C_PITCHJITTER: {         // lld/pitchJitter.cpp:45-78
      auto &q = c->u.pitchjitter;
      snprintf(q.F0field, sizeof q.F0field, "%s", "F0final");
      q.searchRangeRel = 0.10; q.lgHNRfloor = -100.0; q.minNumPeriods = 2; q.minCC = 0.5; q.useBrokenJitterThresh = 1;
      break;
    }
    case OSM_B200_C_SPECRESAMPLE: c->u.specresample.targetFs = 16000.0; c->u.specresample.resampleRatio = -1.0; break;   // dsp/specResample.cpp:40-41
    case OSM_B200_C_LPC: c->u.lpc.p = 8; c->u.lpc.saveLPCoeff = 1; break;                                               // lld/lpc.cpp:33-45
    case OSM_B200_C_LSP: c->u.lsp.processArrayFields = 1; break;                                                       // core/vectorProcessor.cpp:37
    case OSM_B200_C_DATASELECTOR: c->u.dataselector.elementMode = 1; break;                                              // core/dataSelector.cpp:39
    case OSM_B200_C_TONESPEC:              // lld/tonespec.cpp:46-52
      c->u.tonespec.nOctaves = 6; c->u.tonespec.firstNote = 55.0; c->u.tonespec.filterType = OSM_B200_TONE_GAU; c->u.tonespec.dbA = 1;
      break;
    case OSM_B200_C_CHROMA: c->u.chroma.octaveSize = 12; c->u.chroma.silThresh = 0.001; c->copyInputName = 0; break;   // lld/chroma.cpp:46-49
    case OSM_B200_C_TONEFILT:              // lld/tonefilt.cpp:35-41
      c->u.tonefilt.nNotes = 48; c->u.tonefilt.firstNote = 55.0; c->u.tonefilt.decayF0 = 0.9995; c->u.tonefilt.decayFN = 0.998;
      c->u.tonefilt.outputPeriod = 0.1;
      break;
    case OSM_B200_C_CENS:                  // lld/cens.cpp:41-47
      c->u.cens.window = OSM_B200_WIN_HANNING; c->u.cens.winlength = 41; c->u.cens.l2norm = 1; c->u.cens.downsampleRatio = 10;
      c->u.cens.winlength_sec = 0.41; c->copyInputName = 0;
      break;
    case OSM_B200_C_HARMONICS: {           // lld/harmonics.cpp:28-56
      auto &q = c->u.harmonics;
      snprintf(q.f0ElementName, sizeof q.f0ElementName, "%s", "F0final");
      snprintf(q.magSpecFieldName, sizeof q.magSpecFieldName, "%s", "pcm_fftMag");
      q.f0ElementNameIsFull = 1; q.formantFrequencyFieldNameIsFull = 1; q.formantBandwidthFieldNameIsFull = 1;
      q.nHarmonics = 100; q.firstHarmonicMagnitude = 1; q.outputLogRelMagnitudes = 1; q.harmonicDifferencesLog = 1;
      q.formantAmplitudesLogRel = 1; q.formantAmplitudesStart = 1; q.formantAmplitudesEnd = -1; q.logRelValueFloorUnvoiced = -201.0;
      break;
    }
    case OSM_B200_C_FORMANTLPC: {          // lld/formantLpc.cpp:40-52
      auto &q = c->u.formantlpc;
      q.nFormants = -1; q.saveFormants = 1; q.minF = 50.0; q.maxF = 5500.0;
      break;
    }
    default: break;
  }
  return OSM_B200_OK;
}

static void build_twiddles(int M, std::vector<float2> &tw, int twOff[4])
{
  // factorisation must match Fact<M> in kernels.cu
  int R[3] = {0, 0, 0}, ns = 0;
  if (M == 256) { R[0] = 16; R[1] = 16; ns = 2; }
  else if (M == 512) { R[0] = 8; R[1] = 8; R[2] = 8; ns = 3; }
  else if (M == 1024) { R[0] = 16; R[1] = 16; R[2] = 4; ns = 3; }
  else { R[0] = 16; R[1] = 16; R[2] = 8; ns = 3; }
  int MS = M;
  tw.clear();
  for (int s = 0; s < 4; s++) twOff[s] = 0;
  for (int s = 0; s < ns - 1; s++) {       // the last stage has no twiddles
    const int stride = MS / R[s];
    twOff[s] = (int)tw.size();
    for (int j = 0; j < stride; j++)
      for (int q = 0; q < R[s]; q++) {
        const double ang = -2.0 * M_PI * (double)j * (double)q / (double)MS;
        tw.push_back(make_float2((float)cos(ang), (float)sin(ang)));
      }
    MS = stride;
  }
}


// pack the constant tables of one lld_kernel pass of a stream (front end + optional band op `opIdx`)
// and fill its LldParams.  `dumps`: this pass writes the magnitude level.
static osm_b200_status build_pass(osm_b200_plan *pl, int si, int opIdx, bool dumps, const cudaDeviceProp &prop,
                                  LldParams &kp, PassRt &pr)
{
  const PlanDesc &d = pl->d;
  const Stream &sd = d.streams[si];
  StreamRt &rt = pl->st[si];
  const FrontEnd &fe = sd.fe;
  rt.runLld = sd.hasFft && (sd.fusedOp >= 0 || sd.dumpMag);
  rt.tileF = lld_supported_fft(fe.nfft) ? lld_tile_frames(fe.nfft) : 32;
  pr.op = opIdx;
  memset(&kp, 0, sizeof kp);
  kp.opKind = -1;
  kp.nChan = kernel_nchan(fe); kp.pcmF32 = fe.format != OSM_B200_PCM_S16;
  kp.frameSize = fe.frameSize; kp.frameStep = fe.frameStep; kp.frameCenter = fe.frameCenter;
  kp.hopMagic = (unsigned)((0x100000000ull + (unsigned long long)fe.frameStep - 1) / (unsigned long long)fe.frameStep);
  // per-lane stride S = frameStep + sPad of the shared-memory sample tile: odd S (scalar loads)
  // or even S with S/2 odd (64-bit sample-pair loads) is bank-conflict free across the lanes
  kp.sPad = (fe.frameStep % 2 != 0) ? 0 : (((fe.frameStep / 2) % 2 != 0) ? 0 : 2);
  kp.preemph = fe.preemph; kp.preDe = fe.preDe; kp.preK = fe.preK;
  kp.oneMinusK = 1 - fe.preK;                     // (1-k), float arithmetic (vectorPreemphasis.cpp:94)
  kp.winOffset = fe.winOffset; kp.hasWinOffset = fe.winOffset != 0.f;

  auto up16 = [](size_t x) { return (x + 15) / 16 * 16; };
  size_t o = 0;
  std::vector<unsigned char> blob;
  auto put = [&](const void *src, size_t bytes) { const size_t at = o; blob.resize(up16(o + bytes), 0); if (bytes) memcpy(&blob[at], src, bytes); o = up16(o + bytes); return at; };
  const size_t oWindow = put(fe.window.data(), fe.window.size() * sizeof(float));
  size_t oWin = 0, oTw = 0, oSplit = 0, oCoef = 0, oRange = 0, oDct = 0, oLift = 0, oEql = 0, oVisit = 0, oVB = 0;
  if (rt.runLld) {
    const int M = fe.nfft / 2;
    std::vector<float4> winLut(M, make_float4(0.f, 0.f, 0.f, 0.f));
    for (int e = 0; e < M; e++) {
      const int n = 2 * e;
      if (n < fe.frameSize) winLut[e].x = fe.window[n];
      if (n + 1 < fe.frameSize) winLut[e].y = fe.window[n + 1];
      const int off = (n < fe.frameSize) ? n + (n / fe.frameStep) * kp.sPad : 0;
      memcpy(&winLut[e].z, &off, sizeof(int));
      winLut[e].w = (n + 1 < fe.frameSize) ? 2.f : ((n < fe.frameSize) ? 1.f : 0.f);
    }
    std::vector<float2> tw;
    build_twiddles(M, tw, kp.twOff);
    kp.twCount = (int)tw.size();
    std::vector<float2> split(M / 2 + 1);
    for (int k = 0; k <= M / 2; k++) {
      const double ang = -2.0 * M_PI * (double)k / (double)fe.nfft;
      split[k] = make_float2((float)cos(ang), (float)sin(ang));
    }
    oWin = put(winLut.data(), winLut.size() * sizeof(float4));
    tw.push_back(make_float2(0.f, 0.f));
    oTw = put(tw.data(), tw.size() * sizeof(float2));
    oSplit = put(split.data(), split.size() * sizeof(float2));
    if (opIdx >= 0) {
      const StaticOp &op = d.ops[opIdx];
      const bool isPlp = op.kind == SOP_PLP, isTone = op.kind == SOP_TONE;
      const MelBank &mb = isTone ? op.tone.bank : d.mels[isPlp ? op.plp.melIdx : op.mfcc.melIdx];
      const MfccOp &mf = op.mfcc;
      const PlpOp &po = op.plp;
      if (isPlp && po.doLpToCeps && po.firstCC > 1) return fail(OSM_B200_ERR_UNSUPPORTED, "cPlp: firstCC > 1 is not supported");
      kp.opKind = isTone ? 2 : (isPlp ? 1 : 0);
      kp.nBands = mb.nBands; kp.melUsePower = mb.usePower;
      // without a magnitude dump the kernel keeps 2X (4|X|^2) out of the real-FFT split and the
      // exact factor 1/4 of the power path is folded into the band scale
      kp.melScale = (mb.usePower && !dumps) ? mb.outScale * 0.25f : mb.outScale;
      if (isTone) {
        // band phase: mean of the weighted bins per note (division by the bin count, sqrt under usePower); back end: the
        // tone values themselves or the chroma fold.  The per-note bin counts take the DCT table's place.
        const ToneOp &to = op.tone;
        kp.nStat = to.nOut; kp.doLog = 0;
        kp.dctStride = mb.nBands; kp.dctRows = 1;
        kp.toneSqrt = to.usePower; kp.chromaOct = to.octaveSize; kp.chromaSilThresh = to.silThresh;
      } else if (!isPlp) {
        kp.nStat = mf.nMfcc; kp.melfloor = mf.melfloor; kp.logMelfloor = mf.logMelfloor; kp.doLog = mf.doLog;
        kp.dctStride = (mb.nBands + 3) / 4 * 4; kp.dctRows = mf.nMfcc;
      } else {
        kp.nStat = po.nOut; kp.melfloor = po.melfloor; kp.logMelfloor = po.logMelfloor; kp.doLog = po.doLog;
        kp.plpAud = po.doAud; kp.plpInvLog = po.doInvLog; kp.plpIDFT = po.doIDFT; kp.plpLP = po.doLP; kp.plpCeps = po.doLpToCeps;
        kp.plpHtk = po.htk; kp.plpLifter = po.lifter; kp.plpOrder = po.lpOrder; kp.plpNAuto = po.nAuto; kp.plpNFreq = po.nFreq;
        kp.plpFirstCC = po.firstCC; kp.plpLastCC = po.lastCC; kp.plpCompression = po.compression;
        kp.dctStride = po.nFreq; kp.dctRows = po.nAuto;
      }
      // split the bands over the virtual warps: contiguous band groups, minimising the most expensive
      // group (cost model from the kernel's SASS: ~6 instructions per visited bin, ~50 per band for
      // scale / floor / log / store, ~12 per group) -- all warps meet at a barrier after this phase
      {
        const int nvw = lld_virtual_warps(fe.nfft);
        const int nB = mb.nBands;
        // the 512-point MFCC instance (lld_fast.cu) also adds every finished band into its DCT partial sums (~20 more)
        const double bandCost = (!isPlp && !isTone && !dumps && lld_fast_applies(kp, fe.nfft)) ? 70.0 : 50.0;
        auto cost = [&](int bs, int be) -> double {          // bands [bs, be) visit ranges bs..be
          if (be <= bs) return 0.0;
          return 6.0 * (mb.rangeBegin[be + 1] - mb.rangeBegin[bs]) + bandCost * (be - bs) + 12.0;
        };
        // best[w][b] = minimal max-cost of covering bands [0, b) with w groups
        std::vector<std::vector<double>> best(nvw + 1, std::vector<double>(nB + 1, 1e30));
        std::vector<std::vector<int>> from(nvw + 1, std::vector<int>(nB + 1, 0));
        best[0][0] = 0.0;
        for (int w = 1; w <= nvw; w++)
          for (int b = 0; b <= nB; b++)
            for (int a = 0; a <= b; a++) {
              const double c = std::max(best[w - 1][a], cost(a, b));
              if (c < best[w][b]) { best[w][b] = c; from[w][b] = a; }
            }
        int b = nB;
        kp.melSplit[nvw] = nB;
        for (int w = nvw; w >= 1; w--) { b = from[w][b]; kp.melSplit[w - 1] = b; }
        for (int w = nvw + 1; w <= kMaxVW; w++) kp.melSplit[w] = nB;
      }
      std::vector<float> dctPad((size_t)kp.dctRows * kp.dctStride, 0.f);
      if (isTone) {
        dctPad = op.tone.divisor;
      } else if (!isPlp) {
        for (int i = 0; i < mf.nMfcc; i++)
          memcpy(&dctPad[(size_t)i * kp.dctStride], &mf.cosT[(size_t)i * mb.nBands], sizeof(float) * mb.nBands);
      } else {
        memcpy(dctPad.data(), po.cosT.data(), sizeof(float) * po.cosT.size());
      }
      const std::vector<float> &liftV = isPlp ? po.lift : (isTone ? op.tone.divisor : mf.liftFactor);   // the tone op reads no lifter
      std::vector<float> eqlV = isPlp ? po.eql : std::vector<float>(1, 0.f);
      oCoef = put(mb.coef.data(), mb.coef.size() * sizeof(float));
      oRange = put(mb.rangeBegin.data(), mb.rangeBegin.size() * sizeof(int));
      {
        std::vector<float2> visit;
        std::vector<int> vb(mb.nBands + 2, 0);
        for (int r = 0; r <= mb.nBands; r++) {
          vb[r] = (int)visit.size();
          for (int n = mb.rangeBegin[r]; n < mb.rangeBegin[r + 1]; n++) visit.push_back(make_float2(mb.coef[n], mb.oneTap ? 0.f : 1.0f - mb.coef[n]));
          while (visit.size() % 4) visit.push_back(make_float2(0.f, 0.f));
        }
        vb[mb.nBands + 1] = (int)visit.size();
        kp.melVCount = (int)visit.size();
        visit.push_back(make_float2(0.f, 0.f));
        oVisit = put(visit.data(), visit.size() * sizeof(float2));
        oVB = put(vb.data(), vb.size() * sizeof(int));
      }
      oDct = put(dctPad.data(), dctPad.size() * sizeof(float));
      oLift = put(liftV.data(), liftV.size() * sizeof(float));
      oEql = put(eqlV.data(), eqlV.size() * sizeof(float));
    }
  }
  CU(pr.dConst.upload(blob.data(), blob.size()));
  const unsigned char *dC = pr.dConst.p;
  if (!rt.dWindow) rt.dWindow = reinterpret_cast<const float *>(dC + oWindow);
  if (rt.runLld) {
    kp.winLut = reinterpret_cast<const float4 *>(dC + oWin);
    kp.twiddles = reinterpret_cast<const float2 *>(dC + oTw);
    kp.splitTw = reinterpret_cast<const float2 *>(dC + oSplit);
    if (opIdx >= 0) {
      kp.melCoef = reinterpret_cast<const float *>(dC + oCoef);
      kp.melRange = reinterpret_cast<const int *>(dC + oRange);
      kp.melVisit = reinterpret_cast<const float2 *>(dC + oVisit);
      kp.melVB = reinterpret_cast<const int *>(dC + oVB);
      kp.dctCos = reinterpret_cast<const float *>(dC + oDct);
      kp.dctLift = reinterpret_cast<const float *>(dC + oLift);
      kp.plpEql = reinterpret_cast<const float *>(dC + oEql);
      const StaticOp &op = d.ops[opIdx];
      if (op.kind == SOP_PLP && op.plp.rasta) {
        // RASTA sits in the middle of cPlp: the kernel pass stops at the (log) band level, a
        // sequential filter runs over time, plp_tail_kernel finishes the op
        pr.rasta = true;
        pr.tail = kp;
        kp.plpAud = 0; kp.plpInvLog = 0; kp.plpIDFT = 0; kp.plpLP = 0; kp.plpCeps = 0; kp.plpLifter = 0;
        kp.nStat = kp.nBands;
        memset(&pr.rp, 0, sizeof pr.rp);
        pr.rp.nBands = kp.nBands; pr.rp.frameSize = fe.frameSize; pr.rp.frameStep = fe.frameStep; pr.rp.frameCenter = fe.frameCenter;
        pr.rp.mode = op.plp.rasta; pr.rp.iir = op.plp.rastaIir;
        for (int i = 0; i < 5; i++) pr.rp.fir[i] = op.plp.rastaFir[i];
      }
    }
    if (rt.forceNarrow || (lld_smem_bytes(kp, fe.nfft) > (size_t)prop.sharedMemPerBlockOptin && fe.nfft >= 1024)) {
      kp.narrow = 1;                                   // long stereo strides: half-width tiles
      rt.tileF = lld_tile_frames(fe.nfft, true);
      rt.forceNarrow = true;                           // every pass of a stream uses the same tile width
    }
    if (lld_smem_bytes(kp, fe.nfft) > (size_t)prop.sharedMemPerBlockOptin)
      return fail(OSM_B200_ERR_UNSUPPORTED, "configuration needs more shared memory than the device offers");
  }
  return OSM_B200_OK;
}

// ---- output groups / execution mode: pl->staticDirect (`simple` plans, one stream with one fused band op and nothing else, write
// their static rows straight into the output rows), pl->pp, pl->sp, and seqLagDescOp: the pitch chain the sequential groups follow ----
static osm_b200_status build_groups(osm_b200_plan *pl, bool simple, int &seqLagDescOp)
{
  const PlanDesc &d = pl->d;
  PostParams &pp = pl->pp;
  memset(&pp, 0, sizeof pp);
  pl->staticDirect = false;
  if (simple)
    for (const auto &g : d.groups)
      if (g.stages.empty() && g.srcCol == 0 && g.n == d.nStatic) { pl->staticDirect = true; pl->identityOutCol = g.outCol; break; }
  memset(&pl->sp, 0, sizeof pl->sp);
  for (const auto &g : d.groups) {
    if (g.stages.empty() && pl->staticDirect && g.srcCol == 0 && g.n == d.nStatic && g.outCol == pl->identityOutCol) continue;
    if (g.lagKind != 0 && !g.stages.empty()) {
      SeqPostParams &sq = pl->sp;
      if (sq.nGroups >= kMaxSeqGroups) return fail(OSM_B200_ERR_UNSUPPORTED, "too many output groups behind the pitch chain");
      if (seqLagDescOp >= 0 && seqLagDescOp != g.lagOp) return fail(OSM_B200_ERR_UNSUPPORTED, "more than one SHS pitch chain per graph is not supported");
      seqLagDescOp = g.lagOp;
      SeqGroup &G = sq.groups[sq.nGroups++];
      G.srcCol = g.srcCol; G.n = g.n; G.outCol = g.outCol; G.lagKind = g.lagKind; G.nStages = (int)g.stages.size();
      G.noZero = g.stages[0].flags & 1;
      G.deltaWin = g.stages.size() > 1 ? g.stages[1].win : 0;
      G.segId = g.segId;
      G.gateCol = g.gateCol; G.gateFlags = (g.gateInvert ? 1 : 0) | (g.gateAllowEqual ? 2 : 0); G.gateThr = g.gateThreshold; G.gateOut = g.gateOutVal;
      if (G.nStages == 2 && G.deltaWin != 2) return fail(OSM_B200_ERR_UNSUPPORTED, "cDeltaRegression(onlyInSegments) behind the pitch chain: deltawin must be 2");
      if (G.nStages == 2) {
        int segCols = 0;
        for (int q = 0; q < sq.nGroups; q++) if (sq.groups[q].nStages == 2 && sq.groups[q].segId == G.segId) segCols += sq.groups[q].n;
        if (segCols > 32) return fail(OSM_B200_ERR_UNSUPPORTED, "cDeltaRegression(onlyInSegments): more than 32 elements");
      }
      if (G.segId >= kMaxSegIds) return fail(OSM_B200_ERR_UNSUPPORTED, "too many onlyInSegments delta components");
      sq.frameSize = d.streams[g.stream].fe.frameSize; sq.frameStep = d.streams[g.stream].fe.frameStep; sq.frameCenter = d.streams[g.stream].fe.frameCenter;
      continue;
    }
    if (pp.nGroups >= kMaxPostGroups) return fail(OSM_B200_ERR_UNSUPPORTED, "too many output groups");
    PostGroup &pg = pp.groups[pp.nGroups++];
    pg.srcCol = g.srcCol; pg.n = g.n; pg.outCol = g.outCol; pg.nStages = (int)g.stages.size();
    pg.frameSize = d.streams[g.stream].fe.frameSize; pg.frameStep = d.streams[g.stream].fe.frameStep; pg.frameCenter = d.streams[g.stream].fe.frameCenter;
    pg.nLim = 0;
    for (int ls : g.limitStreams) if (pg.nLim < 3) {
      pg.limSize[pg.nLim] = d.streams[ls].fe.frameSize; pg.limStep[pg.nLim] = d.streams[ls].fe.frameStep; pg.limCenter[pg.nLim] = d.streams[ls].fe.frameCenter;
      pg.nLim++;
    }
    for (size_t i = 0; i < g.stages.size(); i++) { pg.kind[i] = g.stages[i].kind; pg.win[i] = g.stages[i].win; pg.flags[i] = g.stages[i].flags; if (g.stages[i].kind == ST_CMS) pl->needMeans = true; }
  }
  pp.nStat = d.nStatic; pp.maxN = 1; pp.halo = 0;
  for (int g = 0; g < pp.nGroups; g++) {
    int h = 0;
    for (int s2 = 0; s2 < pp.groups[g].nStages; s2++) h += pp.groups[g].win[s2];
    if (h > pp.halo) pp.halo = h;
    if (pp.groups[g].n > pp.maxN) pp.maxN = pp.groups[g].n;
  }
  if (pp.halo > 12) return fail(OSM_B200_ERR_UNSUPPORTED, "summed temporal half windows exceed 12 frames");
  pp.rows = post_tile_rows(pp.nStat, pp.maxN, pp.halo);
  if ((size_t)(pp.rows + 2 * pp.halo) * (pp.nStat + 2 * pp.maxN) * sizeof(float) > 200 * 1024)
    return fail(OSM_B200_ERR_UNSUPPORTED, "the static level is too wide for the row assembly kernel");
  return OSM_B200_OK;
}

// fused pattern: [static | delta(W1) | delta(W1,W2)] over the whole static vector, evaluated inside lld_kernel
static void detect_fused_delta(osm_b200_plan *pl, bool simple)
{
  const PlanDesc &d = pl->d;
  LldParams &kp = pl->st[0].kp;
  pl->fused = false;
  kp.fused = 0; kp.halo = 0; kp.fW1 = kp.fW2 = 0; kp.fNorm1 = kp.fNorm2 = 1.f;
  if (!(simple && pl->staticDirect && pl->identityOutCol == 0 && d.groups.size() == 3 && d.nOut == 3 * d.nStatic)) return;
  const auto &g1 = d.groups[1], &g2 = d.groups[2];
  const bool shape = d.groups[0].stages.empty() && g1.stages.size() == 1 && g2.stages.size() == 2 &&
                     g1.srcCol == 0 && g2.srcCol == 0 && g1.n == d.nStatic && g2.n == d.nStatic &&
                     g1.outCol == d.nStatic && g2.outCol == 2 * d.nStatic &&
                     g1.stages[0].kind == ST_DELTA && g2.stages[0].kind == ST_DELTA && g2.stages[1].kind == ST_DELTA &&
                     g1.stages[0].win == g2.stages[0].win &&
                     g1.stages[0].flags == 0 && g2.stages[0].flags == 0 && g2.stages[1].flags == 0;   // plain regression only
  // OSM_B200_NO_FUSE=1 forces the two-kernel path (used by the tests to cross-check both)
  const char *nf = getenv("OSM_B200_NO_FUSE");
  // the kernel keeps the statics of two tiles (2F frames).  After a tile it emits the rows from hl before the tile's start to
  // hl before its end; their delta-deltas read statics back to 2*hl before the tile's start, which the ring still holds
  // only when 2*hl <= F (wider halos at 8- or 4-frame tiles run through post_kernel)
  const int hl = g1.stages[0].win + g2.stages[1].win, tF = pl->st[0].tileF;
  if (shape && hl <= 8 && 2 * hl <= tF && !(nf && nf[0] == '1')) {
    pl->fused = true;
    kp.fused = 1; kp.fW1 = g1.stages[0].win; kp.fW2 = g2.stages[1].win; kp.halo = kp.fW1 + kp.fW2;
    auto normOf = [](int W) { float n = 0.f; for (int i = 1; i <= W; i++) n += (float)i * (float)i; return n * 2.0f; };
    kp.fNorm1 = normOf(kp.fW1); kp.fNorm2 = normOf(kp.fW2);    // deltaRegression.cpp:77-80
    // divisors with an exhaustively verified exact reciprocal+FMA division (kernels.cu div_exact)
    auto rcpOf = [](float n) { return (n == 2.f || n == 10.f || n == 28.f || n == 60.f) ? 1.0f / n : 0.f; };
    kp.fRcp1 = rcpOf(kp.fNorm1); kp.fRcp2 = rcpOf(kp.fNorm2);
  }
}

// ---- standalone ops: one builder per kind fills `rt` (its tables included) ----
static osm_b200_status build_spectral(const PlanDesc &d, const StaticOp &op, const StreamRt &srt, OpRt &rt)
{
  const SpectralOp &so = op.spectral;
  SpectralParams &sp = rt.sp;
  memset(&sp, 0, sizeof sp);
  sp.F = srt.tileF; sp.statStride = d.nStatic; sp.outCol = op.outCol;
  sp.nSrc = so.nSrc; sp.loBin = so.loBin; sp.hiBin = so.hiBin; sp.F0 = so.F0;
  sp.squareInput = so.squareInput; sp.useLog = so.useLog; sp.normBand = so.normBand; sp.buggyRollOff = so.buggyRollOff;
  sp.oldSlopeScale = so.oldSlopeScale; sp.reqMag = so.reqMag; sp.reqPow = so.reqPow; sp.reqLog = so.reqLog;
  sp.specFloor = so.specFloor; sp.logSpecFloor = so.logSpecFloor;
  sp.nBands = (int)so.bandIL.size();
  for (int i = 0; i < sp.nBands; i++) { sp.bandIL[i] = so.bandIL[i]; sp.bandIR[i] = so.bandIR[i]; sp.bandWL[i] = so.bandWL[i]; sp.bandWR[i] = so.bandWR[i]; }
  sp.nSlopes = (int)so.slopeIL.size();
  for (int i = 0; i < sp.nSlopes; i++) { sp.slopeIL[i] = so.slopeIL[i]; sp.slopeIR[i] = so.slopeIR[i]; sp.slopeWL[i] = so.slopeWL[i]; sp.slopeWR[i] = so.slopeWR[i]; sp.slopeNind[i] = so.slopeNind[i]; }
  sp.nRollOff = (int)so.rollOff.size();
  for (int i = 0; i < sp.nRollOff; i++) sp.rollOff[i] = so.rollOff[i];
  sp.alphaRatio = so.alphaRatio; sp.hammarberg = so.hammarberg; sp.flux = so.flux; sp.centroid = so.centroid;
  sp.maxPos = so.maxPos; sp.minPos = so.minPos; sp.entropy = so.entropy; sp.stddev = so.stddev; sp.variance = so.variance;
  sp.skewness = so.skewness; sp.kurtosis = so.kurtosis; sp.slope = so.slope; sp.sharpness = so.sharpness;
  sp.harmonicity = so.harmonicity; sp.flatness = so.flatness; sp.logFlatness = so.logFlatness;
  CU(rt.dSharpW.upload(so.sharpW.data(), so.sharpW.size()));
  sp.sharpW = rt.dSharpW.p;
  return OSM_B200_OK;
}

static osm_b200_status build_harmonics(const PlanDesc &d, const StaticOp &op, const StreamRt &srt, OpRt &rt)
{
  const HarmonicsOp &ho = op.harmonics;
  HarmonicsParams &hp = rt.hrm;
  memset(&hp, 0, sizeof hp);
  const int N = (ho.nb - 1) * 2;
  std::vector<double> ct(N);
  for (int m = 0; m < N; m++) ct[m] = cos(2.0 * M_PI * (double)m / (double)N);
  CU(rt.dCosTab.upload(ct.data(), ct.size()));
  hp.F = srt.tileF; hp.nb = ho.nb; hp.binHz = ho.binHz; hp.statStride = d.nStatic; hp.outCol = op.outCol;
  hp.f0Col = ho.f0Col; hp.fmtCol = ho.fmtCol; hp.nFmt = ho.nFmt; hp.cosTab = rt.dCosTab.p;
  hp.nHarm = ho.nHarm; hp.doHnr = ho.hnr; hp.nDiffs = (int)ho.diffs.size() / 4;
  for (size_t i = 0; i < ho.diffs.size() && i < 16; i++) hp.diffs[i] = ho.diffs[i];
  hp.doFa = ho.fa; hp.faStart = ho.faStart; hp.faEnd = ho.faEnd; hp.floorUnvoiced = ho.floorUnvoiced;
  if (harmonics_smem_bytes(hp) > 200 * 1024) return fail(OSM_B200_ERR_UNSUPPORTED, "cHarmonics: spectrum too long for the kernel");
  return OSM_B200_OK;
}

// the SHS pitch chain: cSpecScale + cPitchShs (shs_kernel) and cPitchSmootherViterbi (viterbi_kernel)
static osm_b200_status build_shs_chain(const PlanDesc &d, const StaticOp &op, const FrontEnd &fe, const StreamRt &srt, const cudaDeviceProp &prop, OpRt &rt)
{
  const PitchChainOp &pc = op.chain;
  // one blob: fwdA | fwdP6 | r1 | r2 | bwdD (double[nMag]) | ia | ic | id | audW (double[nPts]) | ik (int[nPts]) | shift (int) | hscale (float)
  // the five recurrence tables are stored lane-interleaved for the blocked scan of shs_kernel (lane l owns points
  // [l * blk, (l+1) * blk)): entry of (lane, step k) at [k * 32 + lane], so a warp reads 32 consecutive doubles
  const int blk = (pc.nMag + 31) / 32;
  const size_t nM = (size_t)blk * 32, nP = (size_t)pc.nPts, nH = pc.shift.size();
  std::vector<unsigned char> blob((5 * nM + 4 * nP) * sizeof(double) + nP * sizeof(int) + nH * (sizeof(int) + sizeof(float)) + 64);
  double *bd = reinterpret_cast<double *>(blob.data());
  const std::vector<double> *tabs[5] = {&pc.fwdA, &pc.fwdP6, &pc.r1, &pc.r2, &pc.bwdD};
  for (int t = 0; t < 5; t++)
    for (int l = 0; l < 32; l++)
      for (int k = 0; k < blk; k++) {
        const int i = l * blk + k;
        bd[(size_t)t * nM + (size_t)k * 32 + l] = i < pc.nMag ? (*tabs[t])[i] : 0.0;
      }
  double *bp = bd + 5 * nM;
  memcpy(bp, pc.ia.data(), nP * 8); memcpy(bp + nP, pc.ic.data(), nP * 8); memcpy(bp + 2 * nP, pc.id.data(), nP * 8);
  if (!pc.audW.empty()) memcpy(bp + 3 * nP, pc.audW.data(), nP * 8);
  int *bi = reinterpret_cast<int *>(bp + 4 * nP);
  memcpy(bi, pc.ik.data(), nP * sizeof(int));
  memcpy(bi + nP, pc.shift.data(), nH * sizeof(int));
  memcpy(bi + nP + nH, pc.hscale.data(), nH * sizeof(float));
  CU(rt.dPitchTab.upload(blob.data(), blob.size()));
  const double *dd = reinterpret_cast<const double *>(rt.dPitchTab.p);
  ShsParams &sh = rt.shs;
  memset(&sh, 0, sizeof sh);
  sh.F = srt.tileF; sh.nShsCols = pc.nShsCols; sh.nMag = pc.nMag; sh.nPts = pc.nPts; sh.blk = (pc.nMag + 31) / 32;
  sh.enhance = pc.enhance; sh.smooth = pc.smooth; sh.hasAudW = !pc.audW.empty();
  sh.fwdA = dd; sh.fwdP6 = dd + nM; sh.r1 = dd + 2 * nM; sh.r2 = dd + 3 * nM; sh.bwdD = dd + 4 * nM;
  const double *dp = dd + 5 * nM;
  sh.ia = dp; sh.ic = dp + nP; sh.id = dp + 2 * nP; sh.audW = dp + 3 * nP;
  const int *di = reinterpret_cast<const int *>(dp + 4 * nP);
  sh.ik = di;
  for (size_t h = 0; h < nH && h < 32; h++) { sh.shift[h] = pc.shift[h]; sh.hscale[h] = pc.hscale[h]; }
  sh.nCand = pc.nCand; sh.nHarm = pc.nHarm; sh.Fmint = pc.Fmint; sh.Fstept = pc.Fstept; sh.logBase = pc.logBase;
  sh.maxPitch = pc.maxPitch; sh.minPitch = pc.minPitch; sh.voicingCutoff = pc.voicingCutoff; sh.lfCutBin = pc.lfCutBin;
  sh.greedy = pc.greedy; sh.octaveCorr = pc.octaveCorr; sh.scores = pc.scores; sh.voicing = pc.voicing; sh.F0C1 = pc.F0C1;
  sh.voicingC1 = pc.voicingC1; sh.F0raw = pc.F0raw; sh.voicingClip = pc.voicingClip;
  if (((size_t)2 * (pc.nMag + 2) * sizeof(double) + (size_t)pc.nPts * sizeof(float) + 128) > (size_t)prop.sharedMemPerBlockOptin ||
      (size_t)pc.nPts * sizeof(float) > (size_t)(pc.nMag + 2) * sizeof(double))
    return fail(OSM_B200_ERR_UNSUPPORTED, "cSpecScale: spectrum too long for the SHS kernel's workspace");
  ViterbiParams &vp = rt.vit;
  memset(&vp, 0, sizeof vp);
  vp.nShsCols = pc.nShsCols; vp.nCand = pc.nCand; vp.frameSize = fe.frameSize; vp.frameStep = fe.frameStep; vp.frameCenter = fe.frameCenter;
  vp.statStride = d.nStatic; vp.outCol = op.outCol; vp.bufLen = pc.bufLen;
  vp.oF0final = pc.oF0final; vp.oF0finalLog = pc.oF0finalLog; vp.oF0finalEnv = pc.oF0finalEnv; vp.oF0finalEnvLog = pc.oF0finalEnvLog;
  vp.oVClipped = pc.oVClipped; vp.oVUnclipped = pc.oVUnclipped;
  vp.wLocal = pc.wLocal; vp.wTvv = pc.wTvv; vp.wTvvd = pc.wTvvd; vp.wTvuv = pc.wTvuv; vp.wThr = pc.wThr; vp.wRange = pc.wRange; vp.wTuu = pc.wTuu;
  vp.voiceThresh = pc.voicingCutoff;                       // level meta data of cPitchShs (lldcore/pitchBase.cpp:150-153)
  vp.hasSel = pc.hasSel; vp.selCol = pc.hasSel ? d.ops[pc.selOp].outCol : 0; vp.selInvert = pc.selInvert; vp.selAllowEqual = pc.selAllowEqual;
  vp.selThreshold = pc.selThreshold; vp.selOutputVal = pc.selOutputVal;
  return OSM_B200_OK;
}

static osm_b200_status build_jitter(const PlanDesc &d, const StaticOp &op, const FrontEnd &fe, OpRt &rt)
{
  const JitterOp &jo = op.jitter;
  JitterParams &jp = rt.jit;
  memset(&jp, 0, sizeof jp);
  jp.nChan = kernel_nchan(fe); jp.pcmF32 = fe.format != OSM_B200_PCM_S16; jp.frameSize = fe.frameSize; jp.frameStep = fe.frameStep; jp.frameCenter = fe.frameCenter;
  jp.Ts = 1.0 / fe.sampleRate;                               // period of the wave level
  jp.pitchT = fe.frameStepSec;                               // period of the F0 level (core/winToVecProcessor.cpp:563)
  jp.statStride = d.nStatic; jp.f0Col = d.ops[jo.pitchOp].outCol + jo.f0Col; jp.outCol = op.outCol;
  jp.searchRangeRel = jo.searchRangeRel; jp.lgHNRfloor = (float)jo.lgHNRfloor; jp.minNumPeriods = jo.minNumPeriods;
  float thr = (float)jo.minCC;                               // lld/pitchJitter.cpp:150-158
  if (thr < 0.01f) thr = 0.01f;
  if (thr > 0.99f) thr = 0.99f;
  jp.threshCC = thr;
  jp.jitterLocal = jo.jitterLocal; jp.jitterDDP = jo.jitterDDP; jp.jitterLocalEnv = jo.jitterLocalEnv; jp.jitterDDPEnv = jo.jitterDDPEnv;
  jp.shimmerLocal = jo.shimmerLocal; jp.shimmerLocalDB = jo.shimmerLocalDB; jp.shimmerLocalEnv = jo.shimmerLocalEnv;
  jp.shimmerLocalDBEnv = jo.shimmerLocalDBEnv; jp.harmonicERMS = jo.harmonicERMS; jp.noiseERMS = jo.noiseERMS; jp.linearHNR = jo.linearHNR;
  jp.logHNR = jo.logHNR; jp.shimmerUseRms = jo.shimmerUseRms; jp.refinedF0 = jo.refinedF0; jp.srcQualRange = jo.srcQualRange;
  jp.srcQualMean = jo.srcQualMean; jp.peakToPeak = jo.peakToPeak; jp.brokenThresh = jo.brokenThresh;
  // F0 comes out of the pitch chain within [minPitch, maxPitch]: longest / shortest period in samples
  const PitchChainOp &pc = d.ops[jo.pitchOp].chain;
  const double fs = fe.sampleRate, fLo = pc.minPitch > 1.0 ? pc.minPitch : 1.0, fHi = pc.maxPitch > fLo ? pc.maxPitch : fLo;
  const double tMax = fs / fLo, tMin = fs / fHi;
  const long maxPer = (long)ceil((1.0 + jo.searchRangeRel) * tMax) + 2;
  long minPer = (long)floor((1.0 - jo.searchRangeRel) * tMin);
  if (minPer < 1) minPer = 1;
  const long ppLen = (long)ceil(fe.frameStepSec * fs) + 1;
  long capWav = fe.frameSize + 2 + ppLen + maxPer + 16;
  const long twoPp = jo.minNumPeriods * maxPer + jo.minNumPeriods + ppLen + 16;
  if (capWav < twoPp) capWav = twoPp;
  jp.capWav = (int)((capWav + 3) & ~3L);
  jp.capCC = (int)(((long)ceil(2.0 * jo.searchRangeRel * tMax) + 8 + 1) & ~1L);
  jp.capAvg = (int)(((long)ceil(tMax) + 8 + 3) & ~3L);
  jp.capPb = (int)((capWav / minPer + 8 + 3) & ~3L);            // period starts of one frame: toRead / T0min + 2 at most
  if (pc.minPitch < 1.0 || (size_t)4 * ((size_t)jp.capCC * 8 + (size_t)(jp.capWav + jp.capAvg) * 4 + (size_t)jp.capPb * 4) > 200 * 1024)
    return fail(OSM_B200_ERR_UNSUPPORTED, "cPitchJitter: frame size / pitch range need more workspace than the kernel has");
  return OSM_B200_OK;
}

static osm_b200_status build_acf_pitch(const PlanDesc &d, const StaticOp &op, const FrontEnd &fe, const StreamRt &srt, OpRt &rt)
{
  if (!acf_pitch_supported_fft(fe.nfft)) return fail(OSM_B200_ERR_UNSUPPORTED, "cAcf / cPitchACF: FFT size must be 512, 1024 or 2048");
  const PitchAcfOp &po = op.pitch;
  AcfPitchParams &ap = rt.ap;
  memset(&ap, 0, sizeof ap);
  ap.F = srt.tileF;     // width of the magnitude level's tiles
  ap.nfft = fe.nfft; ap.nSrc = fe.nBins;
  ap.acfUsePower = po.acfUsePower; ap.cepUsePower = po.cepUsePower; ap.absCepstrum = po.absCepstrum; ap.normOutput = po.normOutput;
  ap.oldCompatCepstrum = po.oldCompatCepstrum;
  ap.maxPitch = po.maxPitch; ap.voicingCutoff = po.voicingCutoff; ap.fsSec = po.fsSec;
  ap.voiceProb = po.voiceProb; ap.voiceQual = po.voiceQual; ap.HNR = po.HNR; ap.HNRdB = po.HNRdB; ap.linHNR = po.linHNR;
  ap.F0 = po.F0; ap.F0raw = po.F0raw; ap.F0env = po.F0env;
  ap.statStride = d.nStatic; ap.outCol = op.outCol; ap.frameSize = fe.frameSize; ap.frameStep = fe.frameStep; ap.frameCenter = fe.frameCenter;
  // complex FFT of size nfft: same factorisation tables as lld_kernel's M = nfft, plus one spare entry (zero)
  std::vector<float2> tw;
  build_twiddles(fe.nfft, tw, ap.twOff);
  ap.twCount = (int)tw.size();
  tw.push_back(make_float2(0.f, 0.f));
  CU(rt.dTw.upload(tw.data(), tw.size()));
  ap.twiddles = rt.dTw.p;
  return OSM_B200_OK;
}

// ops on the framed waveform: energy, mzcr, intensity, formant (cSpecResample + cFormantLpc), LPC / LSP
static osm_b200_status build_time_op(const PlanDesc &d, const StaticOp &op, const FrontEnd &fe, const StreamRt &srt, OpRt &rt)
{
  TimeOpParams &tp = rt.tp;
  memset(&tp, 0, sizeof tp);
  tp.nChan = kernel_nchan(fe); tp.pcmF32 = fe.format != OSM_B200_PCM_S16; tp.F = srt.tileF; tp.statStride = d.nStatic; tp.outCol = op.outCol;
  tp.frameSize = fe.frameSize; tp.frameStep = fe.frameStep; tp.frameCenter = fe.frameCenter;
  tp.windowed = op.windowed; tp.preemph = op.windowed && fe.preemph; tp.preDe = fe.preDe; tp.preK = fe.preK;
  tp.oneMinusK = 1 - fe.preK; tp.winOffset = fe.winOffset; tp.window = srt.dWindow;
  if (op.kind == SOP_INTENSITY) {
    tp.iIntensity = op.intensity.intensity; tp.iLoudness = op.intensity.loudness;
    tp.iW0 = op.intensity.w[0]; tp.iW1 = op.intensity.w[1]; tp.iWinSum = op.intensity.winSum;
  } else if (op.kind == SOP_FORMANT) {
    const FormantOp &fo = op.formant;
    FormantParams &fp = rt.fmt;
    memset(&fp, 0, sizeof fp);
    CU(rt.dFmtD.upload(fo.D.data(), fo.D.size()));
    fp.tp = tp; fp.D = rt.dFmtD.p; fp.nRes = fo.nRes; fp.nResPad = fo.nResPad; fp.p = fo.p; fp.nFormants = fo.nFormants;
    fp.T = fo.T; fp.minF = fo.minF; fp.maxF = fo.maxF;
    fp.refOrder = fo.refOrder ? 1 : 0; fp.kHalf = fo.kHalf; fp.padLeft = fo.padLeft; fp.halfK = fo.halfK;
    fp.saveFormants = fo.saveFormants; fp.saveBandwidths = fo.saveBandwidths; fp.saveNValid = fo.saveNValid;
    // the shared-memory limit of formant_kernel is refused by the graph pass (tables.cpp build_formant)
  } else if (op.kind == SOP_LPC) {
    LpcParams &lp = rt.lpc;
    memset(&lp, 0, sizeof lp);
    tp.preemph = fe.preemph;                   // the level cLpc reads: pre-emphasised whenever its chain has the stage
    lp.tp = tp; lp.p = op.lpc.p; lp.outLpc = op.lpc.lpc; lp.outGain = op.lpc.gain; lp.outLsp = op.lpc.lsp;
    if (lpc_smem_bytes(lp) > 200 * 1024) return fail(OSM_B200_ERR_UNSUPPORTED, "cLpc: frame too long for the LPC kernel");
  } else if (op.kind == SOP_ENERGY) {
    const EnergyOp &e = op.energy;
    tp.eHtk = e.htk; tp.eRms = e.rms; tp.eEnergy2 = e.energy2; tp.eLog = e.lg;
    tp.escaleLog = e.escaleLog; tp.escaleRms = e.escaleRms; tp.escaleSquare = e.escaleSquare;
    tp.ebiasLog = e.ebiasLog; tp.ebiasRms = e.ebiasRms; tp.ebiasSquare = e.ebiasSquare;
  } else {
    const MzcrOp &z = op.mzcr;
    tp.zZcr = z.zcr; tp.zMcr = z.mcr; tp.zAmax = z.amax; tp.zMaxmin = z.maxmin; tp.zDc = z.dc;
  }
  return OSM_B200_OK;
}

// cTonefilt [-> cChroma]: the block tables of tonefilt_math.cuh on the device
static osm_b200_status build_tonefilt_rt(const PlanDesc &d, const StaticOp &op, const FrontEnd &fe, OpRt &rt)
{
  const TonefiltOp &to = op.tonefilt;
  std::vector<double> W, a;
  tf::block_tables(to.freq, to.decay, to.P, to.T, W, a);
  std::vector<double> tab(W);
  tab.insert(tab.end(), a.begin(), a.end());
  tab.insert(tab.end(), to.freq.begin(), to.freq.end());
  CU(rt.dTfTab.upload(tab.data(), tab.size()));
  TonefiltParams &p = rt.tf;
  memset(&p, 0, sizeof p);
  p.tp.nChan = kernel_nchan(fe); p.tp.pcmF32 = fe.format != OSM_B200_PCM_S16; p.tp.statStride = d.nStatic; p.tp.outCol = op.outCol;
  p.W = rt.dTfTab.p; p.nc = tf::padded_cols(to.nNotes); p.kp = tf::padded_rows(to.P);
  p.a = rt.dTfTab.p + W.size(); p.freq = p.a + to.nNotes;
  p.P = to.P; p.nNotes = to.nNotes; p.T = to.T;
  p.chromaK = to.octaveSize; p.silThresh = to.silThresh;
  tonefilt_smem_bytes(to.nNotes, to.octaveSize > 0, &p.smemSums);
  return OSM_B200_OK;
}

// no exception crosses the C boundary (host allocation failures while the plan is built)
osm_b200_status osm_b200_plan_create(const osm_b200_component *comps, int32_t n_comps,
                                     const char *output_level, int32_t device, osm_b200_plan **out)
try {
  if (!comps || n_comps <= 0 || !out) return fail(OSM_B200_ERR_INVALID, "null argument");
  *out = nullptr;
  auto pl = std::make_unique<osm_b200_plan>();
  std::string err;
  osm_b200_status st = compile_graph(comps, n_comps, output_level, pl->d, err);
  if (st != OSM_B200_OK) return fail(st, err);
  const PlanDesc &d = pl->d;
  for (const Stream &sd : d.streams)
    if (sd.hasFft && (sd.fusedOp >= 0 || sd.dumpMag) && !lld_supported_fft(sd.fe.nfft))
      return fail(OSM_B200_ERR_UNSUPPORTED, "FFT size " + std::to_string(sd.fe.nfft) + " not supported (512, 1024, 2048, 4096)");
  if (device < 0) {
    // description-only plan: geometry, names and frame-count rules without touching CUDA
    // (used by host-side tooling and CPU-only tests); it can never run.
    *out = pl.release();
    return OSM_B200_OK;
  }
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev <= 0) {
    cudaGetLastError();
    return fail(OSM_B200_ERR_CUDA, "no usable CUDA device (this library has no CPU fallback)");
  }
  if (device >= ndev) return fail(OSM_B200_ERR_INVALID, "bad device index");
  pl->device = device;
  CU(cudaSetDevice(device));
  cudaDeviceProp prop;
  CU(cudaGetDeviceProperties(&prop, device));
  pl->numSMs = prop.multiProcessorCount;

  pl->st.resize(d.streams.size());
  for (size_t s = 0; s < d.streams.size(); s++) {
    StreamRt &rt = pl->st[s];
    const std::vector<int> &bo = d.streams[s].bandOps;
    // pass 0: first band op (or none) + the magnitude dump; passes 1..: the other band ops
    st = build_pass(pl.get(), (int)s, bo.empty() ? -1 : bo[0], d.streams[s].dumpMag, prop, rt.kp, rt.pass0x);
    if (st != OSM_B200_OK) return st;
    rt.extra.resize(bo.size() > 1 ? bo.size() - 1 : 0);
    for (size_t j = 1; j < bo.size(); j++) {
      st = build_pass(pl.get(), (int)s, bo[j], false, prop, rt.extra[j - 1].kp, rt.extra[j - 1]);
      if (st != OSM_B200_OK) return st;
    }
    if (rt.forceNarrow) {                              // a later pass switched to half-width tiles: all must agree
      rt.kp.narrow = 1;
      for (PassRt &pr : rt.extra) pr.kp.narrow = 1;
    }
  }

  const bool simple = d.streams.size() == 1 && d.ops.size() == 1 && d.streams[0].fusedOp == 0 && !d.streams[0].dumpMag &&
                      !(d.ops[0].kind == SOP_PLP && d.ops[0].plp.rasta);
  int seqLagDescOp = -1;
  st = build_groups(pl.get(), simple, seqLagDescOp);
  if (st != OSM_B200_OK) return st;
  detect_fused_delta(pl.get(), simple);

  for (size_t oi = 0; oi < d.ops.size(); oi++) {
    const StaticOp &op = d.ops[oi];
    if (op.kind == SOP_MFCC || op.kind == SOP_PLP || op.kind == SOP_TONE) continue;      // fused into its stream's lld_kernel
    OpRt rt;
    rt.kind = op.kind; rt.stream = op.stream; rt.descOp = (int)oi;
    StreamRt &srt = pl->st[op.stream];
    if (op.kind != SOP_VECOP && op.kind != SOP_TONEFILT && op.kind != SOP_CENS) srt.needTiles = true;      // the op reads its stream tile by tile
    if (op.kind == SOP_MAG) {
      rt.vN = d.streams[op.stream].fe.nBins; rt.vOutCol = op.outCol;
      rt.magMode = op.magMode; rt.magN = (float)d.streams[op.stream].fe.nfft; rt.magDbNorm = op.magDbNorm; rt.magMinDb = op.magMinDb;
    } else if (op.kind == SOP_VECOP) {
      const StaticOp &src = d.ops[op.srcOp];
      if (src.kind != SOP_MFCC && src.kind != SOP_PLP) return fail(OSM_B200_ERR_UNSUPPORTED, "cVectorOperation: the input must be a cMfcc / cPlp level");
      rt.vSrcCol = src.outCol; rt.vN = src.nOut; rt.vOutCol = op.outCol;
    } else if (op.kind == SOP_CENS) {
      const CensOp &co = op.cens;
      if (cens_smem_bytes(co.N, co.W) > (size_t)prop.sharedMemPerBlockOptin) return fail(OSM_B200_ERR_UNSUPPORTED, "cCens: too many chroma elements for the kernel's shared memory");
      CU(cens_configure(co.N, co.W, (size_t)prop.sharedMemPerBlockOptin));
      CU(rt.dCensWin.upload(co.win.data(), co.win.size()));
      CensParams &cp = rt.cens;
      memset(&cp, 0, sizeof cp);
      cp.srcCol = d.ops[op.srcOp].outCol; cp.outCol = op.outCol; cp.N = co.N; cp.W = co.W;
      cp.win = rt.dCensWin.p; cp.l2norm = co.l2norm ? 1 : 0; cp.unit = co.unit;
    } else {
      const FrontEnd &fe = d.streams[op.stream].fe;
      switch (op.kind) {
        case SOP_SPECTRAL: st = build_spectral(d, op, srt, rt); break;
        case SOP_HARMONICS: st = build_harmonics(d, op, srt, rt); break;
        case SOP_PITCH: st = build_shs_chain(d, op, fe, srt, prop, rt); break;
        case SOP_JITTER: st = build_jitter(d, op, fe, rt); break;
        case SOP_PITCHACF: st = build_acf_pitch(d, op, fe, srt, rt); break;
        case SOP_TONEFILT: st = build_tonefilt_rt(d, op, fe, rt); break;
        default: st = build_time_op(d, op, fe, srt, rt); break;
      }
      if (st != OSM_B200_OK) return st;
    }
    pl->ops.push_back(std::move(rt));
  }

  if (seqLagDescOp >= 0) {
    CU(pl->auxStream.create(cudaStreamNonBlocking));
    CU(pl->evFork.create(cudaEventDisableTiming));
    CU(pl->evJoin.create(cudaEventDisableTiming));
    for (size_t i = 0; i < pl->ops.size(); i++) if (pl->ops[i].descOp == seqLagDescOp) pl->seqLagOp = (int)i;
  }
  CU(pl->dErr.reserve_exact(1));
  CU(cudaMemset(pl->dErr.p, 0, sizeof(int)));
  CU(pl->evMetaDone.create(cudaEventDisableTiming));
  CU(pl->evK0.create());
  CU(pl->evK1.create());
  CU(pl->evKm.create());
  *out = pl.release();
  return OSM_B200_OK;
} catch (const std::bad_alloc &) { return fail(OSM_B200_ERR_NOMEM, "out of host memory"); }
catch (const std::exception &e) { return fail(OSM_B200_ERR_INVALID, e.what()); }

void osm_b200_plan_destroy(osm_b200_plan *pl)
{
  if (!pl) return;
  delete pl;
}

int32_t osm_b200_plan_num_elements(const osm_b200_plan *pl) { return pl ? pl->d.nOut : 0; }

const char *osm_b200_plan_element_name(const osm_b200_plan *pl, int32_t idx)
{
  if (!pl || idx < 0 || idx >= (int)pl->d.names.size()) return nullptr;
  return pl->d.names[idx].c_str();
}

// a cCens level's period is its input's times downsampleRatio; its rows keep the time stamps of their input rows (lld/cens.cpp:107-114,
// core/vectorProcessor.cpp:308), so osm_b200_plan_row_time does not scale
double osm_b200_plan_frame_period(const osm_b200_plan *pl) { return pl ? pl->d.fe0().frameStepSec * (double)pl->d.periodScale : 0.0; }
double osm_b200_plan_row_time(const osm_b200_plan *pl, int64_t r)
{
  if (!pl) return 0.0;
  const FrontEnd &fe = pl->d.fe0();
  if (fe.rowSampleStep > 0) return (double)(r * fe.rowSampleStep) * (1.0 / fe.sampleRate);
  if (fe.frameCenter == 0 && fe.timeOffset == 0.0) return (double)r * fe.frameStepSec;
  // a centred frame carries the time of its first sample read (clamped at the input start) + frameCenter
  // (core/winToVecProcessor.cpp:1076-1079, core/dataMemoryLevel.cpp:1651-1697); a time of exactly 0 is replaced by
  // r * frame period when the frame is written (core/dataMemoryLevel.cpp:1211-1212), which `right` gives its padded frames
  const long long s0 = frame_first_sample(r, fe.frameStep, fe.frameCenter);
  const double t = (double)(s0 > 0 ? s0 : 0) * (1.0 / fe.sampleRate) + fe.timeOffset;
  return t == 0.0 ? (double)r * fe.frameStepSec : t;
}
int32_t osm_b200_plan_frame_size_samples(const osm_b200_plan *pl) { return pl ? pl->d.fe0().frameSize : 0; }
int32_t osm_b200_plan_frame_step_samples(const osm_b200_plan *pl) { return pl ? pl->d.fe0().frameStep : 0; }
int32_t osm_b200_plan_fft_size(const osm_b200_plan *pl) { return pl ? pl->d.fe0().nfft : 0; }

int64_t osm_b200_plan_num_frames(const osm_b200_plan *pl, int64_t n) { return pl ? desc_num_frames(pl->d, n) : 0; }

int64_t osm_b200_plan_num_time_frames(const osm_b200_plan *pl, int64_t n)
{
  if (!pl || pl->d.groups.empty()) return 0;
  const OutGroup &g = pl->d.groups[0];
  int64_t t = desc_num_static_frames(pl->d, g.stream, n);
  for (int ls : g.limitStreams) t = std::min<int64_t>(t, desc_num_static_frames(pl->d, ls, n));
  return t < 0 ? 0 : t;
}

osm_b200_status osm_b200_plan_frame_offsets(const osm_b200_plan *pl, const int64_t *utt_offsets, int32_t n_utt,
                                            int64_t *frame_offsets)
{
  if (!pl || !utt_offsets || !frame_offsets || n_utt < 0) return fail(OSM_B200_ERR_INVALID, "null argument");
  frame_offsets[0] = 0;
  for (int u = 0; u < n_utt; u++) {
    if (utt_offsets[u + 1] < utt_offsets[u]) return fail(OSM_B200_ERR_INVALID, "utt_offsets must be non-decreasing");
    frame_offsets[u + 1] = frame_offsets[u] + desc_num_frames(pl->d, utt_offsets[u + 1] - utt_offsets[u]);
  }
  return OSM_B200_OK;
}

// (re)build the per-batch tables when the utterance layout changed
static osm_b200_status prepare_batch(osm_b200_plan *pl, const int64_t *uttOff, int nUtt, const int64_t *frameOff,
                                     cudaStream_t st)
{
  const PlanDesc &d = pl->d;
  const bool same = (int)pl->cachedUttOff.size() == nUtt + 1 &&
                    memcmp(pl->cachedUttOff.data(), uttOff, sizeof(int64_t) * (nUtt + 1)) == 0;
  if (!same) {
    // the host tables below are rewritten in place: until the rebuild has completed no layout counts as cached (a rebuild that
    // fails half way must not be mistaken for the previous one)
    pl->cachedUttOff.clear();
    if (pl->metaPending) { CU(cudaEventSynchronize(pl->evMetaDone)); pl->metaPending = false; }
    const size_t nm = (size_t)(nUtt + 1);
    CU(pl->hMeta.reserve(3 * nm));
    long long *hU = pl->hMeta.p, *hR = hU + nm, *hS = hR + nm;
    const int PR = pl->pp.rows;
    const int KT = lld_max_chunk_tiles();
    const bool needPost = pl->pp.nGroups > 0 && !pl->fused;
    size_t nPost = 0;
    pl->uttPost0.assign(nm, 0);
    hR[0] = 0; hS[0] = 0;
    for (int u = 0; u < nUtt; u++) {
      if (uttOff[u + 1] < uttOff[u]) return fail(OSM_B200_ERR_INVALID, "utt_offsets must be non-decreasing");
      const int64_t L = uttOff[u + 1] - uttOff[u];
      hU[u] = uttOff[u];
      hR[u + 1] = hR[u] + desc_num_frames(d, L);
      hS[u + 1] = hS[u] + desc_max_static_frames(d, L);
      pl->uttPost0[u] = (int32_t)nPost;
      if (needPost) nPost += (size_t)((hR[u + 1] - hR[u] + PR - 1) / PR);
    }
    hU[nUtt] = uttOff[nUtt];
    pl->uttPost0[nUtt] = (int32_t)nPost;
    CU(pl->hPost.reserve(nPost + 1));
    {
      size_t ti = 0;
      if (needPost)
        for (int u = 0; u < nUtt; u++) {
          const int64_t To = hR[u + 1] - hR[u];
          for (int64_t r0 = 0; r0 < To; r0 += PR) pl->hPost.p[ti++] = TileRef{u, (int32_t)r0};
        }
    }
    pl->nPostTiles = nPost;
    pl->totalWork = 0;
    // per stream: chunks for lld_kernel, tiles for the standalone ops
    for (size_t si = 0; si < pl->st.size(); si++) {
      StreamRt &rt = pl->st[si];
      const int F = rt.tileF, H = rt.kp.halo;
      std::vector<ChunkRef> chunks;
      std::vector<OpTile> tiles;
      rt.uttChunk0.assign(nm, 0); rt.uttTile0.assign(nm, 0);
      std::vector<int64_t> T(nUtt);
      for (int u = 0; u < nUtt; u++) T[u] = desc_num_static_frames(d, (int)si, uttOff[u + 1] - uttOff[u]);
      if (rt.runLld) {
        // one run of chunks per resident CTA of the instance the launch will select (same parameters as launch_range)
        cut_chunks(T.data(), nUtt, F, H, KT, 0, chunks, rt.uttChunk0.data(), rt.uttTile0.data());
        if (rt.kp.opKind < 0 || d.streams[si].dumpMag)
          CU(rt.dMag.reserve((size_t)rt.uttTile0[nUtt] * d.streams[si].fe.nBins * F + 64));
        LldParams kq = rt.kp;
        kq.magOut = d.streams[si].dumpMag ? rt.dMag.p : nullptr;
        LldLaunchInfo li{};
        CU(launch_lld(kq, d.streams[si].fe.nfft, pl->numSMs, st, &li, false));
        rt.lldCtas = std::max(li.grid, 1);
        rt.ctaTiles = (int)balanced_chunks(T.data(), nUtt, F, H, KT, rt.lldCtas, chunks, rt.uttChunk0.data(), rt.uttTile0.data());
      } else {
        cut_chunks(T.data(), nUtt, F, H, KT, 0, chunks, rt.uttChunk0.data(), rt.uttTile0.data());
      }
      if (rt.needTiles)
        for (int u = 0; u < nUtt; u++)
          for (int64_t f0 = 0; f0 < T[u]; f0 += F)
            tiles.push_back(OpTile{u, (int32_t)f0, (int32_t)std::min<int64_t>(F, T[u] - f0), f0 > 0 ? 1 : 0});
      rt.nChunks = rt.runLld ? chunks.size() - 1 : 0;
      rt.nTiles = tiles.size();
      pl->totalWork += rt.nChunks + rt.nTiles;
      if (rt.runLld) {
        CU(rt.hChunks.reserve(chunks.size()));
        memcpy(rt.hChunks.p, chunks.data(), chunks.size() * sizeof(ChunkRef));
        CU(rt.dChunks.reserve(chunks.size()));
        CU(cudaMemcpyAsync(rt.dChunks.p, rt.hChunks.p, chunks.size() * sizeof(ChunkRef), cudaMemcpyHostToDevice, st));
      }
      if (rt.needTiles) {
        CU(rt.hTiles.reserve(tiles.size() + 1));
        if (!tiles.empty()) memcpy(rt.hTiles.p, tiles.data(), tiles.size() * sizeof(OpTile));
        CU(rt.dTiles.reserve(tiles.size() + 1));
        if (!tiles.empty()) CU(cudaMemcpyAsync(rt.dTiles.p, rt.hTiles.p, tiles.size() * sizeof(OpTile), cudaMemcpyHostToDevice, st));
      }
    }
    // cTonefilt segments: an utterance of up to kTfWhole rows is one segment, a longer one is cut every kTfSeg rows (the cut depends
    // on the utterance alone: its rows do not depend on the batch)
    for (OpRt &o : pl->ops) {
      if (o.kind != SOP_TONEFILT) continue;
      constexpr int64_t kTfWhole = 1024, kTfSeg = 128;
      std::vector<ChunkRef> segs;
      o.uttSeg0.assign(nm, 0);
      for (int u = 0; u < nUtt; u++) {
        o.uttSeg0[u] = (int32_t)segs.size();
        const int64_t Tu = desc_num_static_frames(d, o.stream, uttOff[u + 1] - uttOff[u]);
        const int64_t step = Tu <= kTfWhole ? kTfWhole : kTfSeg;
        for (int64_t a = 0; a < Tu; a += step) segs.push_back(ChunkRef{u, (int32_t)a, (int32_t)std::min<int64_t>(a + step, Tu), 0, 0});
      }
      o.uttSeg0[nUtt] = (int32_t)segs.size();
      const size_t ns = segs.size();
      CU(o.hSegs.reserve(ns + 1));
      if (ns) memcpy(o.hSegs.p, segs.data(), ns * sizeof(ChunkRef));
      CU(o.dSegs.reserve(ns + 1));
      if (ns) CU(cudaMemcpyAsync(o.dSegs.p, o.hSegs.p, ns * sizeof(ChunkRef), cudaMemcpyHostToDevice, st));
      CU(o.dUttSeg0.reserve(nm));
      CU(cudaMemcpyAsync(o.dUttSeg0.p, o.uttSeg0.data(), nm * sizeof(int32_t), cudaMemcpyHostToDevice, st));
      CU(o.dAgg.reserve(ns * o.tf.nNotes + 1));
      CU(o.dCin.reserve(ns * o.tf.nNotes + 1));
      pl->totalWork += ns;
    }
    for (OpRt &o : pl->ops) {
      if (o.kind != SOP_CENS) continue;
      std::vector<OpTile> tiles;
      o.uttTile0.assign(nm, 0);
      for (int u = 0; u < nUtt; u++) {
        o.uttTile0[u] = (int32_t)tiles.size();
        const int64_t Tu = desc_num_static_frames(d, o.stream, uttOff[u + 1] - uttOff[u]);
        for (int64_t a = 0; a < Tu; a += kCensRows) tiles.push_back(OpTile{u, (int32_t)a, (int32_t)std::min<int64_t>(kCensRows, Tu - a), 0});
      }
      o.uttTile0[nUtt] = (int32_t)tiles.size();
      CU(o.hCensTiles.reserve(tiles.size() + 1));
      if (!tiles.empty()) memcpy(o.hCensTiles.p, tiles.data(), tiles.size() * sizeof(OpTile));
      CU(o.dCensTiles.reserve(tiles.size() + 1));
      if (!tiles.empty()) CU(cudaMemcpyAsync(o.dCensTiles.p, o.hCensTiles.p, tiles.size() * sizeof(OpTile), cudaMemcpyHostToDevice, st));
      pl->totalWork += tiles.size();
    }
    pl->totalRows = hR[nUtt];
    pl->totalStat = hS[nUtt];
    pl->totalSamples = uttOff[nUtt];
    CU(pl->dMeta.reserve(3 * nm));
    CU(pl->dPost.reserve(nPost + 1));
    CU(cudaMemcpyAsync(pl->dMeta.p, pl->hMeta.p, 3 * nm * sizeof(long long), cudaMemcpyHostToDevice, st));
    if (nPost) CU(cudaMemcpyAsync(pl->dPost.p, pl->hPost.p, nPost * sizeof(TileRef), cudaMemcpyHostToDevice, st));
    CU(cudaEventRecord(pl->evMetaDone, st));
    pl->metaPending = true;
    pl->cachedUttOff.assign(uttOff, uttOff + nUtt + 1);
  }
  if (frameOff) {
    // the caller's row offsets must be the ones the plan derives (bit-exact integer rule)
    const size_t nm = (size_t)(nUtt + 1);
    const long long *hR = pl->hMeta.p + nm;
    for (int u = 0; u <= nUtt; u++)
      if ((long long)frameOff[u] != hR[u]) return fail(OSM_B200_ERR_INVALID, "frame_offsets do not match osm_b200_plan_frame_offsets()");
  }
  return OSM_B200_OK;
}

static cudaError_t prof_mark(osm_b200_plan *pl, const char *name, cudaStream_t st)
{
  if (!pl->profile) return cudaSuccess;
  if (pl->profN >= (int)pl->profEv.size()) {
    CudaEvent e;
    cudaError_t r = e.create();
    if (r != cudaSuccess) return r;
    pl->profEv.push_back(std::move(e));
    pl->profName.push_back(name);
  }
  pl->profName[pl->profN] = name;
  return cudaEventRecord(pl->profEv[pl->profN++], st);
}
#define PROF(name) CU(prof_mark(pl, name, st))

// launch the kernels for utterances [u0, u1) of the prepared batch
static osm_b200_status launch_range(osm_b200_plan *pl, const void *d_pcm, float *d_out, int n_utt, int u0, int u1,
                                    cudaStream_t st)
{
  const PlanDesc &d = pl->d;
  const size_t nm = (size_t)(n_utt + 1);
  const long long *dU = pl->dMeta.p, *dR = dU + nm, *dS = dR + nm;
  PROF("begin");
  const bool f32in = d.fe0().format != OSM_B200_PCM_S16;
  if (f32in) {
    // inputs in another format than 16-bit integer: one conversion pass into mono floats (the caller reserved dPcmF)
    const long long *hU = pl->hMeta.p;
    const long long f0 = hU[u0], f1 = hU[u1];
    const int nc = d.fe0().nChan;
    if (f1 > f0) {
      pcm_convert_kernel<<<(unsigned)((f1 - f0 + 255) / 256), 256, 0, st>>>(
          reinterpret_cast<const unsigned char *>(d_pcm) + (size_t)f0 * nc * sample_bytes(d.fe0().format), d.fe0().format, nc, f1 - f0, pl->dPcmF.p + f0);
      CU(cudaGetLastError());
      pl->lastLaunches++;
    }
    d_pcm = pl->dPcmF.p;
    PROF("pcm_convert_kernel");
  }
  // 1. per stream: FFT front end (+ fused band op / magnitude dump)
  for (size_t si = 0; si < pl->st.size(); si++) {
    StreamRt &rt = pl->st[si];
    if (!rt.runLld) continue;
    const int c0 = rt.uttChunk0[u0], c1 = rt.uttChunk0[u1];
    if (c1 <= c0) continue;
    const long long *hS = pl->hMeta.p + 2 * nm;
    const long long row0 = hS[u0], row1 = hS[u1];
    for (size_t j = 0; j <= rt.extra.size(); j++) {
      PassRt &pr = j == 0 ? rt.pass0x : rt.extra[j - 1];
      LldParams kp = j == 0 ? rt.kp : pr.kp;
      kp.pcm = reinterpret_cast<const int16_t *>(d_pcm);
      kp.uttOff = dU;
      kp.chunks = rt.dChunks.p + c0;
      kp.nChunks = c1 - c0;
      {
        // the whole batch runs the schedule prepare_batch cut; a part of it (run_host's pieces) is dealt over the
        // resident CTAs in runs of whole chunks
        const int64_t W = rt.hChunks.p[c1].w0 - rt.hChunks.p[c0].w0;
        kp.ctaTiles = (c0 == 0 && c1 == (int)rt.nChunks) ? rt.ctaTiles : (int)((W + rt.lldCtas - 1) / rt.lldCtas);
        kp.nRuns = (int)((W + kp.ctaTiles - 1) / kp.ctaTiles);
      }
      kp.magOut = (j == 0 && d.streams[si].dumpMag) ? rt.dMag.p : nullptr;
      if (pl->staticDirect) {
        kp.out = d_out; kp.outStride = d.nOut; kp.outCol = pl->identityOutCol; kp.rowOff = dR;
      } else {
        kp.out = pl->dStat.p; kp.outStride = d.nStatic; kp.rowOff = dS;
        kp.outCol = pr.op >= 0 ? d.ops[pr.op].outCol : 0;
      }
      if (pr.rasta) {
        CU(pr.dBand.reserve((size_t)pl->totalStat * kp.nBands + 64));
        kp.out = pr.dBand.p; kp.outStride = kp.nBands; kp.outCol = 0; kp.rowOff = dS;
      }
      CU(launch_lld(kp, d.streams[si].fe.nfft, pl->numSMs, st, &pl->lastInfo, true));
      pl->lastLaunches++;
      PROF("lld_kernel");
      if (pr.rasta) {
        RastaParams rp = pr.rp;
        rp.band = pr.dBand.p; rp.uttOff = dU; rp.statOff = dS;
        CU(launch_rasta(rp, u0, u1, st));
        PROF("rasta_kernel");
        CU(launch_plp_tail(pr.tail, pr.dBand.p, pl->dStat.p, d.nStatic, d.ops[pr.op].outCol, row0, row1, st));
        pl->lastLaunches += 2;
        PROF("plp_tail_kernel");
      }
    }
  }
  if (u0 == 0) CU(cudaEventRecord(pl->evKm, st));
  // 2. standalone ops
  bool forked = false;
  for (OpRt &o : pl->ops) {
    StreamRt &rt = pl->st[o.stream];
    if ((o.kind == SOP_PITCH || o.kind == SOP_JITTER) && pl->auxStream && !forked && !pl->profile) {
      // everything the chain reads (magnitude level, selector energy) has been launched on `st` by now
      CU(cudaEventRecord(pl->evFork, st));
      CU(cudaStreamWaitEvent(pl->auxStream, pl->evFork, 0));
      forked = true;
    }
    if (o.kind == SOP_HARMONICS || o.kind == SOP_CENS) continue;   // read the columns of other ops: launched after the join below
    if (o.kind == SOP_TONEFILT) {
      const int s0 = o.uttSeg0[u0], s1 = o.uttSeg0[u1];
      if (s1 <= s0) continue;
      bool carry = false;
      for (int u = u0; u < u1 && !carry; u++) carry = o.uttSeg0[u + 1] - o.uttSeg0[u] > 1;
      TonefiltParams tp = o.tf;
      tp.tp.pcm = reinterpret_cast<const int16_t *>(d_pcm);
      tp.tp.uttOff = dU; tp.tp.statOff = dS; tp.tp.stat = pl->dStat.p;
      tp.segs = o.dSegs.p + s0; tp.nSegs = s1 - s0;
      tp.agg = o.dAgg.p + (size_t)s0 * tp.nNotes; tp.cin = o.dCin.p + (size_t)s0 * tp.nNotes;
      CU(launch_tonefilt(tp, o.dUttSeg0.p, u0, u1, carry, st));
      pl->lastLaunches += carry ? 3 : 1;
      PROF("tonefilt_kernel");
      continue;
    }
    cudaStream_t ks = (forked && (o.kind == SOP_PITCH || o.kind == SOP_JITTER)) ? pl->auxStream : st;
    if (o.kind == SOP_VECOP) {
      const long long *hS = pl->hMeta.p + 2 * nm;
      CU(launch_vecop_ll1(pl->dStat.p, d.nStatic, o.vSrcCol, o.vN, o.vOutCol, hS[u0], hS[u1], st));
      pl->lastLaunches++;
      PROF("vecop_kernel");
      continue;
    }
    const int t0 = rt.uttTile0[u0], t1 = rt.uttTile0[u1];
    if (t1 <= t0) continue;
    if (o.kind == SOP_MAG) {
      CU(launch_mag_rows(rt.dMag.p + (size_t)t0 * o.vN * rt.tileF, rt.dTiles.p + t0, t1 - t0, rt.tileF, o.vN, dS,
                         pl->dStat.p, d.nStatic, o.vOutCol, st, o.magMode, o.magN, o.magDbNorm, o.magMinDb));
      pl->lastLaunches++;
      PROF("mag_rows_kernel");
      continue;
    }
    if (o.kind == SOP_SPECTRAL) {
      SpectralParams sp = o.sp;
      sp.mag = rt.dMag.p + (size_t)t0 * sp.nSrc * sp.F;
      sp.tiles = rt.dTiles.p + t0; sp.nTiles = t1 - t0;
      sp.statOff = dS; sp.stat = pl->dStat.p;
      CU(launch_spectral(sp, st, &pl->lastSpecStaged, &pl->lastSpecSmem));
      PROF("spectral_kernel");
    } else if (o.kind == SOP_PITCH) {
      ShsParams sh = o.shs;
      CU(o.dShs.reserve((size_t)pl->totalStat * sh.nShsCols + 64));
      CU(o.dLag.reserve((size_t)n_utt + 64));
      sh.mag = rt.dMag.p + (size_t)t0 * sh.nMag * sh.F;
      sh.tiles = rt.dTiles.p + t0; sh.nTiles = t1 - t0;
      sh.statOff = dS; sh.shs = o.dShs.p;
      CU(launch_shs(sh, ks));
      PROF("shs_kernel");
      if (d.ops[o.descOp].chain.shsOnly) {
        // the op's output is the cPitchShs level: its rows (indexed by statOff like dStat) into the op's static columns
        const long long *hS = pl->hMeta.p + 2 * nm;
        const long long r0 = hS[u0], nr = hS[u1] - hS[u0];
        if (nr > 0)
          CU(cudaMemcpy2DAsync(pl->dStat.p + (size_t)r0 * d.nStatic + d.ops[o.descOp].outCol, (size_t)d.nStatic * sizeof(float),
                               o.dShs.p + (size_t)r0 * sh.nShsCols, (size_t)sh.nShsCols * sizeof(float), (size_t)sh.nShsCols * sizeof(float),
                               (size_t)nr, cudaMemcpyDeviceToDevice, ks));
        pl->lastLaunches++;
        continue;
      }
      ViterbiParams vp = o.vit;
      vp.shs = o.dShs.p; vp.uttOff = dU; vp.statOff = dS; vp.stat = pl->dStat.p; vp.lag = o.dLag.p;
      CU(launch_viterbi(vp, u0, u1, ks));
      pl->lastLaunches++;
      PROF("viterbi_kernel");
    } else if (o.kind == SOP_JITTER) {
      JitterParams jp = o.jit;
      jp.pcm = reinterpret_cast<const int16_t *>(d_pcm);
      jp.uttOff = dU; jp.statOff = dS; jp.stat = pl->dStat.p; jp.errFlag = pl->dErr.p;
      CU(launch_jitter(jp, u0, u1, ks));
      PROF("jitter_kernel");
    } else if (o.kind == SOP_PITCHACF) {
      AcfPitchParams ap = o.ap;
      CU(o.dRaw.reserve((size_t)pl->totalStat + 64));
      ap.mag = rt.dMag.p + (size_t)t0 * ap.nSrc * ap.F;
      ap.tiles = rt.dTiles.p + t0; ap.nTiles = t1 - t0;
      ap.statOff = dS; ap.uttOff = dU; ap.raw = o.dRaw.p; ap.stat = pl->dStat.p; ap.nUtt = n_utt;
      CU(launch_acf_pitch(ap, st));
      PROF("acf_pitch_kernel");
      CU(launch_pitch_smooth(ap, u0, u1, st));
      pl->lastLaunches++;
      PROF("pitch_smooth_kernel");
    } else {
      TimeOpParams tp = o.tp;
      tp.pcm = reinterpret_cast<const int16_t *>(d_pcm);
      tp.uttOff = dU; tp.statOff = dS;
      tp.tiles = rt.dTiles.p + t0; tp.nTiles = t1 - t0;
      tp.stat = pl->dStat.p;
      if (o.kind == SOP_FORMANT) { FormantParams fp = o.fmt; fp.tp = tp; CU(launch_formant(fp, st)); PROF("formant_kernel"); }
      else if (o.kind == SOP_LPC) { LpcParams lp = o.lpc; lp.tp = tp; CU(launch_lpc(lp, st)); PROF("lpc_kernel"); }
      else {
        CU(o.kind == SOP_ENERGY ? launch_energy(tp, st) : (o.kind == SOP_INTENSITY ? launch_intensity(tp, st) : launch_mzcr(tp, st)));
        PROF(o.kind == SOP_ENERGY ? "energy_kernel" : (o.kind == SOP_INTENSITY ? "intensity_kernel" : "mzcr_kernel"));
      }
    }
    pl->lastLaunches++;
  }
  if (forked) {
    CU(cudaEventRecord(pl->evJoin, pl->auxStream));
    CU(cudaStreamWaitEvent(st, pl->evJoin, 0));
  }
  for (OpRt &o : pl->ops) {
    if (o.kind == SOP_CENS) {                           // the chroma columns (lld_kernel or tonefilt_kernel, both on `st`)
      const int t0 = o.uttTile0[u0], t1 = o.uttTile0[u1];
      if (t1 <= t0) continue;
      CensParams cp = o.cens;
      cp.stat = pl->dStat.p; cp.statStride = d.nStatic; cp.statOff = dS;
      cp.tiles = o.dCensTiles.p + t0; cp.nTiles = t1 - t0;
      CU(launch_cens(cp, st));
      pl->lastLaunches++;
      PROF("cens_kernel");
      continue;
    }
    if (o.kind != SOP_HARMONICS) continue;
    StreamRt &rt = pl->st[o.stream];
    const int t0 = rt.uttTile0[u0], t1 = rt.uttTile0[u1];
    if (t1 <= t0) continue;
    HarmonicsParams hp = o.hrm;
    hp.mag = rt.dMag.p + (size_t)t0 * hp.nb * hp.F;
    hp.tiles = rt.dTiles.p + t0; hp.nTiles = t1 - t0;
    hp.statOff = dS; hp.stat = pl->dStat.p;
    CU(launch_harmonics(hp, st));
    pl->lastLaunches++;
    PROF("harmonics_kernel");
  }
  // 3. temporal stages + assembly of the output rows
  if (pl->pp.nGroups > 0 && !pl->fused) {
    PostParams pp = pl->pp;
    if (pl->staticDirect) { pp.stat = d_out + pl->identityOutCol; pp.statStride = d.nOut; pp.statOff = dR; }
    else { pp.stat = pl->dStat.p; pp.statStride = d.nStatic; pp.statOff = dS; }
    pp.out = d_out; pp.outStride = d.nOut; pp.rowOff = dR; pp.uttOff = dU; pp.nUtt = n_utt;
    pp.tiles = pl->dPost.p + pl->uttPost0[u0]; pp.nTiles = pl->uttPost0[u1] - pl->uttPost0[u0];
    pp.means = nullptr;
    if (pl->needMeans) {
      CU(pl->dMeans.reserve((size_t)n_utt * d.nStatic + 64));
      CU(launch_cms_means(pp, pl->dMeans.p, u0, u1, st));
      pl->lastLaunches++;
      PROF("cms_means_kernel");
      pp.means = pl->dMeans.p;
    }
    if (pp.nTiles > 0) {
      CU(launch_post(pp, st));
      pl->lastLaunches++;
      PROF("post_kernel");
    }
  }
  // 4. levels behind the Viterbi-smoothed pitch chain
  if (pl->sp.nGroups > 0 && pl->seqLagOp >= 0) {
    SeqPostParams sq = pl->sp;
    sq.stat = pl->dStat.p; sq.statStride = d.nStatic; sq.statOff = dS; sq.rowOff = dR; sq.uttOff = dU;
    sq.out = d_out; sq.outStride = d.nOut; sq.lag = pl->ops[pl->seqLagOp].dLag.p;
    CU(launch_seq_post(sq, u0, u1, st));
    pl->lastLaunches++;
    PROF("seq_post_kernel");
  }
  return OSM_B200_OK;
}

// pcm_pack_kernel over the prepared batch: the padded batch d_pcm ([n_utt][nChan][stride]) into pl->dPadPcm
static osm_b200_status launch_pack(osm_b200_plan *pl, const void *d_pcm, int64_t stride, int n_utt, int64_t maxLen, cudaStream_t st)
{
  const int nc = pl->d.fe0().nChan, sz = sample_bytes(pl->d.fe0().format);
  CU(pl->dPadPcm.reserve((size_t)pl->totalSamples * nc * sz + 16));
  if (maxLen == 0) return OSM_B200_OK;
  const int tileF = nc == 1 ? kPackMonoFrames : std::max(1, std::min(kPackMonoFrames, kPackTileBytes / (nc * sz)));
  const size_t smem = nc == 1 ? 0 : (size_t)tileF * nc * sz;
  if (smem > 48 * 1024) return fail(OSM_B200_ERR_UNSUPPORTED, "padded device batch: too many channels for the packing kernel's tile");
  const dim3 grid((unsigned)((maxLen + tileF - 1) / tileF), (unsigned)std::min(n_utt, 65535));
  if (sz == 2)
    pcm_pack_kernel<uint16_t><<<grid, kPackThreads, smem, st>>>(static_cast<const uint16_t *>(d_pcm), stride, nc, tileF, pl->dMeta.p, n_utt,
                                                                reinterpret_cast<uint16_t *>(pl->dPadPcm.p));
  else
    pcm_pack_kernel<uint32_t><<<grid, kPackThreads, smem, st>>>(static_cast<const uint32_t *>(d_pcm), stride, nc, tileF, pl->dMeta.p, n_utt,
                                                                reinterpret_cast<uint32_t *>(pl->dPadPcm.p));
  CU(cudaGetLastError());
  pl->lastLaunches++;
  return OSM_B200_OK;
}

// run_device on a packed batch (padStride < 0), or on a padded one that is packed first (padStride = its stride, maxLen = the longest
// utterance)
static osm_b200_status run_device_impl(osm_b200_plan *pl, const void *d_pcm, const int64_t *utt_offsets, int32_t n_utt,
                                       const int64_t *frame_offsets, float *d_out, void *stream, int64_t padStride, int64_t maxLen)
{
  if (!pl || !utt_offsets || n_utt < 0) return fail(OSM_B200_ERR_INVALID, "null argument");
  if (pl->device < 0) return fail(OSM_B200_ERR_CUDA, "description-only plan (device < 0) cannot run; no CPU fallback");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CU(cudaSetDevice(pl->device));
  pl->lastLaunches = 0;
  pl->lastInfo = LldLaunchInfo{};
  pl->lastPieces = 0; pl->lastSpecStaged = -1; pl->lastSpecSmem = 0;
  pl->timed = false;
  pl->profN = 0;
  osm_b200_status s = prepare_batch(pl, utt_offsets, n_utt, frame_offsets, st);
  if (s != OSM_B200_OK) return s;
  if (pl->totalRows == 0 || pl->totalWork == 0) return OSM_B200_OK;
  if (!d_pcm || !d_out) return fail(OSM_B200_ERR_INVALID, "null device buffer");
  if (pl->d.fe0().format != OSM_B200_PCM_S16) CU(pl->dPcmF.reserve((size_t)utt_offsets[n_utt] + 16));
  if (!pl->staticDirect) CU(pl->dStat.reserve((size_t)pl->totalStat * pl->d.nStatic + 64));
  if (padStride >= 0) {
    s = launch_pack(pl, d_pcm, padStride, n_utt, maxLen, st);
    if (s != OSM_B200_OK) return s;
    d_pcm = pl->dPadPcm.p;
  }
  CU(cudaEventRecord(pl->evK0, st));
  s = launch_range(pl, d_pcm, d_out, n_utt, 0, n_utt, st);
  if (s != OSM_B200_OK) return s;
  CU(cudaEventRecord(pl->evK1, st));
  pl->timed = true;
  return OSM_B200_OK;
}

osm_b200_status osm_b200_plan_run_device(osm_b200_plan *pl, const void *d_pcm, const int64_t *utt_offsets,
                                         int32_t n_utt, const int64_t *frame_offsets, float *d_out, void *stream)
{
  return run_device_impl(pl, d_pcm, utt_offsets, n_utt, frame_offsets, d_out, stream, -1, 0);
}

// no exception crosses the C boundary (the utterance offsets are a host vector)
osm_b200_status osm_b200_plan_run_device_padded(osm_b200_plan *pl, const void *d_pcm, int64_t stride, const int64_t *lengths,
                                                int32_t n_utt, const int64_t *frame_offsets, float *d_out, void *stream)
try {
  if (!pl || !lengths || n_utt < 0) return fail(OSM_B200_ERR_INVALID, "null argument");
  const int format = pl->d.fe0().format;
  if (format != OSM_B200_PCM_S16 && format != OSM_B200_PCM_F32)
    return fail(OSM_B200_ERR_INVALID, "a padded device batch holds int16 (OSM_B200_PCM_S16) or float32 (OSM_B200_PCM_F32) samples");
  std::vector<int64_t> off((size_t)n_utt + 1, 0);
  int64_t maxLen = 0;
  for (int u = 0; u < n_utt; u++) {
    if (lengths[u] < 0 || lengths[u] > stride)
      return fail(OSM_B200_ERR_INVALID, "utterance " + std::to_string(u) + ": length " + std::to_string(lengths[u]) + " outside 0 .. stride (" +
                                            std::to_string(stride) + ")");
    off[u + 1] = off[u] + lengths[u];
    maxLen = std::max(maxLen, lengths[u]);
  }
  return run_device_impl(pl, d_pcm, off.data(), n_utt, frame_offsets, d_out, stream, stride, maxLen);
} catch (const std::bad_alloc &) { return fail(OSM_B200_ERR_NOMEM, "out of host memory"); }

// Host buffers.  The batch is cut into pieces of whole utterances and pipelined over three
// streams: H2D of piece k+1, kernels of piece k and D2H of piece k-1 overlap (the two copy
// directions use separate copy engines).  Host memory should be pinned (cudaHostAlloc /
// torch pin_memory) for the copies to be asynchronous; pageable memory works but serialises.
static osm_b200_status run_host_impl(osm_b200_plan *pl, const void *pcm, const int64_t *utt_offsets, int32_t n_utt,
                                     const int64_t *frame_offsets, float *out, bool resident)
{
  if (!pl || !utt_offsets || n_utt < 0) return fail(OSM_B200_ERR_INVALID, "null argument");
  if (pl->device < 0) return fail(OSM_B200_ERR_CUDA, "description-only plan (device < 0) cannot run; no CPU fallback");
  CU(cudaSetDevice(pl->device));
  if (!pl->hostStream) {
    CU(pl->hostStream.create(cudaStreamNonBlocking));
    CU(pl->h2dStream.create(cudaStreamNonBlocking));
    CU(pl->d2hStream.create(cudaStreamNonBlocking));
  }
  cudaStream_t st = pl->hostStream;
  pl->lastLaunches = 0;
  pl->lastInfo = LldLaunchInfo{};
  pl->lastPieces = 0; pl->lastSpecStaged = -1; pl->lastSpecSmem = 0;
  pl->timed = false;
  osm_b200_status s = prepare_batch(pl, utt_offsets, n_utt, frame_offsets, st);
  if (s != OSM_B200_OK) return s;
  const long long rows = pl->totalRows;
  if (rows == 0 || pl->totalWork == 0) return OSM_B200_OK;
  if (!pcm || (!out && !resident)) return fail(OSM_B200_ERR_INVALID, "null host buffer");
  const int nOut = pl->d.nOut;
  const int64_t frameBytes = (int64_t)pl->d.fe0().nChan * sample_bytes(pl->d.fe0().format);
  const int64_t totalBytes = utt_offsets[n_utt] * frameBytes;
  CU(pl->dPcm.reserve((size_t)(totalBytes + 1) / 2 + 16));
  if (pl->d.fe0().format != OSM_B200_PCM_S16) CU(pl->dPcmF.reserve((size_t)utt_offsets[n_utt] + 16));
  CU(pl->dOut.reserve((size_t)rows * nOut));
  if (!pl->staticDirect) CU(pl->dStat.reserve((size_t)pl->totalStat * pl->d.nStatic + 64));
  const long long *hR = pl->hMeta.p + (size_t)(n_utt + 1);

  // pieces of ~24 MB of PCM, at most 16, cut at utterance boundaries
  // (plans with per-utterance sequential kernels -- Viterbi, jitter -- get their parallelism from the number of
  // utterances in flight: fewer, larger pieces)
  const int64_t maxPieces = pl->sp.nGroups > 0 ? 4 : 16;
  int nPieces = (int)std::min<int64_t>(maxPieces, std::max<int64_t>(1, totalBytes / (24 << 20)));
  if (nPieces > n_utt) nPieces = n_utt;
  while ((int)pl->evPiece.size() < 2 * nPieces) {
    CudaEvent e;
    CU(e.create(cudaEventDisableTiming));
    pl->evPiece.push_back(std::move(e));
  }
  CU(cudaEventRecord(pl->evK0, st));
  int u0 = 0;
  for (int k = 0; k < nPieces; k++) {
    int u1 = u0;
    const int64_t target = utt_offsets[n_utt] * (int64_t)(k + 1) / nPieces;
    while (u1 < n_utt && (utt_offsets[u1 + 1] <= target || u1 == u0)) u1++;
    if (k == nPieces - 1) u1 = n_utt;
    if (u1 == u0) continue;
    const int64_t sa = utt_offsets[u0] * frameBytes, sb = utt_offsets[u1] * frameBytes;
    CU(cudaMemcpyAsync(reinterpret_cast<unsigned char *>(pl->dPcm.p) + sa, reinterpret_cast<const unsigned char *>(pcm) + sa, (size_t)(sb - sa),
                       cudaMemcpyHostToDevice, pl->h2dStream));
    CU(cudaEventRecord(pl->evPiece[2 * k], pl->h2dStream));
    CU(cudaStreamWaitEvent(st, pl->evPiece[2 * k], 0));
    s = launch_range(pl, pl->dPcm.p, pl->dOut.p, n_utt, u0, u1, st);
    if (s != OSM_B200_OK) {
      // copies of earlier pieces into the caller's buffers may still be in flight: let them land before reporting the error
      cudaStreamSynchronize(pl->h2dStream); cudaStreamSynchronize(st); cudaStreamSynchronize(pl->d2hStream);
      return s;
    }
    pl->lastPieces++;
    CU(cudaEventRecord(pl->evPiece[2 * k + 1], st));
    CU(cudaStreamWaitEvent(pl->d2hStream, pl->evPiece[2 * k + 1], 0));
    const long long ra = hR[u0], rb = hR[u1];
    if (rb > ra && out)
      CU(cudaMemcpyAsync(out + ra * nOut, pl->dOut.p + ra * nOut, (size_t)(rb - ra) * nOut * sizeof(float),
                         cudaMemcpyDeviceToHost, pl->d2hStream));
    u0 = u1;
  }
  CU(cudaEventRecord(pl->evK1, st));
  pl->timed = true;
  CU(cudaStreamSynchronize(pl->d2hStream));
  CU(cudaStreamSynchronize(st));
  return osm_b200_plan_check_device_flags(pl, st);
}

osm_b200_status osm_b200_plan_check_device_flags(osm_b200_plan *pl, void *stream)
{
  if (!pl) return fail(OSM_B200_ERR_INVALID, "null plan");
  // only cPitchJitter raises the flag: a plan without it has nothing to wait for
  if (pl->device < 0 || std::none_of(pl->ops.begin(), pl->ops.end(), [](const OpRt &o) { return o.kind == SOP_JITTER; })) return OSM_B200_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CU(cudaSetDevice(pl->device));
  int flag = 0;
  CU(cudaMemcpyAsync(&flag, pl->dErr.p, sizeof flag, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  if (flag) {
    CU(cudaMemsetAsync(pl->dErr.p, 0, sizeof(int), st));
    CU(cudaStreamSynchronize(st));
    return fail(OSM_B200_ERR_UNSUPPORTED, "cPitchJitter: a frame left the supported geometry (F0 period / read window too long for the kernel's workspace); its rows were zeroed");
  }
  return OSM_B200_OK;
}

osm_b200_status osm_b200_plan_run_host(osm_b200_plan *pl, const void *pcm, const int64_t *utt_offsets, int32_t n_utt,
                                       const int64_t *frame_offsets, float *out)
{
  return run_host_impl(pl, pcm, utt_offsets, n_utt, frame_offsets, out, false);
}

// Host PCM in, rows left in HBM: the H2D pipeline and kernels of run_host without the copy back.  *d_rows = the plan's own
// row buffer ([rows][num_elements], valid until the plan's next run): the hand-over point to a consumer that summarises the
// rows on the device (osm_b200_functionals_run_device).
osm_b200_status osm_b200_plan_run_host_resident(osm_b200_plan *pl, const void *pcm, const int64_t *utt_offsets, int32_t n_utt,
                                                const int64_t *frame_offsets, const float **d_rows)
{
  if (!d_rows) return fail(OSM_B200_ERR_INVALID, "null argument");
  *d_rows = nullptr;
  osm_b200_status s = run_host_impl(pl, pcm, utt_offsets, n_utt, frame_offsets, nullptr, true);
  if (s == OSM_B200_OK) *d_rows = pl->dOut.p;
  return s;
}

osm_b200_status osm_b200_window_table(const osm_b200_windower *w, int32_t n, float *out)
{
  if (!w || !out || n <= 0) return fail(OSM_B200_ERR_INVALID, "null argument");
  if (w->winFunc < OSM_B200_WIN_RECTANGLE || w->winFunc > OSM_B200_WIN_LANCZOS) return fail(OSM_B200_ERR_INVALID, "unknown window function");
  const double al[4] = {w->alpha0, w->alpha1, w->alpha2, w->alpha3};
  std::vector<float> t;
  build_window(w->winFunc, n, w->sigma, w->gain, t, al, w->squareRoot, std::min(std::max(w->fade, 0.0), 0.5));
  memcpy(out, t.data(), sizeof(float) * (size_t)n);
  return OSM_B200_OK;
}

osm_b200_status osm_b200_tone_tables(const osm_b200_tonespec *cfg, int32_t n_bins, double frame_size_sec, float *pitch_class_freq,
                                     int32_t *bin_key, int32_t *bin_count, float *filter_map, int32_t *fl_bin)
try {
  if (!cfg || !pitch_class_freq || !bin_key || !bin_count || !filter_map || !fl_bin || n_bins < 2 || !(frame_size_sec > 0.0))
    return fail(OSM_B200_ERR_INVALID, "bad argument");
  if (cfg->nOctaves < 1) return fail(OSM_B200_ERR_INVALID, "cTonespec.nOctaves must be >= 1");
  ToneTables t;
  std::string err;
  if (!build_tone_tables(*cfg, n_bins, frame_size_sec, t, err)) return fail(OSM_B200_ERR_UNSUPPORTED, err);
  memcpy(pitch_class_freq, t.pitchClassFreq.data(), sizeof(float) * t.pitchClassFreq.size());
  memcpy(bin_key, t.binKey.data(), sizeof(int32_t) * t.binKey.size());
  memcpy(bin_count, t.nbins.data(), sizeof(int32_t) * t.nbins.size());
  memcpy(filter_map, t.filterMap.data(), sizeof(float) * t.filterMap.size());
  fl_bin[0] = t.firstBin; fl_bin[1] = t.lastBin;
  return OSM_B200_OK;
} catch (const std::bad_alloc &) { return fail(OSM_B200_ERR_NOMEM, "out of host memory"); }

int64_t osm_b200_plan_num_frames_first_eoi(const osm_b200_plan *pl, int64_t n) { return pl ? desc_num_frames_first_eoi(pl->d, n) : 0; }
int64_t osm_b200_plan_num_frames_first_eoi_v(const osm_b200_plan *pl, int64_t n, int64_t v) { return pl ? desc_num_frames_first_eoi(pl->d, n, v) : 0; }

osm_b200_status osm_b200_plan_copy_seq_lag(osm_b200_plan *pl, int32_t *out, int32_t n_utt)
{
  if (!pl || !out || n_utt < 0) return fail(OSM_B200_ERR_INVALID, "null argument");
  for (int u = 0; u < n_utt; u++) out[u] = -1;
  if (pl->device < 0 || pl->seqLagOp < 0 || n_utt == 0) return OSM_B200_OK;
  CU(cudaSetDevice(pl->device));
  CU(cudaDeviceSynchronize());
  if (!pl->ops[pl->seqLagOp].dLag.p) return OSM_B200_OK;
  CU(cudaMemcpy(out, pl->ops[pl->seqLagOp].dLag.p, sizeof(int) * (size_t)n_utt, cudaMemcpyDeviceToHost));
  return OSM_B200_OK;
}

osm_b200_status osm_b200_plan_copy_seq_lag_stream(osm_b200_plan *pl, int32_t *out, int32_t n_utt, void *stream)
{
  if (!pl || !out || n_utt < 0) return fail(OSM_B200_ERR_INVALID, "null argument");
  for (int u = 0; u < n_utt; u++) out[u] = -1;
  if (pl->device < 0 || pl->seqLagOp < 0 || n_utt == 0 || !pl->ops[pl->seqLagOp].dLag.p) return OSM_B200_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CU(cudaSetDevice(pl->device));
  CU(cudaMemcpyAsync(out, pl->ops[pl->seqLagOp].dLag.p, sizeof(int) * (size_t)n_utt, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return OSM_B200_OK;
}

int32_t osm_b200_plan_last_launch_count(const osm_b200_plan *pl) { return pl ? pl->lastLaunches : 0; }

osm_b200_status osm_b200_plan_last_lld_launch(const osm_b200_plan *pl, const char **kernel, int32_t *grid, int64_t *n_chunks)
{
  if (!pl) return fail(OSM_B200_ERR_INVALID, "null plan");
  if (kernel) *kernel = pl->lastInfo.kernel;
  if (grid) *grid = pl->lastInfo.grid;
  if (n_chunks) *n_chunks = pl->lastInfo.nChunks;
  return OSM_B200_OK;
}

osm_b200_status osm_b200_plan_last_run_info(const osm_b200_plan *pl, int32_t *pieces, int32_t *spectral_staged, int32_t *spectral_smem)
{
  if (!pl) return fail(OSM_B200_ERR_INVALID, "null plan");
  if (pieces) *pieces = pl->lastPieces;
  if (spectral_staged) *spectral_staged = pl->lastSpecStaged;
  if (spectral_smem) *spectral_smem = pl->lastSpecSmem;
  return OSM_B200_OK;
}

int32_t osm_b200_plan_sample_frame_bytes(const osm_b200_plan *pl) { return pl ? pl->d.fe0().nChan * sample_bytes(pl->d.fe0().format) : 0; }

int32_t osm_b200_plan_take_device_flags(osm_b200_plan *pl)
{
  if (!pl || pl->device < 0 || !pl->dErr.p) return 0;
  int flag = 0;
  if (cudaSetDevice(pl->device) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) return -1;
  if (cudaMemcpy(&flag, pl->dErr.p, sizeof flag, cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  if (flag && cudaMemset(pl->dErr.p, 0, sizeof(int)) != cudaSuccess) return -1;
  return flag;
}

float osm_b200_plan_last_kernel_ms(osm_b200_plan *pl)
{
  if (!pl || !pl->timed) return -1.f;
  if (cudaEventSynchronize(pl->evK1) != cudaSuccess) return -1.f;
  float ms = -1.f;
  if (cudaEventElapsedTime(&ms, pl->evK0, pl->evK1) != cudaSuccess) return -1.f;
  return ms;
}

void osm_b200_plan_set_profiling(osm_b200_plan *pl, int32_t on) { if (pl) pl->profile = on != 0; }

int32_t osm_b200_plan_profile_count(osm_b200_plan *pl) { return (pl && pl->profN > 1) ? pl->profN - 1 : 0; }

osm_b200_status osm_b200_plan_profile_entry(osm_b200_plan *pl, int32_t idx, const char **name, float *ms)
{
  if (!pl || idx < 0 || idx + 1 >= pl->profN) return fail(OSM_B200_ERR_INVALID, "profile entry out of range");
  CU(cudaSetDevice(pl->device));
  CU(cudaEventSynchronize(pl->profEv[idx + 1]));
  float t = 0.0f;
  CU(cudaEventElapsedTime(&t, pl->profEv[idx], pl->profEv[idx + 1]));
  if (name) *name = pl->profName[idx + 1];
  if (ms) *ms = t;
  return OSM_B200_OK;
}

osm_b200_status osm_b200_plan_last_kernel_times(osm_b200_plan *pl, float *lld_ms, float *post_ms)
{
  if (!pl || !pl->timed) return fail(OSM_B200_ERR_INVALID, "no timed run");
  CU(cudaEventSynchronize(pl->evK1));
  float a = 0.f, b = 0.f;
  CU(cudaEventElapsedTime(&a, pl->evK0, pl->evKm));
  CU(cudaEventElapsedTime(&b, pl->evKm, pl->evK1));
  if (lld_ms) *lld_ms = a;
  if (post_ms) *post_ms = b;
  return OSM_B200_OK;
}

}  // extern "C"
