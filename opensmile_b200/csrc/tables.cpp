// tables.cpp -- host-side construction of the constant tables the fused kernel consumes.
// These are the "finalise time" computations of the reference's components
// (cWindower::precomputeWinFunc, cMelspec::computeFilters, cMfcc::initTables); they run once
// per plan on the CPU exactly as the reference runs them once per component instance, with
// the same float/double casting order so that the tables are bit-identical.
// Citations are relative to /root/reference/src.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "plan.hpp"
#include "formant_math.cuh"

#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif

namespace osm {

// cWindower::precomputeWinFunc (dspcore/windower.cpp:159-217) over the double tables of
// smileutil/smileUtil.c:1218-1349; the per-sample use casts to float (windower.cpp:226).
void build_window(int winFunc, int N, double sigma, double gain, std::vector<float> &out, const double *alpha, int squareRoot, double fade)
{
  std::vector<double> w(N);
  const double NN = (double)N;
  for (int n = 0; n < N; n++) {
    const double i = (double)n;
    switch (winFunc) {
      case OSM_B200_WIN_HANNING:   // smileUtil.c:1277-1288
        w[n] = 0.5 * (1.0 - cos((2.0 * M_PI * i) / (NN - 1.0)));
        break;
      case OSM_B200_WIN_HAMMING:   // smileUtil.c:1291-1303
        w[n] = 0.54 - 0.46 * cos((2.0 * M_PI * i) / (NN - 1.0));
        break;
      case OSM_B200_WIN_GAUSS: {   // smileUtil.c:1334-1349
        double s = sigma;
        if (s <= 0.0) s = 0.01;
        if (s > 0.5) s = 0.5;
        const double tmp = (i - (NN - 1.0) / 2.0) / (s * (NN - 1.0) / 2.0);
        w[n] = exp(-0.5 * (tmp * tmp));
        break;
      }
      case OSM_B200_WIN_SINE:      // smileUtil.c:1306-1317
        w[n] = sin((1.0 * M_PI * i) / (NN - 1.0));
        break;
      case OSM_B200_WIN_TRIANGLE:  // smileUtil.c:1232-1246
        w[n] = (n < N / 2) ? 2.0 * (double)(n + 1) / (double)N : 2.0 * (double)(N - n) / (double)N;
        break;
      case OSM_B200_WIN_BARTLETT:  // smileUtil.c:1261-1274
        w[n] = (n < N / 2) ? 2.0 * (double)n / (double)(N - 1)
                           : 2.0 * (double)(N - 1 - n) / (double)(N - 1);
        break;
      case OSM_B200_WIN_BLACKMAN: {   // smileUtil.c:1352-1367
        const double tmp = (2.0 * M_PI * i) / (NN - 1.0);
        w[n] = alpha[0] - alpha[1] * cos(tmp) + alpha[2] * cos(2.0 * tmp);
        break;
      }
      case OSM_B200_WIN_BLACKHARR: {  // smileUtil.c:1386-1402
        const double tmp = (2.0 * M_PI * i) / (NN - 1.0);
        w[n] = alpha[0] - alpha[1] * cos(tmp) + alpha[2] * cos(2.0 * tmp) - alpha[3] * cos(3.0 * tmp);
        break;
      }
      case OSM_B200_WIN_BARTHANN:     // smileUtil.c:1370-1383
        w[n] = alpha[0] - alpha[1] * fabs(i / (NN - 1.0) - 0.5) - alpha[2] * cos((2.0 * M_PI * i) / (NN - 1.0));
        break;
      case OSM_B200_WIN_LANCZOS: {    // smileUtil.c:1320-1331, smileDsp_lcSinc :1205-1209 (0/0 at the centre of an odd window, like the reference)
        const double y = M_PI * ((2.0 * i) / (NN - 1.0) - 1.0);
        w[n] = sin(y) / y;
        break;
      }
      default:                     // rectangle, smileUtil.c:1218-1228
        w[n] = 1.0;
        break;
    }
  }
  if (squareRoot)                  // dspcore/windower.cpp:178-188 (negative values become 0)
    for (int n = 0; n < N; n++) w[n] = w[n] >= 0.0 ? sqrt(w[n]) : 0.0;
  if (fade > 0.0) {                // :201-208
    const long fadeSize = (long)((double)N * fade);
    for (long k = 0; k < fadeSize; k++) {
      const double a = -0.5 * (cos(M_PI * (double)k / (double)fadeSize) - 1.0);
      w[k] *= a;
      w[N - k - 1] *= a;
    }
  }
  if (gain != 1.0)
    for (int n = 0; n < N; n++) w[n] *= gain;  // windower.cpp:192-196
  out.resize(N);
  for (int n = 0; n < N; n++) out[n] = (float)w[n];
}

// smileDsp_specScaleTransfFwd / Inv for SPECTSCALE_MEL (smileutil/smileUtil.c:1139-1142,1197)
static double mel_fwd(double x) { return x > 0.0 ? 1127.0 * log(1.0 + x / 700.0) : 0.0; }
static double mel_inv(double x) { return 700.0 * (exp(x / 1127.0) - 1.0); }
// smileDsp_specScaleTransfFwd / Inv (smileutil/smileUtil.c:1097-1204)
static double scale_fwd(double x, int scale, double param)
{
  switch (scale) {
    case OSM_B200_SCALE_LOG: return x > 0 ? log(x) / log(param) : 0.0;
    case OSM_B200_SCALE_SEMITONE: return x / param > 1.0 ? 12.0 * (log(x / param) / log(2.0)) : 0.0;     // smileMath_log2 = log(x) / log(2)
    case OSM_B200_SCALE_BARK: {
      if (!(x > 0)) return 0.0;
      const double zz = (26.81 / (1.0 + 1960.0 / x)) - 0.53;
      if (zz < 2) return 0.85 * zz + 0.3;
      if (zz > 20.1) return 1.22 * zz - 0.22 * 20.1;
      return zz;
    }
    case OSM_B200_SCALE_BARK_SCHROED: { if (!(x > 0)) return 0.0; const double f6 = x / 600.0; return 6.0 * log(f6 + sqrt(f6 * f6 + 1.0)); }
    case OSM_B200_SCALE_BARK_SPEEX: return 13.1 * atan(.00074 * x) + 2.24 * atan(x * x * 1.85e-8) + 1e-4 * x;
    case OSM_B200_SCALE_LINEAR: return x;
    default: return mel_fwd(x);
  }
}
static double scale_inv(double x, int scale, double param)
{
  switch (scale) {
    case OSM_B200_SCALE_LOG: return exp(x * log(param));
    case OSM_B200_SCALE_SEMITONE: return param * pow(2.0, x / 12.0);
    case OSM_B200_SCALE_BARK: {
      double zz = x;
      if (x > 20.1) zz = (x + 0.22 * 20.1) / 1.22;
      else if (x < 2) zz = (x - 0.3) / 0.85;
      const double z0 = 26.81 / (zz + 0.53);
      return z0 != 1.0 ? 1960.0 / (z0 - 1.0) : 0.0;
    }
    case OSM_B200_SCALE_BARK_SCHROED: return 600.0 * sinh(x / 6.0);
    case OSM_B200_SCALE_LINEAR: return x;
    default: return mel_inv(x);                  // mel; bark_speex has no inverse in the reference and falls through to mel (:1187-1190)
  }
}

// cMelspec::computeFilters, standard triangular bank (lldcore/melspec.cpp:184-240,391-447),
// specScale = mel (forced when htkcompatible, melspec.cpp:127-131).
void build_mel(const osm_b200_melspec &cfg, int blocksize, double frameSizeSec, MelBank &mb)
{
  const int nBands = cfg.nBands;
  const int scale = cfg.htkcompatible ? (int)OSM_B200_SCALE_MEL : cfg.specScale;     // melspec.cpp:127-131
  double param = 0.0;                                                                // :133-135
  if (scale == OSM_B200_SCALE_LOG) param = (cfg.scaleParam <= 0.0 || cfg.scaleParam == 1.0) ? 2.0 : cfg.scaleParam;   // :117-121
  else if (scale == OSM_B200_SCALE_SEMITONE) param = cfg.scaleParam;
  mb.nBands = nBands;
  mb.nBins = blocksize;
  mb.coef.assign(blocksize, 0.f);
  mb.chanMap.assign(blocksize, -3);
  mb.bandHz.assign(nBands, 0.0);
  std::vector<float> cfs(nBands + 2);

  const float N = (float)((blocksize - 1) * 2);               // :217
  const float F0 = (float)(1.0 / frameSizeSec);               // :220
  const float Fs = (float)(N / frameSizeSec);                 // :221
  const float M = (float)nBands;
  float lofreq = (float)cfg.lofreq, hifreq = (float)cfg.hifreq;  // FLOAT_DMEM members, melspec.hpp:48
  if ((lofreq < 0.0) || (lofreq > Fs / 2.0) || (lofreq > hifreq)) lofreq = 0.0;             // :224
  if ((hifreq < lofreq) || (hifreq > Fs / 2.0) || (hifreq <= 0.0)) hifreq = Fs / (float)2.0; // :226
  const float LoF = (float)scale_fwd(lofreq, scale, param);                   // :228
  const float HiF = (float)scale_fwd(hifreq, scale, param);                   // :230
  long nLoF = (long)round((double)(lofreq / F0));             // FtoN, melspec.hpp:107-110
  long nHiF = (long)round((double)(hifreq / F0));
  if (nLoF > blocksize) nLoF = blocksize;
  if (nHiF > blocksize) nHiF = blocksize;
  if (nLoF < 0) nLoF = 0;
  if (nHiF < 0) nHiF = 0;
  mb.nLo = (int)nLoF;
  mb.nHi = (int)nHiF;

  const float mBandw = (HiF - LoF) / (M + (float)1.0);        // :394
  for (int m = 0; m <= nBands + 1; m++) cfs[m] = LoF + (float)m * mBandw;   // :395-397
  for (int m = 1; m <= nBands; m++) mb.bandHz[m - 1] = scale_inv(cfs[m], scale, param);     // :408-411

  // channel map :427-438 ; NtoFmel(n,F0) = (float)fwd((float)n * F0), melspec.hpp:119-122
  int m = 0;
  for (int n = 0; n < blocksize; n++) {
    if ((n <= nLoF) || (n >= nHiF)) {
      mb.chanMap[n] = -3;
    } else {
      while (cfs[m] < (float)scale_fwd(((float)n) * F0, scale, param)) {
        if (m > nBands) break;
        m++;
      }
      mb.chanMap[n] = m - 2;
    }
  }
  // rising-slope weights :441-447
  m = 0;
  for (long n = nLoF; n < nHiF; n++) {
    const float nM = (float)scale_fwd(((float)n) * F0, scale, param);
    while ((nM > cfs[m + 1]) && (m <= nBands)) m++;
    mb.coef[n] = (cfs[m + 1] - nM) / (cfs[m + 1] - cfs[m]);
  }

  // kernel view: the visited bins nLo..nHi-1 with chanMap > -2 form nBands+1 contiguous
  // runs ("ranges"), range r holding the bins with chanMap == r-1.  The per-frame loop
  // (melspec.cpp:543-553) then is, for a bin of range r:  band[r-1] += a ; band[r] += p - a.
  mb.rangeBegin.assign(nBands + 2, 0);
  {
    int n = (int)nLoF;
    while (n < nHiF && mb.chanMap[n] <= -2) n++;  // skipped bins (chanMap -3) at the low edge
    for (int r = 0; r <= nBands; r++) {
      mb.rangeBegin[r] = n;
      while (n < nHiF && mb.chanMap[n] == r - 1) n++;
    }
    mb.rangeBegin[nBands + 1] = n;
    // anything left (chanMap >= nBands or -3 inside) contributes nothing in the reference
    // either only if chanMap <= -2; a chanMap >= nBands cannot occur (m-2 <= nBands-1).
  }
  mb.usePower = cfg.usePower != 0;
  if (cfg.htkcompatible)                                       // :559-569
    mb.outScale = cfg.usePower ? (float)(32767.0 * 32767.0) : (float)32767.0;
  else
    mb.outScale = 1.f;
}

// cMfcc::initTables (lldcore/mfcc.cpp:136-170) + the output-order permutation and lifter
// product of processVector (:251-272).
void build_mfcc(const osm_b200_mfcc &cfg, int nBands, MfccOp &op)
{
  const int first = cfg.firstMfcc, last = cfg.lastMfcc;
  const int nM = last - first + 1;
  op.first = first; op.last = last; op.nMfcc = nM;
  float melfloor = (float)cfg.melfloor;                        // :71
  if (cfg.htkcompatible) melfloor = 1.0f;                      // :88-91
  op.melfloor = melfloor;
  op.logMelfloor = std::log(melfloor);                         // float overload, :240
  op.doLog = cfg.doLog != 0;
  const float cepLifter = (float)cfg.cepLifter;                // :75

  std::vector<float> cost((size_t)nBands * nM), sint(nM);
  const double fnM = (double)nBands;
  for (int i = first; i <= last; i++) {                        // :146-152
    const double fi = (double)i;
    for (int m = 0; m < nBands; m++)
      cost[m + (i - first) * nBands] = (float)cos((double)M_PI * (fi / fnM) * ((double)m + 0.5));
  }
  for (int i = first; i <= last; i++) {                        // :158-166
    if (cepLifter > 0.0)
      sint[i - first] = ((float)1.0 + cepLifter / (float)2.0 * std::sin((float)M_PI * ((float)i) / cepLifter));
    else
      sint[i - first] = 1.0f;
  }
  const float factor = (float)sqrt((double)2.0 / (double)nBands);  // :251
  op.cosT.assign((size_t)nBands * nM, 0.f);
  op.liftFactor.assign(nM, 0.f);
  for (int i = first; i <= last; i++) {                        // :252-258 output slot -> table row
    const int slot = i - first;
    int i0 = slot;
    if (cfg.htkcompatible && first == 0) i0 = (i == last) ? 0 : i0 + 1;
    memcpy(&op.cosT[(size_t)slot * nBands], &cost[(size_t)i0 * nBands], sizeof(float) * nBands);
    op.liftFactor[slot] = sint[i0] * factor;                   // :272
  }
}

// smileDsp_equalLoudnessWeight(_htk), smileutil/smileUtil.c:1041-1061
static double eql_htk(double f)
{
  const double f2 = f * f, fs = f2 / (f2 + 1.6e5);
  return fs * fs * ((f2 + 1.44e6) / (f2 + 9.61e6));
}
static double eql_hermansky(double f)
{
  const double w = 2.0 * M_PI * f, w2 = w * w, c = w2 + 6300000.0;
  if (c > 0.0) return (1e32 * ((w2 + 56.8e6) * w2 * w2) / (c * c * (w2 + 0.38e9) * (w2 * w2 * w2 * w + 1.7e31)));
  return 0.0;
}

// cPlp::myFetchConfig (lldcore/plp.cpp:88-171) + cPlp::initTables (:276-341).
// RASTA / newRASTA (a recurrence over frames) is not fused yet.
bool build_plp(const osm_b200_plp &cfg, const MelBank &mb, double levelPeriod, PlpOp &op, std::string &err)
{
  op.rasta = cfg.newRASTA ? 2 : (cfg.RASTA ? 1 : 0);                                      // :176 newRASTA disables RASTA
  if (op.rasta) {                                                                       // :361-397, T = reader level period
    const float upper = (float)cfg.rastaUpperCutoff, lower = (float)cfg.rastaLowerCutoff;   // :171-173 (FLOAT_DMEM)
    op.rastaIir = (float)(1.0 - sin(2.0 * M_PI * lower * levelPeriod));
    const float om = (float)cos(2.0 * M_PI * upper * levelPeriod);
    const float norm = (float)sqrt(10.0 * (32.0 * om * om + 8.0));
    op.rastaFir[0] = (float)(2.0 / norm);
    op.rastaFir[1] = (float)(-4.0 * om / norm);
    op.rastaFir[2] = 0.0;
    op.rastaFir[3] = -op.rastaFir[1];
    op.rastaFir[4] = -op.rastaFir[0];
  }
  int lpOrder = cfg.lpOrder;
  bool doLP = cfg.doLP != 0, doLpToCeps = cfg.doLpToCeps != 0, doIDFT = cfg.doIDFT != 0;
  if (lpOrder <= 0) { lpOrder = 0; doLP = false; doLpToCeps = false; }                 // :103-106
  int nCeps = cfg.nCeps, firstCC = cfg.firstCC, lastCC = cfg.lastCC;
  if (firstCC > lpOrder) { firstCC = lpOrder; nCeps = 1; lastCC = lpOrder; }           // :111-112
  else if (firstCC < 0) firstCC = 0;
  if (nCeps < 0) nCeps = lpOrder - firstCC + 1;                                         // :114-116
  if (lastCC < 0) lastCC = firstCC + nCeps - 1;                                         // :118-121
  else if (lastCC >= firstCC) nCeps = lastCC - firstCC + 1;
  if (lastCC > lpOrder) { lastCC = lpOrder; nCeps = lastCC - firstCC + 1; }             // :122-126
  if (nCeps == 0) doLpToCeps = false;                                                   // :132
  if (doLpToCeps) doLP = true;                                                          // :134-136
  if (doLP) doIDFT = true;                                                              // :137-139
  if (lpOrder > 8) { err = "cPlp: lpOrder > 8 is not supported"; return false; }
  op.lpOrder = lpOrder; op.nCeps = nCeps; op.firstCC = firstCC; op.lastCC = lastCC;
  op.doLP = doLP; op.doLpToCeps = doLpToCeps; op.doIDFT = doIDFT;
  float compression = (float)cfg.compression;                                           // :142-143
  if (compression < 0.0) compression = 0.0;
  op.compression = compression;
  float cepLifter = (float)(int)cfg.cepLifter;                                          // :146 getInt
  if (cepLifter < 0) cepLifter = 0;
  op.melfloor = (float)cfg.melfloor;
  op.doLog = cfg.doLog != 0; op.doAud = cfg.doAud != 0; op.doInvLog = cfg.doInvLog != 0;
  op.htk = cfg.htkcompatible != 0;
  if (op.htk) { op.melfloor = 1.0f; op.doAud = true; op.doLog = false; op.doInvLog = false; }   // :152-163
  if (op.rasta) { op.doLog = true; op.doInvLog = true; }                                     // :169-170 RASTA works in the log domain
  op.logMelfloor = std::log(op.melfloor);
  const int nBands = mb.nBands;
  op.nFreq = nBands + 2;                                                                // :288
  op.nAuto = lpOrder + 1;
  op.cosT.assign((size_t)op.nAuto * op.nFreq, 0.f);
  {
    const float a = (float)M_PI / (float)(op.nFreq - 1);                                // :298
    for (int i = 0; i < op.nAuto; i++) {
      const int ib = i * op.nFreq;
      int m;
      op.cosT[ib] = 1.0;
      for (m = 1; m < (op.nFreq - 1); m++) op.cosT[m + ib] = (float)(2.0 * cos(a * (double)i * (double)m));
      op.cosT[m + ib] = (float)(cos(a * (double)i * (double)m));
    }
  }
  op.lifter = cepLifter > 0.0;
  std::vector<float> sint(nCeps > 0 ? nCeps : 1, 1.f);
  for (int i = firstCC; i <= lastCC; i++) {                                             // :320-327
    if (cepLifter > 0.0)
      sint[i - firstCC] = ((float)1.0 + cepLifter / (float)2.0 * std::sin((float)M_PI * ((float)(i)) / cepLifter));
    else
      sint[i - firstCC] = 1.0;
  }
  op.lift.assign(nCeps > 0 ? nCeps : 1, 1.f);
  for (int i = firstCC; i <= lastCC; i++) {                                             // :560-573 output slot -> table index
    const int i0 = i - firstCC;
    int i1 = i0;
    if (op.htk && firstCC == 0) i1 = (i == lastCC) ? 0 : i1 + 1;
    op.lift[i0] = sint[i1];
  }
  op.eql.assign(nBands, 1.f);
  for (int i = 0; i < nBands; i++) {                                                    // :345-357 (band centres = melspec field info)
    op.eql[i] = op.htk ? (float)eql_htk(mb.bandHz[i]) : (float)eql_hermansky(mb.bandHz[i]);
    if (op.doLog) op.eql[i] = std::log(op.eql[i]);
  }
  op.nOut = doLpToCeps ? nCeps : (doLP ? lpOrder : (doIDFT ? op.nAuto : nBands));        // :232-267
  return true;
}

// Traunmueller bark (smileutil/smileUtil.c:1113-1128) and Zwicker's g(z) (:1064-1079)
static double bark_fwd(double x)
{
  if (x > 0) {
    const double zz = (26.81 / (1.0 + 1960.0 / x)) - 0.53;
    if (zz < 2) return (0.85 * zz + 0.3);
    if (zz > 20.1) return (1.22 * zz - 0.22 * 20.1);
    return zz;
  }
  return 0.0;
}
static double sharp_g(double z) { return z <= 16.0 ? 1.0 : pow((z - 16.0) / 4.0, 1.5849625) + 1.0; }

// cSpectral::myFetchConfig (lldcore/spectral.cpp:219-376) + the lazily computed, frame
// independent parts of processVector: spectral range (:625-647), band / slope edges
// (:781-825, :879-925), sharpness weights (:1443-1453).  Input = magnitude bins with the
// bin-frequency field info written by cTransformFFT (linear scale).
bool build_spectral(const osm_b200_spectral &cfg, int nSrc, double fftFrameSizeSec, SpectralOp &op, std::string &err)
{
  op = SpectralOp();
  op.nSrc = nSrc;
  op.F0 = (double)(1.0) / (double)fftFrameSizeSec;           // transformFft.cpp:111
  std::vector<double> frq(nSrc);
  for (int i = 0; i < nSrc; i++) frq[i] = op.F0 * (double)i;
  op.squareInput = cfg.squareInput != 0; op.useLog = cfg.useLogSpectrum != 0; op.normBand = cfg.normBandEnergies != 0;
  op.buggyRollOff = cfg.buggyRollOff != 0; op.oldSlopeScale = cfg.oldSlopeScale != 0;
  if (op.useLog) {                                            // :228-237
    float sf = (float)cfg.specFloor;
    sf = sf * sf;
    op.specFloor = sf;
    op.logSpecFloor = (float)(10.0 * log(sf) / log(10.0));
  }
  op.flux = cfg.flux != 0; op.centroid = cfg.centroid != 0; op.maxPos = cfg.maxPos != 0; op.minPos = cfg.minPos != 0;
  op.entropy = cfg.entropy != 0; op.stddev = cfg.standardDeviation != 0; op.variance = cfg.variance != 0;
  op.skewness = cfg.skewness != 0; op.kurtosis = cfg.kurtosis != 0; op.slope = cfg.slope != 0;
  op.alphaRatio = cfg.alphaRatio != 0; op.hammarberg = cfg.hammarbergIndex != 0; op.sharpness = cfg.sharpness != 0;
  op.harmonicity = cfg.harmonicity != 0; op.flatness = cfg.flatness != 0; op.logFlatness = false;
  auto lorp = [&]() { if (op.useLog) op.reqLog = true; else op.reqPow = true; };
  op.reqMag = op.flux;
  if (op.centroid) lorp(); if (op.maxPos) lorp(); if (op.minPos) lorp(); if (op.entropy) lorp();
  if (op.stddev) lorp(); if (op.variance) lorp(); if (op.skewness) lorp(); if (op.kurtosis) lorp(); if (op.slope) lorp();
  if (op.alphaRatio) op.reqPow = true; if (op.hammarberg) op.reqPow = true;
  if (cfg.nBands > 0) op.reqPow = true; if (cfg.nSlopes > 0) lorp(); if (cfg.nRollOff > 0) op.reqPow = true;
  if (op.sharpness) op.reqPow = true; if (op.harmonicity) lorp(); if (op.flatness) lorp();
  if (!op.reqPow && !op.reqLog && !op.reqMag) { err = "cSpectral: no descriptor is enabled"; return false; }
  if (op.useLog && !op.reqLog) op.reqLog = true;

  const long lo = (long)cfg.freqRangeLo, hi = (long)cfg.freqRangeHi;      // :625-647
  if (lo == hi && hi == 0) { op.loBin = 1; op.hiBin = nSrc - 1; }
  else {
    int lb = -1, hb = -1;
    for (int i = 0; i < nSrc; i++) {
      if ((double)lo >= frq[i]) lb = i;
      if ((double)hi > frq[i]) hb = i;
    }
    if (hb == -1 || hb >= nSrc) hb = nSrc - 1;
    if (lb < 0) lb = 0;
    op.loBin = lb; op.hiBin = hb;
  }
  auto edgeLo = [&](double f, double &idx, double &w) {       // :781-795
    int ii;
    for (ii = 0; ii < nSrc; ii++) if (frq[ii] > f) break;
    if ((ii < nSrc) && (ii > 0)) w = (frq[ii] - f) / (frq[ii] - frq[ii - 1]); else w = 1.0;
    idx = (double)ii - 1.0;
    if (idx < 0) idx = 0;
    if (idx >= nSrc) idx = nSrc;
  };
  auto edgeHi = [&](double f, double &idx, double &w) {       // :808-825
    int ii;
    for (ii = 0; ii < nSrc; ii++) if (frq[ii] >= (float)f) break;
    if ((ii < nSrc) && (ii > 0)) w = (f - frq[ii - 1]) / (frq[ii] - frq[ii - 1]); else w = 1.0;
    if ((ii < nSrc) && (frq[ii] == (float)f)) idx = (double)ii; else idx = (double)ii - 1.0;
    if (idx >= nSrc) idx = nSrc - 1;
  };
  auto resolve = [&](double fl, double fh, int &iL, int &iR, double &wL, double &wR, double &nind) {
    double idxL, idxR;
    edgeLo((double)(long)fl, idxL, wL); if (wL == 0.0) wL = 1.0;
    edgeHi((double)(long)fh, idxR, wR); if (wR == 0.0) wR = 1.0;
    long l = (long)floor(idxL), r = (long)floor(idxR);          // :833-839
    if (l >= nSrc) { l = r = nSrc - 1; wR = 0.0; wL = 0.0; }
    if (r >= nSrc) { r = nSrc - 1; wR = 1.0; }
    if (l < 0) l = 0; if (r < 0) r = 0;
    iL = (int)l; iR = (int)r; nind = idxR - idxL;
  };
  for (int i = 0; i < cfg.nBands && i < OSM_B200_MAX_LIST; i++) {
    if (!((long)cfg.bandLo[i] >= 0 && (long)cfg.bandHi[i] > 0)) continue;   // isBandValid, spectral.hpp:64-68
    int iL, iR; double wL, wR, nind;
    resolve(cfg.bandLo[i], cfg.bandHi[i], iL, iR, wL, wR, nind);
    op.bandIL.push_back(iL); op.bandIR.push_back(iR); op.bandWL.push_back(wL); op.bandWR.push_back(wR);
  }
  for (int i = 0; i < cfg.nSlopes && i < OSM_B200_MAX_LIST; i++) {
    if (!((long)cfg.slopeLo[i] >= 0 && (long)cfg.slopeHi[i] > 0)) continue;
    int iL, iR; double wL, wR, nind;
    resolve(cfg.slopeLo[i], cfg.slopeHi[i], iL, iR, wL, wR, nind);
    op.slopeIL.push_back(iL); op.slopeIR.push_back(iR); op.slopeWL.push_back(wL); op.slopeWR.push_back(wR);
    op.slopeNind.push_back(nind);
  }
  for (int i = 0; i < cfg.nRollOff && i < OSM_B200_MAX_LIST; i++) {
    double r = cfg.rollOff[i];
    if (r < 0.0) r = 0.0; else if (r > 1.0) r = 1.0;           // :340-347
    op.rollOff.push_back(r);
  }
  op.sharpW.assign(op.hiBin - op.loBin + 1, 0.0);
  for (int j = op.loBin; j <= op.hiBin; j++) {                 // :1443-1453 (linear axis -> bark)
    const double fb = bark_fwd(frq[j]);
    op.sharpW[j - op.loBin] = fb * sharp_g(fb);
  }
  op.nOut = (int)(op.bandIL.size() + op.slopeIL.size() + op.rollOff.size()) + op.alphaRatio + op.hammarberg + op.flux +
            op.centroid + op.maxPos + op.minPos + op.entropy + op.stddev + op.variance + op.skewness + op.kurtosis +
            op.slope + op.sharpness + op.harmonicity + op.flatness;
  if (op.hiBin - op.loBin < 4) { err = "cSpectral: spectral range too narrow"; return false; }
  return true;
}

// cEnergy::myFetchConfig (lldcore/energy.cpp:60-80)
void build_energy(const osm_b200_energy &cfg, EnergyOp &op)
{
  op.htk = cfg.htkcompatible != 0; op.rms = cfg.rms != 0; op.energy2 = cfg.energy2 != 0; op.lg = cfg.log != 0;
  if (op.htk) { op.lg = true; op.rms = false; }
  op.escaleLog = (float)cfg.escaleLog; op.escaleRms = (float)cfg.escaleRms; op.escaleSquare = (float)cfg.escaleSquare;
  op.ebiasLog = (float)cfg.ebiasLog; op.ebiasRms = (float)cfg.ebiasRms; op.ebiasSquare = (float)cfg.ebiasSquare;
  op.nOut = (int)op.rms + (int)op.energy2 + (int)op.lg;
}

void build_mzcr(const osm_b200_mzcr &cfg, MzcrOp &op)
{
  op.zcr = cfg.zcr != 0; op.mcr = cfg.mcr != 0; op.amax = cfg.amax != 0; op.maxmin = cfg.maxmin != 0; op.dc = cfg.dc != 0;
  op.nOut = (int)op.zcr + (int)op.mcr + (int)op.amax + 2 * (int)op.maxmin + (int)op.dc;
}

// cTonefilt::myFetchConfig (lld/tonefilt.cpp:65-98), configureWriter (:101-134) and the tables of setupNewNames (:180-189)
bool build_tonefilt(const osm_b200_tonefilt &cfg, double fs, TonefiltOp &op, std::string &err)
{
  double period = cfg.outputPeriod;
  if (period <= 0.0) period = 0.1;
  double dN = cfg.decayFN;
  if (dN < 0.0) dN = 0.0;
  if (dN > 1.0) dN = 1.0;
  double d0 = cfg.decayF0;
  if (d0 < dN) d0 = dN;
  if (d0 < 0.0) d0 = 0.0;
  if (d0 > 1.0) d0 = 1.0;
  double first = cfg.firstNote;
  if (first <= 0.0) first = 1.0;
  int n = cfg.nNotes;
  if (n < 1) n = 1;
  if (n > 128) { err = "cTonefilt.nNotes above 128 is not supported"; return false; }
  const double T = 1.0 / fs;                     // the wave level's period (iocore/waveSource.cpp)
  long P = (long)round(period / T);
  if (period < T) { period = T; P = 1; }
  if (P < 1 || P > (1L << 20)) { err = "cTonefilt.outputPeriod out of the supported range"; return false; }
  op.nNotes = n; op.P = (int)P; op.T = T; op.period = period;
  op.freq.resize(n); op.decay.resize(n);
  for (int k = 0; k < n; k++) op.freq[k] = first * pow(2.0, (double)k / 12.0);
  for (int k = 0; k < n; k++) op.decay[k] = dN + (d0 - dN) * (op.freq[k] - op.freq[0]) / (op.freq[n - 1]);   // the last frequency, not the span
  return true;
}

// cSpecScale::dataProcessorCustomFinalise (dsp/specScale.cpp:236-313), cPitchShs::setupNewNames
// (lld/pitchShs.cpp:160-215), cPitchBase / cPitchSmootherViterbi configuration.  The spline's abscissa
// terms (smileUtilSpline.c:124-140) are folded into recurrence coefficients, see PitchChainOp.
bool build_pitch_chain(const osm_b200_specscale &sc, const osm_b200_pitchshs &ps, const osm_b200_pitchsmootherviterbi *vcp,
                       int nMag, double fftFrameSizeSec, PitchChainOp &op, std::string &err)
{
  if (!(sc.scaleOctave && sc.sourceLin && sc.splineInterp)) { err = "cSpecScale: only scale=octave (log base 2), sourceScale=lin, interpMethod=spline are supported"; return false; }
  op.nMag = nMag;
  op.nPts = sc.nPointsTarget > 0 ? sc.nPointsTarget : nMag;
  if (nMag < 8 || op.nPts < 8 || op.nPts > 4096) { err = "cSpecScale: unsupported number of points"; return false; }
  op.enhance = sc.specEnhance != 0; op.smooth = sc.specSmooth != 0;
  const double fsSec = (double)(float)fftFrameSizeSec;              // specScale.cpp:184-187
  const double deltaF = 1.0 / fsSec;
  double minF = sc.minF < 1.0 ? 1.0 : sc.minF, maxF = sc.maxF;
  const double samplF = deltaF * (double)(nMag - 1);
  if (maxF <= minF || maxF > samplF) maxF = samplF;
  const double fmin_t = log(minF) / log(2.0), fmax_t = log(maxF) / log(2.0);
  const double deltaF_t = (fmax_t - fmin_t) / (double)(op.nPts - 1);
  std::vector<double> x(nMag);
  for (int i = 1; i < nMag; i++) x[i] = log((double)i * deltaF) / log(2.0);
  x[0] = 2.0 * x[1] - x[2];
  op.fwdA.assign(nMag, 0.0); op.fwdP6.assign(nMag, 0.0); op.r1.assign(nMag, 0.0); op.r2.assign(nMag, 0.0); op.bwdD.assign(nMag, 0.0);
  double dPrev = 0.0;                                               // y2[0] = 0 (natural boundary, y1p = 1e30)
  for (int i = 1; i < nMag - 1; i++) {
    const double sigma = (x[i] - x[i - 1]) / (x[i + 1] - x[i - 1]);
    const double diff1 = (x[i + 1] - x[i]) * (x[i + 1] - x[i - 1]);
    const double diff2 = (x[i] - x[i - 1]) * (x[i + 1] - x[i - 1]);
    const double p = 1.0 / (sigma * dPrev + 2.0);
    dPrev = (sigma - 1.0) * p;
    op.bwdD[i] = dPrev;
    op.fwdA[i] = -p * sigma;
    op.fwdP6[i] = 6.0 * p;
    op.r1[i] = 1.0 / diff1;
    op.r2[i] = 1.0 / diff2;
  }
  op.ik.resize(op.nPts); op.ia.resize(op.nPts); op.ic.resize(op.nPts); op.id.resize(op.nPts);
  long kupper = 1;
  for (int i = 0; i < op.nPts; i++) {                               // smileUtilSpline.c:301-352
    const double xi = fmin_t + (double)i * deltaF_t;
    if (i == 0 && xi < x[0]) { err = "cSpecScale: minF below the source axis"; return false; }
    while (kupper < nMag && x[kupper] < xi) kupper++;
    if (kupper == nMag) { err = "cSpecScale: target axis exceeds the source axis"; return false; }
    const long klower = kupper - 1;
    const double range = x[kupper] - x[klower];
    if (range == 0.0) { err = "cSpecScale: degenerate source axis"; return false; }
    const double a = (x[kupper] - xi) / range, b = 1.0 - a, range2 = range * range / 6.0;
    op.ik[i] = (int)klower; op.ia[i] = a; op.ic[i] = (a * a * a - a) * range2; op.id[i] = (b * b * b - b) * range2;
  }
  const double nOct = log(maxF / minF) / log(2.0);
  const double ppo = (double)op.nPts / nOct;
  op.audW.clear();
  if (sc.auditoryWeighting) {                                       // specScale.cpp:289-297
    const double atan_s = ppo * (log(65.0 / 50.0) / log(2.0)) - 1.0;
    op.audW.resize(op.nPts);
    for (int i = 0; i < op.nPts; i++) op.audW[i] = 0.5 + atan(3.0 * ((double)(i + 1) - atan_s) / ppo) / M_PI;
  }
  // level meta data is stored as float (specScale.cpp:299-311) and read back by cPitchShs (pitchShs.cpp:166-194)
  const float fMinF = (float)minF, fNOct = (float)nOct, fPpo = (float)ppo, fFminT = (float)fmin_t, fFmaxT = (float)fmax_t;
  if (fNOct == 0.0f) { err = "cSpecScale: zero octaves"; return false; }
  double base = exp(log((double)fMinF) / (double)fFminT);
  if (fabs(base - 2.0) < 0.00001) base = 2.0;
  op.logBase = log(base);
  op.Fmint = fFminT;
  op.Fstept = (fFmaxT - fFminT) / (float)(op.nPts - 1);
  // cPitchBase (lldcore/pitchBase.cpp:80-118)
  op.maxPitch = ps.maxPitch < 0.0 ? 0.0 : ps.maxPitch;
  op.minPitch = ps.minPitch < 0.0 ? 0.0 : ps.minPitch;
  if (op.minPitch > op.maxPitch) op.minPitch = op.maxPitch;
  op.nCand = ps.nCandidates < 1 ? 1 : (ps.nCandidates > 20 ? 20 : ps.nCandidates);
  if (op.nCand > 8) { err = "cPitchShs.nCandidates > 8 is not supported"; return false; }
  op.scores = ps.scores != 0; op.voicing = ps.voicing != 0; op.F0C1 = ps.F0C1 != 0; op.voicingC1 = ps.voicingC1 != 0;
  op.F0raw = ps.F0raw != 0; op.voicingClip = ps.voicingClip != 0;
  op.shsOnly = vcp == nullptr;
  if (!op.voicing && !op.shsOnly) { err = "cPitchShs.voicing=0 below cPitchSmootherViterbi is not supported"; return false; }
  op.voicingCutoff = (float)ps.voicingCutoff;
  op.octaveCorr = ps.octaveCorrection != 0; op.greedy = ps.greedyPeakAlgo != 0;
  op.nHarm = ps.nHarmonics;
  if (op.nHarm < 1 || op.nHarm > 32) { err = "cPitchShs.nHarmonics out of range"; return false; }
  op.shift.clear(); op.hscale.clear();
  const float comp = (float)ps.compressionFactor;
  float scale = comp;
  for (int i = 2; i < op.nHarm + 1; i++) {                          // pitchShs.cpp:246-254
    op.shift.push_back((int)(long)floor((double)fPpo * (log((double)i) / log(2.0))));
    op.hscale.push_back(scale);
    scale *= comp;
  }
  op.lfCutBin = -1;
  if (ps.lfCut > 0.0) op.lfCutBin = (int)((ceil(log(ps.lfCut) / log(base)) - op.Fmint) / op.Fstept);   // :230-236
  op.nShsCols = 1 + op.nCand * (1 + (int)op.voicing + (int)op.scores) + (int)op.F0C1 + (int)op.voicingC1 + (int)op.F0raw + (int)op.voicingClip;
  if (op.shsOnly) { op.nOut = op.nShsCols; return true; }
  // cPitchSmootherViterbi (lld/pitchSmootherViterbi.cpp:260-292; setWeights stores tvv in wTvvd, hpp:291-299)
  const osm_b200_pitchsmootherviterbi &vc = *vcp;
  op.bufLen = vc.bufferLength;
  if (op.bufLen < 2 || op.bufLen > 64) { err = "cPitchSmootherViterbi.bufferLength must be 2..64"; return false; }
  if (vc.F0raw || vc.voicingC1 || vc.voicingClip) { err = "cPitchSmootherViterbi: the copied fields F0raw / voicingC1 / voicingClip are not supported"; return false; }
  op.oF0final = vc.F0final != 0; op.oF0finalLog = vc.F0finalLog != 0; op.oF0finalEnv = vc.F0finalEnv != 0; op.oF0finalEnvLog = vc.F0finalEnvLog != 0;
  op.oVClipped = vc.voicingFinalClipped != 0; op.oVUnclipped = vc.voicingFinalUnclipped != 0;
  op.wLocal = vc.wLocal; op.wTvv = vc.wTvv; op.wTvvd = vc.wTvv; op.wTvuv = vc.wTvuv; op.wThr = vc.wThr; op.wRange = vc.wRange; op.wTuu = vc.wTuu;
  op.nOut = (int)op.oF0final + (int)op.oF0finalLog + (int)op.oF0finalEnv + (int)op.oF0finalEnvLog + (int)op.oVClipped + (int)op.oVUnclipped;
  if (op.nOut < 1) { err = "cPitchSmootherViterbi produces no output"; return false; }
  return true;
}

// ---------------------------------------------------------------------------------------
// cTransformFFT -> cSpecResample -> cLpc -> cFormantLpc.
//
// cSpecResample (dsp/specResample.cpp:97-185) reads the packed real FFT a[0..K) of the zero-padded windowed frame
// (K = FFT size; a[0] = R0, a[1] = R(K/2), a[2k] = Rk, a[2k+1] = Ik with X_k = sum_n x[n] exp(+2 pi i nk / K),
// dspcore/fftsg.c:104-122) and evaluates, for i = 0 .. I-1 (smileDsp_initIrdft / smileDsp_irdft,
// smileutil/smileUtil.c:1752-1820):
//   out[i] = ( a[0] + [I >= K] a[1] cos(2 pi (K/2) i / nd) + sum_{k=1}^{kMax/2-1} ( Rk cos(2 pi k i / nd) + Ik sin(2 pi k i / nd) ) ) / (K/2)
// with kMax = min(K, I) rounded down to even (antiAlias) and nd, I from the rounding rules of :150-172.
// Substituting the forward transform gives out[i] = sum_n x[n] D(n, i),
//   D(n, i) = ( 1 + [I >= K] (-1)^n cos(pi K i / nd) + sum_{k=1}^{kMax/2-1} cos(2 pi k (n / K - i / nd)) ) / (K/2),
// evaluated here in double for the samples n = pad .. pad+N-1 the frame occupies in the padded buffer
// (dspcore/transformFft.cpp:175-196).  The reference rounds to float after the FFT and again in the inverse sum; the
// table path rounds once per product -- same quantity, not the same bits (DESIGN.md, formant chain).
// ---------------------------------------------------------------------------------------
bool build_formant(const osm_b200_specresample &rs, const osm_b200_lpc &lp, const osm_b200_formantlpc &fl, const FrontEnd &fe,
                   bool zeroPadSymmetric, FormantOp &op, std::string &err)
{
  if (lp.method != 0) { err = "cLpc: only method=acf is supported"; return false; }
  if (!lp.saveLPCoeff || lp.saveRefCoeff || lp.residual || lp.lpSpectrum) { err = "cLpc: only saveLPCoeff=1 without saveRefCoeff / residual / lpSpectrum is supported"; return false; }
  if (lp.p < 1 || lp.p > 16) { err = "cLpc.p must be in 1..16"; return false; }
  if (fl.useLpSpec || fl.medianFilter || fl.octaveCorrection) { err = "cFormantLpc: useLpSpec / medianFilter / octaveCorrection are not supported"; return false; }
  if (fl.saveIntensity) { err = "cFormantLpc.saveIntensity is not supported"; return false; }
  const int K = fe.nfft, N = fe.frameSize;
  const double bT = 1.0 / fe.sampleRate, sr = 1.0 / bT;
  double ratio, targetFs;
  if (rs.resampleRatio > 0.0) { ratio = rs.resampleRatio; targetFs = ratio * sr; }     // specResample.cpp:72-88,107-115
  else {
    targetFs = rs.targetFs;
    if (targetFs <= 0.0) targetFs = 1.0;
    ratio = targetFs / sr;
  }
  op.T = 1.0 / targetFs;                                                                // :117 (before the adjustment below)
  const double fsSec = fe.fftFrameSizeSec, lastFsSec = fe.frameSizeSec;                 // level frameSizeSec / lastFrameSizeSec
  double nd, nOut0;
  if (fsSec != lastFsSec && lastFsSec != 0.0 && lastFsSec != bT) {                      // :150-160 zero-padded FFT input
    nOut0 = round((double)K * ratio * lastFsSec / fsSec);
    const double nr = nOut0 / ((double)K * (lastFsSec / fsSec));
    if (nr != ratio) ratio = nr;
    nd = (double)K * ratio;
  } else {                                                                              // :161-171
    nOut0 = round((double)K * ratio);
    const double nr = nOut0 / (double)K;
    if (nr != ratio) ratio = nr;
    nd = nOut0;
  }
  const int I = (int)nOut0;
  if (I < lp.p + 2 || I > 4096) { err = "cSpecResample: resampled frame size out of range"; return false; }
  int kMax = std::min(K, I);
  if (kMax & 1) kMax--;
  const int J = kMax / 2 - 1;                                                           // harmonics k = 1 .. J
  const int pad = zeroPadSymmetric ? (K - N) / 2 : 0;
  op.nIn = N; op.nRes = I; op.nResPad = (I + 31) / 32 * 32;
  const double twoPi = 2.0 * M_PI, scale = 1.0 / (double)(K / 2);
  const bool refOrder = K == 512 && I < K && !getenv("OSM_B200_FORMANT_COMPOSED");
  // formant_kernel keeps a batch of frames and their resampled copies in shared memory: refused here, while the graph is
  // compiled, so that a description-only plan refuses what a device plan would
  if (fm::formant_smem_bytes(refOrder, N, op.nResPad) > fm::kFmtSmemLimit) { err = "cSpecResample: frame too long for the formant kernel"; return false; }
  if (refOrder) {
    // Reference-order path: the spectrum is computed with the reference's own rounding sequence (fft_ref_order.cuh) and the
    // inverse sum runs over the reference's float tables in its order (smileDsp_initIrdft / smileDsp_irdft,
    // smileutil/smileUtil.c:1752-1820): cos / sin of (2 pi (k i)) / nd evaluated in double, stored as float.
    op.refOrder = true; op.kHalf = kMax / 2; op.padLeft = pad; op.halfK = (float)(K / 2);
    std::vector<float> wc;
    build_ref_fft_tables(wc);
    const size_t plane = (size_t)op.kHalf * op.nResPad;
    op.D.assign(wc.size() + 2 * plane, 0.0f);
    std::copy(wc.begin(), wc.end(), op.D.begin());
    float *ct = op.D.data() + wc.size(), *st = ct + plane;
    for (int i = 0; i < I; i++)
      for (long k2 = 1; k2 < op.kHalf; k2++) {
        const double kn = twoPi * (double)(k2 * (long)i) / nd;
        ct[(size_t)k2 * op.nResPad + i] = (float)cos(kn);
        st[(size_t)k2 * op.nResPad + i] = (float)sin(kn);
      }
  } else {
  op.D.assign((size_t)N * op.nResPad, 0.0f);
  for (int m = 0; m < N; m++) {
    const int n = pad + m;
    for (int i = 0; i < I; i++) {
      const double th = twoPi * ((double)n / (double)K - (double)i / nd);
      double acc = 1.0;
      if (I >= K) acc += ((n & 1) ? -1.0 : 1.0) * cos(twoPi * (double)(K / 2) * (double)i / nd);
      // sum_{k=1}^{J} cos(k th) by the Chebyshev recurrence c_{k+1} = 2 cos(th) c_k - c_{k-1}, restarted from libm
      // every 16 terms so the recurrence error stays at the rounding level of the direct sum
      for (int k0 = 1; k0 <= J; k0 += 16) {
        double cm = cos((double)(k0 - 1) * th), c0 = cos((double)k0 * th);
        const double t2 = 2.0 * cos(th);
        const int k1 = std::min(J, k0 + 15);
        for (int k = k0; k <= k1; k++) { acc += c0; const double cn = t2 * c0 - cm; cm = c0; c0 = cn; }
      }
      op.D[(size_t)m * op.nResPad + i] = (float)(acc * scale);
    }
  }
  }
  op.p = lp.p;
  int nF = fl.nFormants;                                                                // formantLpc.cpp:160-167
  if (nF > lp.p - 1) nF = lp.p - 1;
  if (nF <= 0) nF = lp.p - 1;
  if (nF < lp.p / 2) {
    // more roots in the upper half plane than slots: the reference keeps the first nFormants in the order its QR
    // iteration lists them, which no other solver reproduces
    err = "cFormantLpc: nFormants < p/2 (the result would depend on the reference's root order) is not supported"; return false;
  }
  op.nFormants = nF;
  op.minF = fl.minF; op.maxF = fl.maxF;
  op.saveFormants = fl.saveFormants != 0; op.saveBandwidths = fl.saveBandwidths != 0; op.saveNValid = fl.saveNumberOfValidFormants != 0;
  op.nOut = (op.saveNValid ? 1 : 0) + (op.saveFormants ? nF : 0) + (op.saveBandwidths ? nF : 0);
  if (op.nOut < 1) { err = "cFormantLpc produces no output"; return false; }
  return true;
}

// Twiddle tables of the reference's real FFT for n = 512 (fft_ref_order.cuh): w[nw = 128] followed by c[nc = 128], element for
// element what Ooura's initialisation produces (dspcore/fftsg.c: makewt :660-718, makect :741-757) with FLOAT_TYPE_FFT = float
// (src/include/dspcore/fftXg.h:16): the angle step is a FLOAT quotient, its multiples are FLOAT products that are widened to
// double for libm's cos / sin, and the results are rounded back to float.  The sub-tables of the coarser levels are copies of
// every other entry group; only their two interpolation constants are recomputed (float division).
void build_ref_fft_tables(std::vector<float> &wc)
{
  const int nw = 128, nc = 128;
  wc.assign(nw + nc, 0.0f);
  float *w = wc.data(), *c = w + nw;
  int nwh = nw >> 1;
  const float delta = (float)atan(1.0) / (float)nwh;
  const float wn4r = (float)cos((double)(delta * (float)nwh));
  w[0] = 1.0f; w[1] = wn4r;
  w[2] = (float)(0.5 / cos((double)(delta * 2.0f)));
  w[3] = (float)(0.5 / cos((double)(delta * 6.0f)));
  for (int j = 4; j < nwh; j += 4) {
    const float d1 = delta * (float)j, d3 = (3.0f * delta) * (float)j;
    w[j] = (float)cos((double)d1);
    w[j + 1] = (float)sin((double)d1);
    w[j + 2] = (float)cos((double)d3);
    w[j + 3] = (float)(-sin((double)d3));
  }
  int nw0 = 0;
  while (nwh > 2) {
    const int nw1 = nw0 + nwh;
    nwh >>= 1;
    w[nw1] = 1.0f; w[nw1 + 1] = wn4r;
    if (nwh == 4) { w[nw1 + 2] = w[nw0 + 4]; w[nw1 + 3] = w[nw0 + 5]; }
    else if (nwh > 4) {
      w[nw1 + 2] = 0.5f / w[nw0 + 4];
      w[nw1 + 3] = 0.5f / w[nw0 + 6];
      for (int j = 4; j < nwh; j += 4) for (int e = 0; e < 4; e++) w[nw1 + j + e] = w[nw0 + 2 * j + e];
    }
    nw0 = nw1;
  }
  const int nch = nc >> 1;
  const float dc = (float)atan(1.0) / (float)nch;
  c[0] = (float)cos((double)(dc * (float)nch));
  c[nch] = 0.5f * c[0];
  for (int j = 1; j < nch; j++) {
    c[j] = (float)(0.5 * cos((double)(dc * (float)j)));
    c[nc - j] = (float)(0.5 * sin((double)(dc * (float)j)));
  }
}

// ---- cTonespec (lld/tonespec.cpp).  The reference is C++: its unqualified pow / log / fabs / ceil / floor / round of a float
// argument resolve to the float overloads (powf, logf, ...); std:: with float arguments names the same functions here. ----

// computeDBA (dsp/dbA.cpp:110-126): curF accumulates F0 in float; bin 0 gets 10^(-inf) = 0.  The compiler folds the float
// pow(x, 2) into x * x (an exact rewrite: one rounding), which is not always what powf returns at a rounding tie.
static void tone_dba(std::vector<float> &x, int n, float F0)
{
  x.assign(n, 0.f);
  float curF = 0.0f;
  for (int i = 0; i < n; i++) {
    const float cf2 = curF * curF;
    float tmp = (float)(pow(12200.0, 2.0) * (cf2 * cf2)) / ((cf2 + (float)pow(20.6, 2.0)) * (cf2 + (float)pow(12200.0, 2.0)));
    tmp /= (float)(sqrt(cf2 + pow(107.7, 2.0)) * sqrt(cf2 + pow(737.9, 2.0)));
    x[i] = (float)pow(10.0, ((10.0 * std::log(tmp) + 2.0) / 10.0));
    curF += F0;
  }
}

bool build_tone_tables(const osm_b200_tonespec &cfg, int nBins, double frameSizeSec, ToneTables &t, std::string &err)
{
  const int nNotes = cfg.nOctaves * 12;                                                      // :93-95
  const float firstNote = (float)cfg.firstNote;
  // setPitchclassFreq (:147-167)
  t.pitchClassFreq.assign(nNotes + 2, 0.f);
  const float firstNote0 = firstNote / (float)pow(2.0, 1.0 / 12.0);
  t.pitchClassFreq[0] = firstNote0;
  double nn = 0.0;
  for (int i = 1; i < nNotes + 2; i++) {
    nn += 1.0;
    t.pitchClassFreq[i] = firstNote0 * (float)pow(2.0, nn / 12.0);
  }
  const float *pcf = t.pitchClassFreq.data();
  // computeFilters (:171-367), blocksize = nBins
  const float F0 = (float)(1.0 / frameSizeSec);                                             // :196
  std::vector<float> db;
  if (cfg.dbA) tone_dba(db, nBins, F0);
  int firstBin = (int)ceil((pcf[0] + pcf[1]) / (2.0 * F0));                                 // :203-207
  int lastBin = (int)floor((pcf[nNotes] + pcf[nNotes + 1]) / (2.0 * F0));
  if (firstBin < 1) firstBin = 1;
  if (lastBin >= nBins) lastBin = nBins - 1;
  t.binKey.assign(nBins, 0);                                                                // :210-227
  int curNote = 0;
  for (int i = 0; i < nBins; i++) {
    if (curNote > nNotes) curNote = nNotes;
    float distance0 = std::fabs(pcf[curNote] - ((float)i * F0));
    int note1 = curNote;
    float distance1 = std::fabs(pcf[++note1] - ((float)i * F0));
    while (distance0 > distance1) {
      if (note1 > nNotes) break;
      distance0 = distance1;
      distance1 = std::fabs(pcf[++note1] - ((float)i * F0));
    }
    curNote = note1 - 1;
    t.binKey[i] = curNote;
  }
  t.nbins.assign(nNotes + 2, 0);                                                            // :254-258
  for (int i = firstBin; i <= lastBin; i++)
    if (t.binKey[i] >= 0) t.nbins[t.binKey[i]]++;
  t.filterMap.assign(nBins, 0.f);                                                           // :268-332
  if (cfg.filterType != OSM_B200_TONE_REC) {
    for (int b = 1; b < nNotes - 1; b++) {
      const float start_freq = (pcf[b - 1] + pcf[b]) / 2.0f;
      const float end_freq = (pcf[b] + pcf[b + 1]) / 2.0f;
      const float start_bin = start_freq / F0, end_bin = end_freq / F0;
      const float middle_bin = pcf[b] / F0;
      int i_start_bin = (int)std::ceil(start_bin);
      int i_end_bin = (int)std::floor(end_bin);
      const int i_middle_bin = (int)std::round(pcf[b] / F0);
      if (i_start_bin > i_end_bin) continue;
      if (i_end_bin >= nBins) i_end_bin = nBins - 1;
      if (i_start_bin >= nBins) i_start_bin = nBins - 1;
      if (i_start_bin < 1) i_start_bin = 1;
      if (cfg.filterType == OSM_B200_TONE_TRI || cfg.filterType == OSM_B200_TONE_TRP) {
        if (i_middle_bin > nBins) {
          // :301-304 would write bins i_start_bin .. i_middle_bin - 1 past the end of the reference's map
          err = "cTonespec: a triangular filter of a note above the spectrum (the reference writes past its filter map); lower nOctaves";
          return false;
        }
        for (int i = i_start_bin; i < i_middle_bin; i++) {
          float &m = t.filterMap[i];
          m = (1.0f - ((middle_bin - (float)i) / (middle_bin - start_bin)));
          if (m > 1.0f) m = 2.0f - m;
        }
        for (int i = i_middle_bin; i <= i_end_bin; i++) {
          float &m = t.filterMap[i];
          m = (1.0f - (((float)i - middle_bin) / (end_bin - middle_bin)));
          if (m > 1.0f) m = 2.0f - m;
        }
      } else {                                                                              // :311-323
        for (int i = i_start_bin; i <= i_end_bin; i++) {
          const double dist_val = (double)(end_bin - start_bin);
          if (dist_val > 0.0) {
            const double x_val = (double)((double)i - middle_bin);
            const double delta = dist_val / 15.0;
            t.filterMap[i] = (float)((10.0 / 4.0) * (1.0 / sqrt(2.0 * M_PI)) * exp(-0.5 * (1.0 / delta) * (1.0 / delta) * pow(x_val, 2.0)));
          }
        }
      }
    }
  }
  if (cfg.filterType == OSM_B200_TONE_TRP)                                                 // :328-332
    for (int i = 0; i < nBins; i++) t.filterMap[i] *= t.filterMap[i];
  for (int i = 0; i < firstBin; i++) t.filterMap[i] = 0;                                   // :347-352
  for (int i = lastBin + 1; i < nBins; i++) t.filterMap[i] = 0;
  if (cfg.dbA)                                                                             // :354-359: db[] applied from bin firstBin on
    for (int i = firstBin; i <= lastBin; i++) t.filterMap[i] *= db[i - firstBin];
  t.firstBin = firstBin; t.lastBin = lastBin;
  return true;
}

// the per-frame sum (:418-434) as a one-tap band bank: note k (output k-1) sums the bins firstBin .. lastBin with binKey == k,
// which are contiguous because binKey never decreases with the bin index
bool build_tone(const osm_b200_tonespec &cfg, int nBins, double fftFrameSizeSec, ToneOp &op, std::string &err)
{
  if (cfg.nOctaves < 1 || cfg.nOctaves > 8) { err = "cTonespec.nOctaves must be in 1..8"; return false; }
  if (!(cfg.firstNote > 0.0)) { err = "cTonespec.firstNote must be > 0"; return false; }
  ToneTables t;
  if (!build_tone_tables(cfg, nBins, fftFrameSizeSec, t, err)) return false;
  const int nNotes = cfg.nOctaves * 12;
  op.nNotes = nNotes; op.nOut = nNotes;
  op.usePower = cfg.usePower != 0;
  MelBank &mb = op.bank;
  mb.nBands = nNotes; mb.nBins = nBins; mb.oneTap = true; mb.usePower = op.usePower; mb.outScale = 1.f;
  mb.coef = t.filterMap;
  mb.rangeBegin.assign(nNotes + 2, t.firstBin);
  int i = t.firstBin;
  for (int r = 0; r <= nNotes; r++) {
    mb.rangeBegin[r] = i;
    while (i <= t.lastBin && t.binKey[i] <= r) {
      if (t.binKey[i] < r) { err = "internal: cTonespec bin keys out of order"; return false; }
      i++;
    }
  }
  mb.rangeBegin[nNotes + 1] = i;
  mb.nLo = t.firstBin; mb.nHi = i;
  op.divisor.assign(nNotes, 0.f);
  for (int k = 0; k < nNotes; k++) op.divisor[k] = (float)t.nbins[k + 1];
  return true;
}

}  // namespace osm
