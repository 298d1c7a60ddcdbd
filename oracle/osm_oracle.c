/*
 * osm_oracle.c -- CPU restatement of openSMILE's LLD hot path (see osm_oracle.h).
 * TEST INFRASTRUCTURE ONLY: never linked into or imported by the product.
 * All `file:line` citations are relative to /root/reference/src.
 */
#include "osm_oracle.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>

#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif

/* ------------------------------------------------------------------ geometry */

/* core/winToVecProcessor.cpp:439-441: frameSizeFrames = (long)round(frameSize / T),
 * T = 1/sampleRate as a double (level period). C round() = half away from zero. */
long osm_or_frame_size_samples(const osm_or_frontend *fe)
{
  double T = 1.0 / fe->sample_rate;
  return (long)round(fe->frame_size_sec / T);
}

/* core/winToVecProcessor.cpp:443-456 */
long osm_or_frame_step_samples(const osm_or_frontend *fe)
{
  double T = 1.0 / fe->sample_rate;
  double step = fe->frame_step_sec;
  if (step == 0.0) step = fe->frame_size_sec;
  long s = (long)round(step / T);
  if (s == 0) s = osm_or_frame_size_samples(fe);
  return s;
}

/* dspcore/transformFft.cpp:124-129 (+ smileutil/smileUtil.c:691-731): next power of two
 * >= n, at least 4 */
long osm_or_fft_size(long n)
{
  long p = 1;
  while (p < n) p <<= 1;
  if (p < 4) p = 4;
  return p;
}

/* core/winToVecProcessor.cpp:868-877 with noPostEOIprocessing=1 + frameCenterSpecial=left:
 * only complete frames are emitted: T = floor((L - size)/step) + 1 for L >= size else 0 */
long osm_or_num_frames(long n_samples, long frame_size, long frame_step)
{
  if (n_samples < frame_size || frame_size <= 0 || frame_step <= 0) return 0;
  return (n_samples - frame_size) / frame_step + 1;
}

/* dspcore/transformFft.cpp:78-85: the level's frameSizeSec is multiplied by nfft/frameSize
 * (NOT replaced by nfft/fs) -- SURVEY.md H2 */
double osm_or_fft_frame_size_sec(const osm_or_frontend *fe)
{
  long n = osm_or_frame_size_samples(fe);
  long nfft = osm_or_fft_size(n);
  double fss = fe->frame_size_sec; /* winToVecProcessor.cpp:563-564: c.frameSizeSec = frameSize */
  if (nfft != n) fss *= (double)nfft / (double)n;
  return fss;
}

/* ------------------------------------------------------------------ a-1 PCM -> float */

/* smileutil/smileUtil.c:2520-2534 (monoMixdown=1, 16 bit): tmp = sum_c (float)x_c ;
 * out = (tmp / (float)nChan) / (float)32767.0 */
void osm_or_pcm16_to_float(const int16_t *pcm, long n_samples, int n_chan, float *out)
{
  for (long i = 0; i < n_samples; i++) {
    float tmp = 0.0f;
    for (int c = 0; c < n_chan; c++) tmp += (float)pcm[i * n_chan + c];
    out[i] = (tmp / (float)n_chan) / (float)32767.0;
  }
}

/* every sample format cWaveSource accepts, monoMixdown = 1 (smileutil/smileUtil.c:2518-2580 integer formats, :2651-2661 IEEE float).
 * format: 0 int16, 1 float32, 2 int8 (the reference reads 8-bit data as SIGNED bytes, :2507), 3 three bytes per sample (:2543-2552),
 * 4 32-bit container with 24 valid bits (masked, NOT sign extended, :2559), 5 int32.  Statement order of the reference: the channel
 * values are summed as floats from 0.0, divided by the channel count, then by the full scale (the float format has no full scale). */
void osm_or_pcm_to_float(const void *buf, int format, long n_samples, int n_chan, float *out)
{
  const int8_t *b8 = (const int8_t *)buf;
  const uint8_t *bu8 = (const uint8_t *)buf;
  const int16_t *b16 = (const int16_t *)buf;
  const int32_t *b32 = (const int32_t *)buf;
  const float *bf = (const float *)buf;
  for (long i = 0; i < n_samples; i++) {
    float tmp = 0.0f;
    for (int c = 0; c < n_chan; c++) {
      const long k = i * n_chan + c;
      switch (format) {
        case 0: tmp += (float)b16[k]; break;
        case 1: tmp += bf[k]; break;
        case 2: tmp += (float)b8[k]; break;
        case 3: {
          uint32_t is = 0;
          is |= (uint32_t)bu8[k * 3] << 8;
          is |= (uint32_t)bu8[k * 3 + 1] << 16;
          is |= (uint32_t)bu8[k * 3 + 2] << 24;
          tmp += (float)((int32_t)is >> 8);
          break;
        }
        case 4: tmp += (float)(b32[k] & 0xFFFFFF); break;
        default: tmp += (float)b32[k]; break;
      }
    }
    switch (format) {
      case 0: out[i] = (tmp / (float)n_chan) / (float)32767.0; break;
      case 1: out[i] = tmp / (float)n_chan; break;
      case 2: out[i] = (tmp / (float)n_chan) / (float)127.0; break;
      case 3: case 4: out[i] = (tmp / (float)n_chan) / (float)(32767.0 * 256.0); break;
      default: out[i] = (tmp / (float)n_chan) / (float)2147483647.0; break;
    }
  }
}

/* ------------------------------------------------------------------ a-4 window table */

/* smileutil/smileUtil.c:1218-1349, dspcore/windower.cpp:159-217 (gain only; no sqrt /
 * fade / xshift in the BASELINE configs) */
void osm_or_window_table(int win_func, long N, double sigma, double gain, double *w)
{
  double NN = (double)N;
  for (long n = 0; n < N; n++) {
    double i = (double)n;
    switch (win_func) {
      case OSM_OR_WIN_HANN:  /* :1277-1288 */
        w[n] = 0.5 * (1.0 - cos((2.0 * M_PI * i) / (NN - 1.0))); break;
      case OSM_OR_WIN_HAMM:  /* :1291-1303 */
        w[n] = 0.54 - 0.46 * cos((2.0 * M_PI * i) / (NN - 1.0)); break;
      case OSM_OR_WIN_GAUSS: { /* :1334-1349 */
        double s = sigma;
        if (s <= 0.0) s = 0.01;
        if (s > 0.5) s = 0.5;
        double tmp = (i - (NN - 1.0) / 2.0) / (s * (NN - 1.0) / 2.0);
        w[n] = exp(-0.5 * (tmp * tmp));
        break; }
      case OSM_OR_WIN_SINE:  /* :1306-1317 */
        w[n] = sin((1.0 * M_PI * i) / (NN - 1.0)); break;
      case OSM_OR_WIN_TRI:   /* :1232-1246 */
        if (n < N / 2) w[n] = 2.0 * (double)(n + 1) / (double)N;
        else w[n] = 2.0 * (double)(N - n) / (double)N;
        break;
      case OSM_OR_WIN_BARTLETT: /* :1261-1274 */
        if (n < N / 2) w[n] = 2.0 * (double)n / (double)(N - 1);
        else w[n] = 2.0 * (double)(N - 1 - n) / (double)(N - 1);
        break;
      default: w[n] = 1.0; break; /* rectangle :1218-1228 */
    }
  }
  if (gain != 1.0) for (long n = 0; n < N; n++) w[n] *= gain; /* windower.cpp:192-196 */
}

/* ------------------------------------------------------------------ a-5 FFT */

/* Real DFT with Ooura's output convention (dspcore/fftsg.c:104-122):
 *   a[2k] = R[k] = sum_j x[j] cos(2 pi j k / n),  a[2k+1] = I[k] = sum_j x[j] sin(2 pi j k / n)
 *   (0 < k < n/2),  a[0] = R[0],  a[1] = R[n/2].
 * Computed in double with an iterative radix-2 complex FFT, rounded to float at the end. */
static void fft_c2c_double(double *re, double *im, long n)
{
  /* bit reversal */
  for (long i = 1, j = 0; i < n; i++) {
    long bit = n >> 1;
    for (; j & bit; bit >>= 1) j ^= bit;
    j ^= bit;
    if (i < j) { double t = re[i]; re[i] = re[j]; re[j] = t; t = im[i]; im[i] = im[j]; im[j] = t; }
  }
  for (long len = 2; len <= n; len <<= 1) {
    double ang = 2.0 * M_PI / (double)len; /* e^{+i ang}: Ooura's forward sign */
    for (long i = 0; i < n; i += len) {
      for (long k = 0; k < len / 2; k++) {
        double wr = cos(ang * (double)k), wi = sin(ang * (double)k);
        double ur = re[i + k], ui = im[i + k];
        double vr = re[i + k + len / 2] * wr - im[i + k + len / 2] * wi;
        double vi = re[i + k + len / 2] * wi + im[i + k + len / 2] * wr;
        re[i + k] = ur + vr; im[i + k] = ui + vi;
        re[i + k + len / 2] = ur - vr; im[i + k + len / 2] = ui - vi;
      }
    }
  }
}

static void rdft_packed(const float *x, long n, float *a)
{
  double *re = (double *)malloc(sizeof(double) * n);
  double *im = (double *)calloc(n, sizeof(double));
  for (long i = 0; i < n; i++) re[i] = (double)x[i];
  fft_c2c_double(re, im, n);
  a[0] = (float)re[0];
  a[1] = (float)re[n / 2];
  for (long k = 1; k < n / 2; k++) { a[2 * k] = (float)re[k]; a[2 * k + 1] = (float)im[k]; }
  free(re); free(im);
}

/* one frame through a-3 .. a-6 */
void osm_or_frame_to_mag(const osm_or_frontend *fe, const float *x, long N, long nfft,
                         const double *win, float *fft_packed, float *mag)
{
  float *y = (float *)malloc(sizeof(float) * N);
  float *z = (float *)calloc(nfft, sizeof(float));
  float *a = fft_packed ? fft_packed : (float *)malloc(sizeof(float) * nfft);

  /* a-3 dspcore/vectorPreemphasis.cpp:89-108 (de=0): y[0]=(1-k)*x[0]; y[n]=x[n]-k*x[n-1] */
  if (fe->preemph_on) {
    float k = (float)fe->preemph_k; /* :55 k = (FLOAT_DMEM)getDouble("k") */
    y[0] = (1 - k) * x[0];
    for (long n = 1; n < N; n++) y[n] = x[n] - k * x[n - 1];
  } else {
    memcpy(y, x, sizeof(float) * N);
  }
  /* a-4 dspcore/windower.cpp:221-229: dst = src * (float)w + (float)offset */
  float off = (float)fe->win_offset;
  for (long n = 0; n < N; n++) y[n] = y[n] * (float)win[n] + off;

  /* a-5 dspcore/transformFft.cpp:175-196: zero padding (end, or symmetric) */
  long pad = fe->zero_pad_symmetric ? (nfft - N) / 2 : 0;
  for (long n = 0; n < N; n++) z[n + pad] = y[n];
  rdft_packed(z, nfft, a);

  /* a-6 dspcore/fftmagphase.cpp:215-221 */
  mag[0] = fabsf(a[0]);
  for (long n = 2; n < nfft; n += 2) mag[n / 2] = sqrtf(a[n] * a[n] + a[n + 1] * a[n + 1]);
  mag[nfft / 2] = fabsf(a[1]);

  if (!fft_packed) free(a);
  free(y); free(z);
}

/* ------------------------------------------------------------------ a-7 mel filterbank */

typedef struct {
  long n_bins, n_lo, n_hi;
  int n_bands;
  float *coef;      /* per bin rising-slope weight */
  long *chan_map;   /* per bin: lower band index, -1, or -3 */
  float *cfs;       /* nBands+2 centre frequencies in mel */
  double *band_hz;  /* nBands band centres in Hz (field info, used by cPlp) */
} mel_bank;

/* smileutil/smileUtil.c:1139-1142 (SPECTSCALE_MEL fwd) */
static double mel_fwd(double x) { return x > 0.0 ? 1127.0 * log(1.0 + x / 700.0) : 0.0; }
/* smileutil/smileUtil.c:1197-1198 (inverse) */
static double mel_inv(double x) { return 700.0 * (exp(x / 1127.0) - 1.0); }

/* smileDsp_specScaleTransfFwd (smileutil/smileUtil.c:1097-1147); scale numbering of osm_or_melspec.spec_scale */
static double scale_fwd(double x, int scale, double param)
{
  double zz, f6;
  switch (scale) {
    case 6: return x > 0 ? log(x) / log(param) : 0.0;
    case 4: return x / param > 1.0 ? 12.0 * (log(x / param) / log(2.0)) : 0.0;       /* smileMath_log2 */
    case 1:
      if (!(x > 0)) return 0.0;
      zz = (26.81 / (1.0 + 1960.0 / x)) - 0.53;
      if (zz < 2) return 0.85 * zz + 0.3;
      if (zz > 20.1) return 1.22 * zz - 0.22 * 20.1;
      return zz;
    case 3: if (!(x > 0)) return 0.0; f6 = x / 600.0; return 6.0 * log(f6 + sqrt(f6 * f6 + 1.0));
    case 2: return 13.1 * atan(.00074 * x) + 2.24 * atan(x * x * 1.85e-8) + 1e-4 * x;
    case 5: return x;
    default: return mel_fwd(x);
  }
}
/* smileDsp_specScaleTransfInv (:1158-1204); bark_speex has no inverse there and falls through to the mel inverse */
static double scale_inv(double x, int scale, double param)
{
  double zz, z0;
  switch (scale) {
    case 6: return exp(x * log(param));
    case 4: return param * pow(2.0, x / 12.0);
    case 1:
      zz = x;
      if (x > 20.1) zz = (x + 0.22 * 20.1) / 1.22;
      else if (x < 2) zz = (x - 0.3) / 0.85;
      z0 = 26.81 / (zz + 0.53);
      return z0 != 1.0 ? 1960.0 / (z0 - 1.0) : 0.0;
    case 3: return 600.0 * sinh(x / 6.0);
    case 5: return x;
    default: return mel_inv(x);
  }
}

/* lldcore/melspec.cpp:184-455, standard (non-ERB) triangular bank, specScale=mel.
 * float/double casts follow the reference line by line. */
static void mel_design(const osm_or_melspec *ms, long blocksize, double frame_size_sec, mel_bank *mb)
{
  int nBands = ms->n_bands;
  const int scale = ms->htkcompatible ? 0 : ms->spec_scale;   /* melspec.cpp:127-131 */
  double param = 0.0;                                          /* :133-135 */
  if (scale == 6) param = (ms->scale_param <= 0.0 || ms->scale_param == 1.0) ? 2.0 : ms->scale_param;
  else if (scale == 4) param = ms->scale_param;
  mb->n_bins = blocksize; mb->n_bands = nBands;
  mb->coef = (float *)calloc(blocksize, sizeof(float));
  mb->chan_map = (long *)malloc(sizeof(long) * blocksize);
  mb->cfs = (float *)malloc(sizeof(float) * (nBands + 2));
  mb->band_hz = (double *)malloc(sizeof(double) * nBands);

  float N = (float)((blocksize - 1) * 2);                 /* :217 */
  float F0 = (float)(1.0 / frame_size_sec);               /* :220 */
  float Fs = (float)(N / frame_size_sec);                 /* :221 */
  float M = (float)nBands;
  float lofreq = (float)ms->lofreq, hifreq = (float)ms->hifreq; /* melspec.hpp:48 FLOAT_DMEM */
  if ((lofreq < 0.0) || (lofreq > Fs / 2.0) || (lofreq > hifreq)) lofreq = 0.0;      /* :224-225 */
  if ((hifreq < lofreq) || (hifreq > Fs / 2.0) || (hifreq <= 0.0)) hifreq = Fs / (float)2.0; /* :226-227 */
  float LoF = (float)scale_fwd(lofreq, scale, param);                     /* :228-229 */
  float HiF = (float)scale_fwd(hifreq, scale, param);                     /* :230-231 */
  long nLoF = (long)round((double)(lofreq / F0));         /* :232 + melspec.hpp:107-110 */
  long nHiF = (long)round((double)(hifreq / F0));
  if (nLoF > blocksize) nLoF = blocksize;
  if (nHiF > blocksize) nHiF = blocksize;
  if (nLoF < 0) nLoF = 0;
  if (nHiF < 0) nHiF = 0;
  mb->n_lo = nLoF; mb->n_hi = nHiF;

  float mBandw = (HiF - LoF) / (M + (float)1.0);          /* :394 */
  for (int m = 0; m <= nBands + 1; m++) mb->cfs[m] = LoF + (float)m * mBandw; /* :395-397 */
  for (int m = 1; m <= nBands; m++) mb->band_hz[m - 1] = scale_inv(mb->cfs[m], scale, param); /* :408-411 */

  /* channel map :427-438 ; NtoFmel(n,F0) = (float)mel_fwd((float)n * F0) (melspec.hpp:119-122) */
  int m = 0;
  for (long n = 0; n < blocksize; n++) {
    if ((n <= nLoF) || (n >= nHiF)) mb->chan_map[n] = -3;
    else {
      while (mb->cfs[m] < (float)scale_fwd(((float)n) * F0, scale, param)) {
        if (m > nBands) break;
        m++;
      }
      mb->chan_map[n] = m - 2;
    }
  }
  /* rising slope weights :441-447 */
  m = 0;
  for (long n = nLoF; n < nHiF; n++) {
    float nM = (float)scale_fwd(((float)n) * F0, scale, param);
    while ((nM > mb->cfs[m + 1]) && (m <= nBands)) m++;
    mb->coef[n] = (mb->cfs[m + 1] - nM) / (mb->cfs[m + 1] - mb->cfs[m]);
  }
}

static void mel_free(mel_bank *mb) { free(mb->coef); free(mb->chan_map); free(mb->cfs); free(mb->band_hz); }

/* lldcore/melspec.cpp:519-570 */
static void mel_apply(const osm_or_melspec *ms, const mel_bank *mb, const float *mag, float *dst)
{
  long Nsrc = mb->n_bins;
  float *p = (float *)malloc(sizeof(float) * Nsrc);
  if (ms->use_power) for (long n = 0; n < Nsrc; n++) p[n] = mag[n] * mag[n]; /* :520-527 */
  else memcpy(p, mag, sizeof(float) * Nsrc);
  memset(dst, 0, sizeof(float) * mb->n_bands);
  for (long n = mb->n_lo; n < mb->n_hi; n++) {            /* :543-553 */
    long m = mb->chan_map[n];
    double a = (double)p[n] * (double)mb->coef[n];
    if (m > -2) {
      if (m > -1) dst[m] += (float)a;
      if (m < mb->n_bands - 1) dst[m + 1] += p[n] - (float)a;
    }
  }
  if (ms->htkcompatible) {                                /* :559-569 */
    for (int m = 0; m < mb->n_bands; m++) {
      if (ms->use_power) dst[m] *= (float)(32767.0 * 32767.0);
      else dst[m] *= (float)32767.0;
    }
  }
  free(p);
}

/* ------------------------------------------------------------------ a-8 MFCC */

/* lldcore/mfcc.cpp:136-170 (tables) + :238-273 (per frame) */
static void mfcc_apply(const osm_or_mfcc *mf, const float *mel, int nBands, float *dst)
{
  int first = mf->first_mfcc, last = mf->last_mfcc, nM = last - first + 1;
  float melfloor = (float)mf->melfloor;
  if (mf->htkcompatible) melfloor = 1.0f;                 /* :88-91 */
  float cepLifter = (float)mf->cep_lifter;
  float *cost = (float *)malloc(sizeof(float) * nBands * nM);
  float *sint = (float *)malloc(sizeof(float) * nM);
  double fnM = (double)nBands;
  for (int i = first; i <= last; i++) {                   /* :146-152 */
    double fi = (double)i;
    for (int m = 0; m < nBands; m++)
      cost[m + (i - first) * nBands] = (float)cos((double)M_PI * (fi / fnM) * ((double)m + 0.5));
  }
  for (int i = first; i <= last; i++) {                   /* :158-166 */
    if (cepLifter > 0.0)
      sint[i - first] = ((float)1.0 + cepLifter / (float)2.0 * sinf((float)M_PI * ((float)i) / cepLifter));
    else sint[i - first] = 1.0f;
  }
  float *l = (float *)malloc(sizeof(float) * nBands);
  for (int i = 0; i < nBands; i++) {                      /* :239-243 */
    if (mel[i] < melfloor) l[i] = logf(melfloor);
    else l[i] = logf(mel[i]);
  }
  float factor = (float)sqrt((double)2.0 / (double)nBands); /* :251 */
  for (int i = first; i <= last; i++) {                   /* :252-272 */
    int i0 = i - first;
    float *outc = dst + i0;
    if (mf->htkcompatible && (first == 0)) {
      if (i == last) i0 = 0; else i0 += 1;
    }
    *outc = 0.0f;
    for (int m = 0; m < nBands; m++) *outc += l[m] * cost[m + i0 * nBands];
    *outc *= sint[i0] * factor;
  }
  free(cost); free(sint); free(l);
}

/* ------------------------------------------------------------------ a-13 / a-14 */

static const float kZeroRow[256] = {0};

/* Tick-order model of chained window processors (cWindowProcessor, core/windowProcessor.cpp:
 * 85-119,167-230; blocksize=1 => one frame per tick; components tick in data-flow order,
 * core/componentManager.cpp:1233-1262).
 *
 * A level is described by (T = final number of frames, n0 = frames already written when EOI is
 * raised).  The static level has n0 = T.  A window processor with half window W reading it has,
 * before EOI, produced c0 = max(n0 - W, 0) frames (it needs t+W < n0); during EOI processing
 * producer and consumer both advance one frame per tick, producer first, so when the consumer
 * computes frame t >= c0 the producer holds  navail(t) = min(n0 + (t - c0) + 1, T)  frames.
 *
 * Reads of the input matrix for output frame t (core/dataMemoryLevel.cpp:1651-1738 getMatrix,
 * :1005-1045 validateIdxRangeR):
 *   window start t-W >= 0 : rows >= navail replicate row navail-1 (end padding, :1698-1708);
 *   window start t-W <  0 : rows < 0 replicate row 0 (:1687-1693), but rows >= navail are read
 *                           straight from the zero-initialised, not-yet-written level buffer
 *                           (:1694-1697 loops to the unclamped vIdxEnd) => 0.0.
 * For n0 >= W this reduces to the closed form "clamp to [0, T-1]" (SURVEY.md 8a-13); the other
 * branch is only reachable for utterances of fewer than W1+W2 frames and is reproduced because
 * the reference does it (verified against oracle/_ref for T = 1..5). */
static long win_navail(long t, long n0, long c0, long T)
{
  if (t < c0) return T;              /* computed before EOI: everything it needs is there */
  long n = n0 + (t - c0) + 1;
  return n < T ? n : T;
}

static const float *row_win(const float *x, long navail, int K, long t, int W, long i)
{
  if (t - W < 0) {
    if (i < 0) return x;
    if (i >= navail) return kZeroRow;
    return x + i * K;
  }
  if (i > navail - 1) i = navail - 1;
  return x + i * K;
}

/* dspcore/deltaRegression.cpp:139-146.  in: T x K with n0 frames written before EOI.
 * out: (T + W) x K; *c0_out = frames of the output level produced before EOI. */
static long delta_stage(const float *in, long T, long n0, int K, int W, float *out, long *c0_out)
{
  long c0 = n0 - W > 0 ? n0 - W : 0;
  if (c0_out) *c0_out = c0;
  if (T <= 0) return 0;
  float norm = 0.0f;
  for (int i = 1; i <= W; i++) norm += (float)i * (float)i; /* :77-79 */
  norm *= 2.0;
  long To = T + W;
  for (long t = 0; t < To; t++) {
    long na = win_navail(t, n0, c0, T);
    for (int k = 0; k < K; k++) {
      float num = 0.0f;
      for (int i = 1; i <= W; i++) {
        float delta = row_win(in, na, K, t, W, t + i)[k] - row_win(in, na, K, t, W, t - i)[k];
        num += (float)i * delta;
      }
      out[t * K + k] = num / norm;
    }
  }
  return To;
}

/* cDeltaRegression with relativeDelta / absOutput / halfWaveRect (dspcore/deltaRegression.cpp:100-108 computeDelta, :157-165 the
 * rectifications; halfWaveRect wins over absOutput), input level complete (n0 = T) */
long osm_or_delta_variant(const float *in, long T, int K, int W, int relative, int abs_output, int half_wave, float *out)
{
  if (T <= 0) return 0;
  float norm = 0.0f;
  for (int i = 1; i <= W; i++) norm += (float)i * (float)i;
  norm *= 2.0;
  long To = T + W, c0 = T - W > 0 ? T - W : 0;
  for (long t = 0; t < To; t++) {
    long na = win_navail(t, T, c0, T);
    for (int k = 0; k < K; k++) {
      float num = 0.0f;
      for (int i = 1; i <= W; i++) {
        float prior = row_win(in, na, K, t, W, t - i)[k], later = row_win(in, na, K, t, W, t + i)[k];
        float delta = later - prior;
        if (relative) delta = prior != 0.0 ? delta / fabsf(prior) : 0.0;
        num += (float)i * delta;
      }
      float y = num / norm;
      if (half_wave) { if (y < 0.0) y = 0.0; }
      else if (abs_output) { if (y < 0.0) y = -y; }
      out[t * K + k] = y;
    }
  }
  return To;
}

/* cDeltaRegression with onlyInSegments=1 (dspcore/deltaRegression.cpp:123-141, hpp:41-45): a pair
 * enters the sum only when neither value is 0 / NaN, and the member `norm` (initialised to
 * 2*sum i^2, :77-79) GROWS by i^2 for every accepted pair and is never reset (SURVEY.md H4), in
 * processing order: frame by frame (one frame per tick), element by element
 * (core/windowProcessor.cpp:190-212), i = 1..W. */
long osm_or_delta_segments(const float *in, long T, long n0, int K, int W, float *out)
{
  long c0 = n0 - W > 0 ? n0 - W : 0;
  if (T <= 0) return 0;
  float norm = 0.0f;
  for (int i = 1; i <= W; i++) norm += (float)i * (float)i;
  norm *= 2.0;
  long To = T + W;
  for (long t = 0; t < To; t++) {
    long na = win_navail(t, n0, c0, T);
    for (int k = 0; k < K; k++) {
      float num = 0.0f;
      for (int i = 1; i <= W; i++) {
        float a = row_win(in, na, K, t, W, t - i)[k], b = row_win(in, na, K, t, W, t + i)[k];
        if (!(b == 0.0f || b != b || a == 0.0f || a != a)) {
          num += (float)i * (b - a);
          norm += (float)i * (float)i;
        }
      }
      out[t * K + k] = norm != 0.0f ? num / norm : 0.0f;
    }
  }
  return To;
}

/* dspcore/contourSmoother.cpp:84-117: y = x[n]; y += x[n-w]; y += x[n+w] (w = 1..smaWin/2);
 * y /= smaWin  (noZeroSma: zeros are skipped and the divisor is the count) */
static long sma_stage(const float *in, long T, long n0, int K, int smaWin, int noZeroSma, float *out, long *c0_out)
{
  int W = smaWin / 2;
  long c0 = n0 - W > 0 ? n0 - W : 0;
  if (c0_out) *c0_out = c0;
  if (T <= 0) return 0;
  long To = T + W;
  for (long t = 0; t < To; t++) {
    long na = win_navail(t, n0, c0, T);
    for (int k = 0; k < K; k++) {
      float x0 = row_win(in, na, K, t, W, t)[k];
      if (noZeroSma) {
        if (x0 != 0.0f) {
          long N = 1;
          float y = x0;
          for (int w = 1; w <= W; w++) {
            float a = row_win(in, na, K, t, W, t - w)[k], b = row_win(in, na, K, t, W, t + w)[k];
            if (a != 0.0f) { y += a; N++; }
            if (b != 0.0f) { y += b; N++; }
          }
          out[t * K + k] = y / (float)N;
        } else out[t * K + k] = 0.0f;
      } else {
        float y = x0;
        for (int w = 1; w <= W; w++) {
          y += row_win(in, na, K, t, W, t - w)[k];
          y += row_win(in, na, K, t, W, t + w)[k];
        }
        out[t * K + k] = y / (float)smaWin;
      }
    }
  }
  return To;
}

/* public single-stage helpers: the input level is complete (n0 = T), as for a stage that
 * reads a static LLD level */
long osm_or_delta(const float *in, long T, int K, int W, float *out)
{
  return delta_stage(in, T, T, K, W, out, NULL);
}
long osm_or_sma(const float *in, long T, int K, int smaWin, int noZeroSma, float *out)
{
  return sma_stage(in, T, T, K, smaWin, noZeroSma, out, NULL);
}
/* chained stage: n0 = frames of `in` written before EOI (see the model above) */
long osm_or_delta_chained(const float *in, long T, long n0, int K, int W, float *out, long *c0_out)
{
  return delta_stage(in, T, n0, K, W, out, c0_out);
}
long osm_or_sma_chained(const float *in, long T, long n0, int K, int smaWin, int noZeroSma, float *out, long *c0_out)
{
  return sma_stage(in, T, n0, K, smaWin, noZeroSma, out, c0_out);
}

/* ------------------------------------------------------------------ whole chains */

/* static features for all frames of one utterance via a per-frame callback */
typedef void (*frame_fn)(void *ctx, const float *mag, long n_bins, float *dst);

static long run_frames(const osm_or_frontend *fe, const int16_t *pcm, long L, int n_chan,
                       frame_fn fn, void *ctx, int n_static, float *stat, float *tap_mag)
{
  long N = osm_or_frame_size_samples(fe), H = osm_or_frame_step_samples(fe);
  long nfft = osm_or_fft_size(N), nb = nfft / 2 + 1;
  long T = osm_or_num_frames(L, N, H);
  if (T <= 0) return 0;
  float *x = (float *)malloc(sizeof(float) * L);
  osm_or_pcm16_to_float(pcm, L, n_chan, x);
  double *win = (double *)malloc(sizeof(double) * N);
  osm_or_window_table(fe->win_func, N, fe->win_sigma, fe->win_gain, win);
  float *mag = (float *)malloc(sizeof(float) * nb);
  for (long t = 0; t < T; t++) {
    osm_or_frame_to_mag(fe, x + t * H, N, nfft, win, NULL, mag); /* a-2: frame t = [t*H, t*H+N) */
    if (tap_mag) memcpy(tap_mag + t * nb, mag, sizeof(float) * nb);
    fn(ctx, mag, nb, stat + t * n_static);
  }
  free(x); free(win); free(mag);
  return T;
}

/* static [T x K] -> [T x 3K] = static | delta | delta-delta, concat truncated to T
 * (other/vectorConcat.cpp:48-53 via core/dataReader.cpp:375-380: min over levels) */
static void add_deltas(const float *stat, long T, int K, int dW, int aW, float *out)
{
  float *d = (float *)malloc(sizeof(float) * (T + dW) * K);
  float *dd = (float *)malloc(sizeof(float) * (T + dW + aW) * K);
  long c0 = 0;
  long Td = delta_stage(stat, T, T, K, dW, d, &c0);
  delta_stage(d, Td, c0, K, aW, dd, NULL);
  for (long t = 0; t < T; t++) {
    memcpy(out + t * 3 * K, stat + t * K, sizeof(float) * K);
    memcpy(out + t * 3 * K + K, d + t * K, sizeof(float) * K);
    memcpy(out + t * 3 * K + 2 * K, dd + t * K, sizeof(float) * K);
  }
  free(d); free(dd);
}

typedef struct { const osm_or_melspec *ms; const osm_or_mfcc *mf; mel_bank mb; float *mel; float *tap_mel; long t; } mfcc_ctx;

static void mfcc_frame(void *vctx, const float *mag, long nb, float *dst)
{
  mfcc_ctx *c = (mfcc_ctx *)vctx;
  (void)nb;
  mel_apply(c->ms, &c->mb, mag, c->mel);
  if (c->tap_mel) memcpy(c->tap_mel + c->t * c->ms->n_bands, c->mel, sizeof(float) * c->ms->n_bands);
  mfcc_apply(c->mf, c->mel, c->ms->n_bands, dst);
  c->t++;
}

long osm_or_mfcc_d_a(const osm_or_frontend *fe, const osm_or_melspec *ms, const osm_or_mfcc *mf,
                     int dW, int aW, const int16_t *pcm, long L, int n_chan,
                     float *out, float *tap_mag, float *tap_mel)
{
  long N = osm_or_frame_size_samples(fe), H = osm_or_frame_step_samples(fe);
  long nfft = osm_or_fft_size(N);
  long T = osm_or_num_frames(L, N, H);
  if (T <= 0) return 0;
  int K = mf->last_mfcc - mf->first_mfcc + 1;
  mfcc_ctx c; c.ms = ms; c.mf = mf; c.tap_mel = tap_mel; c.t = 0;
  mel_design(ms, nfft / 2 + 1, osm_or_fft_frame_size_sec(fe), &c.mb);
  c.mel = (float *)malloc(sizeof(float) * ms->n_bands);
  float *stat = (float *)malloc(sizeof(float) * T * K);
  run_frames(fe, pcm, L, n_chan, mfcc_frame, &c, K, stat, tap_mag);
  add_deltas(stat, T, K, dW, aW, out);
  free(stat); free(c.mel); mel_free(&c.mb);
  return T;
}

/* ------------------------------------------------------------------ a-9 PLP */

/* smileutil/smileUtil.c:1053-1059 (HTK equal loudness) and :1041-1051 (Hermansky) */
static double eql_htk(double f) { double f2 = f * f; double fs = f2 / (f2 + 1.6e5); return fs * fs * ((f2 + 1.44e6) / (f2 + 9.61e6)); }
static double eql_herm(double f)
{
  double w = 2.0 * M_PI * f, w2 = w * w, c = w2 + 6300000.0;
  if (c > 0.0) return (1e32 * ((w2 + 56.8e6) * w2 * w2) / (c * c * (w2 + 0.38e9) * (w2 * w2 * w2 * w + 1.7e31)));
  return 0.0;
}

/* smileutil/smileUtil.c:1572-1627 (Durbin recursion, float) */
static int lpc_acf(const float *r, float *a, int p, float *gain)
{
  int i, m;
  float e, k_m;
  if (r[0] == 0.0f) { for (i = 0; i < p; i++) a[i] = 0.0f; return 0; }
  e = r[0];
  for (m = 1; m <= p; m++) {
    float sum = (float)1.0 * r[m];
    for (i = 1; i < m; i++) sum += a[i - 1] * r[m - i];
    k_m = ((float)-1.0 / e) * sum;
    a[m - 1] = k_m;
    for (i = 1; i <= m / 2; i++) {
      float x = a[i - 1];
      a[i - 1] += k_m * a[m - i - 1];
      if ((i < (m / 2)) || ((m & 1) == 1)) a[m - i - 1] += k_m * x;
    }
    e *= ((float)1.0 - k_m * k_m);
    if (e == 0.0f) { for (i = m; i < p; i++) a[i] = 0.0f; break; }
  }
  *gain = e;
  return 1;
}

/* smileutil/smileUtil.c:1532-1556 (HTK book eq. 5.11) */
static float lp_to_ceps(const float *lp, int nLp, float lpGain, float *ceps, int firstCC, int lastCC)
{
  if (firstCC < 1) firstCC = 1;
  if (lastCC > nLp) lastCC = nLp;
  for (int n = firstCC; n <= lastCC; n++) {
    double sum = 0;
    for (int i = 1; i < n; i++) sum += (n - i) * lp[i - 1] * ceps[n - i - 1];
    ceps[n - firstCC] = -(lp[n - firstCC] + (float)(sum / (double)n));
  }
  if (lpGain <= 0.0) lpGain = (float)1.0;
  return (float)(-log(1.0 / (double)lpGain));
}

typedef struct {
  const osm_or_melspec *ms; const osm_or_plp *pl; mel_bank mb; float *mel; float *tap_mel; long t;
  int nFreq, nAuto, nCeps, firstCC, lastCC;
  float *cost, *sint, *eql;
  float melfloor, compression, cepLifter;
  int doLog, doAud, doInvLog;
  /* RASTA (temporal) filter state, lldcore/plp.cpp:361-397,446-483 */
  double period;            /* reader_->getLevelT(): frame period of the band level */
  int rasta, newRasta, rInit, rPtr;
  float rFir[5], rIir, *rBufFir, *rBufIir;
} plp_ctx;

/* lldcore/plp.cpp:88-171 (config resolution) + :276-341 (tables) */
static void plp_init(plp_ctx *c, int nBands)
{
  const osm_or_plp *pl = c->pl;
  int lpOrder = pl->lp_order;
  c->firstCC = pl->first_cc; c->lastCC = pl->last_cc;
  int nCeps = -1;
  if (c->firstCC > lpOrder) { c->firstCC = lpOrder; nCeps = 1; c->lastCC = lpOrder; }
  else if (c->firstCC < 0) c->firstCC = 0;
  if (nCeps < 0) nCeps = lpOrder - c->firstCC + 1;            /* :116-118 */
  if (c->lastCC < 0) c->lastCC = c->firstCC + nCeps - 1;      /* :120 */
  else if (c->lastCC >= c->firstCC) nCeps = c->lastCC - c->firstCC + 1;
  if (c->lastCC > lpOrder) { c->lastCC = lpOrder; nCeps = c->lastCC - c->firstCC + 1; }
  c->nCeps = nCeps;
  c->compression = (float)pl->compression; if (c->compression < 0.0) c->compression = 0.0;   /* :141-142 */
  c->cepLifter = (float)(int)pl->cep_lifter; if (c->cepLifter < 0) c->cepLifter = 0;          /* :145 getInt */
  c->melfloor = (float)pl->melfloor;
  c->doLog = pl->do_log; c->doAud = pl->do_aud; c->doInvLog = pl->do_inv_log;
  if (pl->htkcompatible) { c->melfloor = 1.0f; c->doAud = 1; c->doLog = 0; c->doInvLog = 0; }   /* :152-163 */
  if (pl->rasta || pl->new_rasta) { c->doLog = 1; c->doInvLog = 1; }                            /* :169-170 */
  c->nFreq = nBands + 2; c->nAuto = lpOrder + 1;               /* :288-290 */
  c->cost = (float *)malloc(sizeof(float) * c->nAuto * c->nFreq);
  float a = (float)M_PI / (float)(c->nFreq - 1);               /* :298 */
  for (int i = 0; i < c->nAuto; i++) {
    int ib = i * c->nFreq, m;
    c->cost[ib] = 1.0;
    for (m = 1; m < (c->nFreq - 1); m++) c->cost[m + ib] = (float)(2.0 * cos(a * (double)i * (double)m));
    c->cost[m + ib] = (float)(cos(a * (double)i * (double)m));
  }
  c->sint = (float *)malloc(sizeof(float) * nCeps);
  for (int i = c->firstCC; i <= c->lastCC; i++) {              /* :320-327 */
    if (c->cepLifter > 0.0) c->sint[i - c->firstCC] = ((float)1.0 + c->cepLifter / (float)2.0 * sinf((float)M_PI * ((float)(i)) / c->cepLifter));
    else c->sint[i - c->firstCC] = 1.0;
  }
  c->rasta = pl->rasta; c->newRasta = pl->new_rasta;
  if (c->newRasta) c->rasta = 0;                               /* :176 */
  if (c->rasta || c->newRasta) {                               /* :361-397 */
    float upper = (float)pl->rasta_upper, lower = (float)pl->rasta_lower;   /* :171-173 (FLOAT_DMEM) */
    c->rIir = (float)(1.0 - sin(2.0 * M_PI * lower * c->period));
    float om = (float)cos(2.0 * M_PI * upper * c->period);
    float norm = (float)sqrt(10.0 * (32.0 * om * om + 8.0));
    c->rFir[0] = (float)(2.0 / norm);
    c->rFir[1] = (float)(-4.0 * om / norm);
    c->rFir[2] = 0.0;
    c->rFir[3] = -c->rFir[1];
    c->rFir[4] = -c->rFir[0];
    c->rBufIir = (float *)calloc(nBands, sizeof(float));
    c->rBufFir = (float *)calloc((size_t)nBands * 5, sizeof(float));
    c->rPtr = 0; c->rInit = 0;
  }
  c->eql = (float *)malloc(sizeof(float) * nBands);
  for (int i = 0; i < nBands; i++) {                           /* :345-357: band centres from the melspec field info */
    c->eql[i] = pl->htkcompatible ? (float)eql_htk(c->mb.band_hz[i]) : (float)eql_herm(c->mb.band_hz[i]);
    if (c->doLog) c->eql[i] = logf(c->eql[i]);
  }
}

/* lldcore/plp.cpp:416-593 */
static void plp_apply(plp_ctx *c, const float *src, int Nsrc, float *dst)
{
  const osm_or_plp *pl = c->pl;
  int lpOrder = pl->lp_order, nFreq = c->nFreq, nAuto = c->nAuto, i, m;
  float s[128], acf[32], lpc[32], ceps[32];
  for (i = 0; i < Nsrc; i++) {
    if (c->doLog) s[i] = (src[i] < c->melfloor) ? logf(c->melfloor) : logf(src[i]);   /* :434-440 */
    else s[i] = src[i];
  }
  if (c->rasta) {                                               /* :447-467 */
    for (i = 0; i < Nsrc; i++) {
      float sum;
      c->rBufFir[i * 5 + c->rPtr] = s[i];
      sum = c->rFir[0] * s[i];
      for (m = 1; m < 5; m++) sum += c->rFir[m] * c->rBufFir[i * 5 + ((5 - m + c->rPtr) % 5)];
      sum += c->rIir * c->rBufIir[i];
      c->rBufIir[i] = sum;
      if (c->rInit >= 5) s[i] = sum; else s[i] = 0;
    }
    if (c->rInit < 5) c->rInit++;
    c->rPtr = (c->rPtr + 1) % 5;
  }
  if (c->newRasta) {                                            /* :468-483 */
    float *b = c->rBufFir;
    for (i = 0; i < Nsrc; i++) {
      float out;
      out = c->rFir[0] * s[i] + b[i * 4 + 0];
      b[i * 4 + 0] = c->rFir[1] * s[i] + b[i * 4 + 1] + (c->rInit >= 5) * c->rIir * out;
      b[i * 4 + 1] = c->rFir[2] * s[i] + b[i * 4 + 2];
      b[i * 4 + 2] = c->rFir[3] * s[i] + b[i * 4 + 3];
      b[i * 4 + 3] = c->rFir[4] * s[i];
      if (c->rInit >= 5) s[i] = out; else s[i] = 0;
    }
    if (c->rInit < 5) c->rInit++;
  }
  if (c->doAud) {
    if (c->doLog) {
      for (i = 0; i < Nsrc; i++) s[i] += c->eql[i];
      for (i = 0; i < Nsrc; i++) s[i] *= c->compression;
    } else {
      for (i = 0; i < Nsrc; i++) { if (s[i] < c->melfloor) s[i] = c->melfloor; s[i] *= c->eql[i]; }   /* :501-504 */
      for (i = 0; i < Nsrc; i++) s[i] = (float)pow((double)s[i], (double)c->compression);              /* :506-508 */
    }
  }
  if (c->doInvLog) for (i = 0; i < Nsrc; i++) s[i] = expf(s[i]);
  if (!pl->do_idft) { memcpy(dst, s, sizeof(float) * Nsrc); return; }
  for (i = 0; i < nAuto; i++) {                                 /* :522-532 */
    double tmp = 0;
    if (pl->htkcompatible) tmp = (double)c->cost[i * nFreq] * (double)s[0];
    for (m = 1; m < nFreq - 1; m++) tmp += (double)c->cost[m + i * nFreq] * (double)s[m - 1];
    tmp += (double)c->cost[m + i * nFreq] * (double)s[nFreq - 3];
    acf[i] = (float)(tmp / (2.0 * (nFreq - 1)));
  }
  if (!pl->do_lp) { memcpy(dst, acf, sizeof(float) * nAuto); return; }
  float lpGain = 0.0f;
  lpc_acf(acf, lpc, lpOrder, &lpGain);                          /* :537 */
  if (!pl->do_lp_to_ceps) { memcpy(dst, lpc, sizeof(float) * lpOrder); return; }
  if (lpGain <= 0) lpGain = (float)1.0;                         /* :541-544 */
  float *cc = ceps;
  if (!pl->htkcompatible && (c->firstCC == 0)) cc++;
  float zeroth = lp_to_ceps(lpc, lpOrder, lpGain, cc, c->firstCC, c->lastCC);
  if (c->firstCC == 0) { if (!pl->htkcompatible) ceps[0] = zeroth; else ceps[c->nCeps - 1] = zeroth; }
  for (i = c->firstCC; i <= c->lastCC; i++) {                   /* :560-573 */
    int i0 = i - c->firstCC, i1 = i0;
    if (pl->htkcompatible && (c->firstCC == 0)) { if (i == c->lastCC) i1 = 0; else i1 += 1; }
    dst[i0] = (c->cepLifter > 0.0) ? ceps[i0] * c->sint[i1] : ceps[i0];
  }
}

static void plp_frame(void *vctx, const float *mag, long nb, float *dst)
{
  plp_ctx *c = (plp_ctx *)vctx;
  (void)nb;
  mel_apply(c->ms, &c->mb, mag, c->mel);
  if (c->tap_mel) memcpy(c->tap_mel + c->t * c->ms->n_bands, c->mel, sizeof(float) * c->ms->n_bands);
  plp_apply(c, c->mel, c->ms->n_bands, dst);
  c->t++;
}

/* number of output elements of the cPlp instance (lldcore/plp.cpp:232-267) */
int osm_or_plp_num_out(const osm_or_plp *pl, int n_bands)
{
  plp_ctx c; memset(&c, 0, sizeof c);
  if (pl->do_lp_to_ceps) {
    int lpOrder = pl->lp_order, first = pl->first_cc, last = pl->last_cc, nCeps = -1;
    if (first > lpOrder) { first = lpOrder; nCeps = 1; last = lpOrder; } else if (first < 0) first = 0;
    if (nCeps < 0) nCeps = lpOrder - first + 1;
    if (last < 0) last = first + nCeps - 1; else if (last >= first) nCeps = last - first + 1;
    if (last > lpOrder) { last = lpOrder; nCeps = last - first + 1; }
    return nCeps;
  }
  if (pl->do_lp) return pl->lp_order;
  if (pl->do_idft) return pl->lp_order + 1;
  return n_bands;
}

/* cPlp static level only (no temporal stages): out = [T][num_out] */
long osm_or_plp_static(const osm_or_frontend *fe, const osm_or_melspec *ms, const osm_or_plp *pl,
                       const int16_t *pcm, long L, int n_chan, float *out)
{
  long N = osm_or_frame_size_samples(fe), H = osm_or_frame_step_samples(fe);
  long nfft = osm_or_fft_size(N);
  long T = osm_or_num_frames(L, N, H);
  if (T <= 0) return 0;
  plp_ctx c; memset(&c, 0, sizeof c);
  c.ms = ms; c.pl = pl; c.t = 0;
  c.period = (fe->frame_step_sec != 0.0) ? fe->frame_step_sec : fe->frame_size_sec;   /* level period = cFramer.frameStep */
  mel_design(ms, nfft / 2 + 1, osm_or_fft_frame_size_sec(fe), &c.mb);
  plp_init(&c, ms->n_bands);
  int K = osm_or_plp_num_out(pl, ms->n_bands);
  c.mel = (float *)malloc(sizeof(float) * ms->n_bands);
  run_frames(fe, pcm, L, n_chan, plp_frame, &c, K, out, NULL);
  free(c.mel); free(c.cost); free(c.sint); free(c.eql); free(c.rBufFir); free(c.rBufIir); mel_free(&c.mb);
  return T;
}

/* cFullinputMean, default mode (dspcore/fullinputMean.cpp:526-546 accumulate, :506-522 subtract):
 * means = frame 0, += every further frame (float), /= (float)n, then x - mean for every frame */
void osm_or_cms(const float *x, long T, int K, float *out)
{
  if (T <= 0) return;
  float *m = (float *)malloc(sizeof(float) * K);
  for (int i = 0; i < K; i++) m[i] = x[i];
  for (long t = 1; t < T; t++) for (int i = 0; i < K; i++) m[i] += x[t * K + i];
  float nM = (float)T;
  for (int i = 0; i < K; i++) m[i] /= nM;
  for (long t = 0; t < T; t++) for (int i = 0; i < K; i++) { float v = x[t * K + i]; v -= m[i]; out[t * K + i] = v; }
  free(m);
}

/* cVectorOperation operation=ll1 (other/vectorOperation.cpp:475-481): float sum / N per row */
void osm_or_ll1(const float *x, long T, int K, float *out)
{
  for (long t = 0; t < T; t++) {
    float d = 0.0;
    for (int i = 0; i < K; i++) d += x[t * K + i];
    if (K > 0) d /= (float)K;
    out[t] = d;
  }
}

long osm_or_plp_d_a(const osm_or_frontend *fe, const osm_or_melspec *ms, const osm_or_plp *pl,
                    int dW, int aW, const int16_t *pcm, long L, int n_chan,
                    float *out, float *tap_mel)
{
  long N = osm_or_frame_size_samples(fe), H = osm_or_frame_step_samples(fe);
  long nfft = osm_or_fft_size(N);
  long T = osm_or_num_frames(L, N, H);
  if (T <= 0) return 0;
  plp_ctx c; memset(&c, 0, sizeof c);
  c.ms = ms; c.pl = pl; c.tap_mel = tap_mel; c.t = 0;
  c.period = (fe->frame_step_sec != 0.0) ? fe->frame_step_sec : fe->frame_size_sec;   /* level period = cFramer.frameStep */
  mel_design(ms, nfft / 2 + 1, osm_or_fft_frame_size_sec(fe), &c.mb);
  plp_init(&c, ms->n_bands);
  int K = osm_or_plp_num_out(pl, ms->n_bands);
  c.mel = (float *)malloc(sizeof(float) * ms->n_bands);
  float *stat = (float *)malloc(sizeof(float) * T * K);
  run_frames(fe, pcm, L, n_chan, plp_frame, &c, K, stat, NULL);
  add_deltas(stat, T, K, dW, aW, out);
  free(stat); free(c.mel); free(c.cost); free(c.sint); free(c.eql); free(c.rBufFir); free(c.rBufIir); mel_free(&c.mb);
  return T;
}


/* ------------------------------------------------------------------ a-12 cEnergy / cMZcr */

int osm_or_energy_num_out(const osm_or_energy_cfg *en)
{
  int rms = en->rms, lg = en->log;
  if (en->htkcompatible) { lg = 1; rms = 0; }                /* lldcore/energy.cpp:67 */
  return (rms ? 1 : 0) + (en->energy2 ? 1 : 0) + (lg ? 1 : 0);
}

/* lldcore/energy.cpp:152-187 */
static void energy_frame(const osm_or_energy_cfg *en, const float *src, long N, float *dst)
{
  int rms = en->rms, lg = en->log, n = 0;
  if (en->htkcompatible) { lg = 1; rms = 0; }
  double d = 0.0;
  for (long i = 0; i < N; i++) { float tmp = src[i]; d += tmp * tmp; }   /* float product, double sum */
  if (rms) dst[n++] = (float)sqrt(d / (float)N) * (float)en->escaleRms + (float)en->ebiasRms;
  if (en->energy2) dst[n++] = (float)(d / (double)N) * (float)en->escaleSquare + (float)en->ebiasSquare;
  if (lg) {
    const double minE = 8.674676e-019;                        /* :19 */
    if (!en->htkcompatible) {
      d /= (float)N;
      if (d < minE) d = minE;
      dst[n++] = (float)log(d) * (float)en->escaleLog + (float)en->ebiasLog;
    } else {
      d *= 32767.0 * 32767.0;
      if (d <= 1.0) d = 1.0;
      dst[n++] = (float)log(d) * (float)en->escaleLog + (float)en->ebiasLog;
    }
  }
}

int osm_or_mzcr_num_out(const osm_or_mzcr_cfg *mz)
{
  return (mz->zcr ? 1 : 0) + (mz->mcr ? 1 : 0) + (mz->amax ? 1 : 0) + (mz->maxmin ? 2 : 0) + (mz->dc ? 1 : 0);
}

/* lldcore/mzcr.cpp:109-157 (note the loop bounds 1..N-2 and nmc starting at 4.0) */
static void mzcr_frame(const osm_or_mzcr_cfg *mz, const float *src, long N, float *dst)
{
  float mean = src[0], nzc = 0.0f, nmc = 4.0f, max = 0, min = 0, absmax = 0;
  long i;
  if (mz->zcr || mz->mcr || mz->dc) {
    for (i = 1; i < N - 1; i++) {
      mean += src[i];
      if (((src[i - 1] * src[i + 1] <= 0.0) && (src[i] == 0.0)) || (src[i - 1] * src[i] < 0.0)) nzc += 1.0;
    }
    nzc /= (float)N;
    mean /= (float)N;
  }
  if (mz->mcr) {
    for (i = 1; i < N - 1; i++) {
      if ((((src[i - 1] - mean) * (src[i + 1] - mean) <= 0.0) && ((src[i] - mean) == 0.0)) || ((src[i - 1] - mean) * (src[i] - mean) < 0.0)) nmc++;
    }
    nmc /= (float)N;
  }
  if (mz->amax || mz->maxmin) {
    max = min = src[0];
    for (i = 1; i < N; i++) { if (src[i] < min) min = src[i]; if (src[i] > max) max = src[i]; }
    if (fabs(min) > fabs(max)) absmax = fabsf(min); else absmax = fabsf(max);
  }
  int n = 0;
  if (mz->zcr) dst[n++] = nzc;
  if (mz->mcr) dst[n++] = nmc;
  if (mz->amax) dst[n++] = absmax;
  if (mz->maxmin) { dst[n++] = max; dst[n++] = min; }
  if (mz->dc) dst[n++] = mean;
}

/* time-domain frames: framer output, optionally through pre-emphasis + window */
typedef void (*tframe_fn)(const void *cfg, const float *x, long N, float *dst);
static long run_time_frames(const osm_or_frontend *fe, int windowed, const int16_t *pcm, long L, int n_chan,
                            tframe_fn fn, const void *cfg, int K, float *out)
{
  long N = osm_or_frame_size_samples(fe), H = osm_or_frame_step_samples(fe);
  long T = osm_or_num_frames(L, N, H);
  if (T <= 0) return 0;
  float *x = (float *)malloc(sizeof(float) * L);
  osm_or_pcm16_to_float(pcm, L, n_chan, x);
  double *win = (double *)malloc(sizeof(double) * N);
  osm_or_window_table(fe->win_func, N, fe->win_sigma, fe->win_gain, win);
  float *y = (float *)malloc(sizeof(float) * N);
  for (long t = 0; t < T; t++) {
    const float *fx = x + t * H;
    if (windowed) {
      if (fe->preemph_on) {
        float k = (float)fe->preemph_k;
        y[0] = (1 - k) * fx[0];
        for (long n = 1; n < N; n++) y[n] = fx[n] - k * fx[n - 1];
      } else memcpy(y, fx, sizeof(float) * N);
      float off = (float)fe->win_offset;
      for (long n = 0; n < N; n++) y[n] = y[n] * (float)win[n] + off;
      fn(cfg, y, N, out + t * K);
    } else {
      fn(cfg, fx, N, out + t * K);
    }
  }
  free(x); free(win); free(y);
  return T;
}

/* cIntensity (lldcore/intensity.cpp:86-146).  NOTE the loop bound MIN(Nsrc, MIN(nWin, Ndst)): Ndst is the
 * number of OUTPUT values of the field (1 or 2), so only the first one or two samples enter the sum --
 * restated as the reference computes it. */
int osm_or_intensity_num_out(const osm_or_intensity_cfg *in) { return (in->intensity ? 1 : 0) + (in->loudness ? 1 : 0); }
static void intensity_tf(const void *c, const float *src, long Nsrc, float *dst)
{
  const osm_or_intensity_cfg *in = (const osm_or_intensity_cfg *)c;
  long Ndst = osm_or_intensity_num_out(in), nWin = Nsrc;
  double winSum = 0.0, NN = (double)Nsrc;
  double *hamWin = (double *)malloc(sizeof(double) * Nsrc);               /* smileDsp_winHam, smileUtil.c:1291-1303 */
  for (long j = 0; j < Nsrc; j++) { hamWin[j] = 0.54 - 0.46 * cos((2.0 * M_PI * (double)j) / (NN - 1.0)); winSum += hamWin[j]; }
  if (winSum <= 0.0) winSum = 1.0;
  double Im = 0.0, I0 = (double)0.000001;
  long safeN = Nsrc < (nWin < Ndst ? nWin : Ndst) ? Nsrc : (nWin < Ndst ? nWin : Ndst);
  for (long i = 0; i < safeN; i++) Im += hamWin[i] * (double)src[i] * (double)src[i];
  Im /= winSum;
  long n = 0;
  if (in->intensity) dst[n++] = (float)Im;
  if (in->loudness) dst[n++] = (float)pow(Im / I0, 0.3);
  free(hamWin);
}
long osm_or_intensity(const osm_or_frontend *fe, const osm_or_intensity_cfg *in, int windowed,
                      const int16_t *pcm, long L, int n_chan, float *out)
{
  return run_time_frames(fe, windowed, pcm, L, n_chan, intensity_tf, in, osm_or_intensity_num_out(in), out);
}

static void energy_tf(const void *c, const float *x, long N, float *d) { energy_frame((const osm_or_energy_cfg *)c, x, N, d); }
static void mzcr_tf(const void *c, const float *x, long N, float *d) { mzcr_frame((const osm_or_mzcr_cfg *)c, x, N, d); }

long osm_or_energy(const osm_or_frontend *fe, const osm_or_energy_cfg *en, int windowed,
                   const int16_t *pcm, long L, int n_chan, float *out)
{
  return run_time_frames(fe, windowed, pcm, L, n_chan, energy_tf, en, osm_or_energy_num_out(en), out);
}
long osm_or_mzcr(const osm_or_frontend *fe, const osm_or_mzcr_cfg *mz, int windowed,
                 const int16_t *pcm, long L, int n_chan, float *out)
{
  return run_time_frames(fe, windowed, pcm, L, n_chan, mzcr_tf, mz, osm_or_mzcr_num_out(mz), out);
}

/* ------------------------------------------------------------------ a-11 cSpectral */

int osm_or_spectral_num_out(const osm_or_spectral_cfg *sp)
{
  int n = 0;
  for (int i = 0; i < sp->nBands; i++) if (sp->bandLo[i] >= 0 && sp->bandHi[i] > 0) n++;
  for (int i = 0; i < sp->nSlopes; i++) if (sp->slopeLo[i] >= 0 && sp->slopeHi[i] > 0) n++;
  n += (sp->alphaRatio ? 1 : 0) + (sp->hammarbergIndex ? 1 : 0) + sp->nRollOff + (sp->flux ? 1 : 0);
  n += (sp->centroid ? 1 : 0) + (sp->maxPos ? 1 : 0) + (sp->minPos ? 1 : 0) + (sp->entropy ? 1 : 0);
  n += (sp->standardDeviation ? 1 : 0) + (sp->variance ? 1 : 0) + (sp->skewness ? 1 : 0) + (sp->kurtosis ? 1 : 0);
  n += (sp->slope ? 1 : 0) + (sp->sharpness ? 1 : 0) + (sp->harmonicity ? 1 : 0) + (sp->flatness ? 1 : 0);
  return n;
}

/* Traunmueller bark, smileutil/smileUtil.c:1113-1128 */
static double bark_fwd(double x)
{
  if (x > 0) {
    double zz = (26.81 / (1.0 + 1960.0 / x)) - 0.53;
    if (zz < 2) return (0.85 * zz + 0.3);
    else if (zz > 20.1) return (1.22 * zz - 0.22 * 20.1);
    else return zz;
  }
  return 0.0;
}
/* smileutil/smileUtil.c:1064-1079 with frqScale == BARK */
static double sharp_g(double z) { return z <= 16.0 ? 1.0 : pow((z - 16.0) / 4.0, 1.5849625) + 1.0; }

/* smileutil/smileUtil.c:2082-2124 */
static float stat_entropy(const float *vals, long N)
{
  const double entropy_floor = 0.0000001;
  double e = 0.0, dn = 0.0, l2 = log(2.0);
  float min = 0.0f;
  long i;
  for (i = 0; i < N; i++) { dn += (double)vals[i]; if (vals[i] < min) min = vals[i]; }
  if (min < 0.0) {
    double mf = entropy_floor + min;
    for (i = 0; i < N; i++) { if (vals[i] <= mf) dn += mf - vals[i]; dn -= (double)min; }
  } else min = 0.0f;
  if (dn < (float)entropy_floor) dn = (float)entropy_floor;
  for (i = 0; i < N; i++) {
    double v = vals[i] - min, ln;
    if (v <= entropy_floor) v = entropy_floor;
    ln = v / dn;
    if (ln > 0.0) e += ln * log(ln) / l2;
  }
  return (float)(-e);
}

typedef struct {
  const osm_or_spectral_cfg *sp;
  double fsSec;            /* frameSizeSec of the fftmag level (transformFft.cpp:78-85) */
  double *frq;             /* bin frequencies, field info (transformFft.cpp:102-117) */
  long Nsrc;
  float *prev; int havePrev;
  double *sharpW;
  long loBin, hiBin;
} spec_ctx;

/* band edge -> (bin index, weight) with the frequency axis from the field info
 * (lldcore/spectral.cpp:781-795 lower, :808-825 upper) */
static void edge_lo(const spec_ctx *c, double f, double *idx, double *w)
{
  long ii, nScale = c->Nsrc;
  for (ii = 0; ii < nScale; ii++) if (c->frq[ii] > f) break;
  if ((ii < nScale) && (ii > 0)) *w = (c->frq[ii] - f) / (c->frq[ii] - c->frq[ii - 1]); else *w = 1.0;
  *idx = (double)ii - 1.0;
  if (*idx < 0) *idx = 0;
  if (*idx >= c->Nsrc) *idx = c->Nsrc;
}
static void edge_hi(const spec_ctx *c, double f, double *idx, double *w)
{
  long ii, nScale = c->Nsrc;
  for (ii = 0; ii < nScale; ii++) if (c->frq[ii] >= (float)f) break;
  if ((ii < nScale) && (ii > 0)) *w = (f - c->frq[ii - 1]) / (c->frq[ii] - c->frq[ii - 1]); else *w = 1.0;
  if ((ii < nScale) && (c->frq[ii] == (float)f)) *idx = (double)ii; else *idx = (double)ii - 1.0;
  if (*idx >= c->Nsrc) *idx = c->Nsrc - 1;
}

/* lldcore/spectral.cpp:586-1555 for magnitude input with bin-frequency info, linear scale */
static void spectral_frame(spec_ctx *c, const float *src, float *dst)
{
  const osm_or_spectral_cfg *sp = c->sp;
  long Nsrc = c->Nsrc, i, j, n = 0;
  const double *frq = c->frq;
  int useLog = sp->useLogSpectrum;
  /* requirements, :219-376 */
  int reqMag = sp->flux, reqPow = 0, reqLog = 0;
#define LORP() do { if (useLog) reqLog = 1; else reqPow = 1; } while (0)
  if (sp->centroid) LORP(); if (sp->maxPos) LORP(); if (sp->minPos) LORP(); if (sp->entropy) LORP();
  if (sp->standardDeviation) LORP(); if (sp->variance) LORP(); if (sp->skewness) LORP(); if (sp->kurtosis) LORP();
  if (sp->slope) LORP();
  if (sp->alphaRatio) reqPow = 1; if (sp->hammarbergIndex) reqPow = 1;
  if (sp->nBands > 0) reqPow = 1; if (sp->nSlopes > 0) LORP(); if (sp->nRollOff > 0) reqPow = 1;
  if (sp->sharpness) reqPow = 1; if (sp->harmonicity) LORP(); if (sp->flatness) LORP();
  float specFloor = 0, logSpecFloor = 0;
  if (useLog) {                                                /* :228-237 */
    specFloor = (float)sp->specFloor;
    specFloor = specFloor * specFloor;
    logSpecFloor = (float)(10.0 * log(specFloor) / log(10.0));
  }
  long loBin = c->loBin, hiBin = c->hiBin, nBins = hiBin - loBin + 1;
  float *srcM = NULL, *srcP = NULL, *srcL = NULL;
  const float *srcLP;
  if (reqMag) {
    srcM = (float *)malloc(sizeof(float) * Nsrc);
    for (i = 0; i < Nsrc; i++) srcM[i] = sp->squareInput ? src[i] : (src[i] > 0.0 ? sqrtf(src[i]) : 0.0f);
  }
  if (reqPow) {
    srcP = (float *)malloc(sizeof(float) * Nsrc);
    for (i = 0; i < Nsrc; i++) srcP[i] = sp->squareInput ? src[i] * src[i] : src[i];
  }
  if (reqLog) {                                                /* :700-729 */
    float logSpecFactor = (float)(10.0 / log(10.0));
    float myF = logSpecFactor;
    const float *mySrc;
    if (reqPow) mySrc = srcP;
    else if (reqMag) { mySrc = srcM; logSpecFactor *= 2.0; }
    else { mySrc = src; if (sp->squareInput) logSpecFactor *= 2.0; }
    srcL = (float *)malloc(sizeof(float) * Nsrc);
    for (i = 0; i < Nsrc; i++) srcL[i] = (mySrc[i] <= specFloor) ? logSpecFloor : myF * logf(mySrc[i]);
  }
  srcLP = useLog ? srcL : srcP;

  double frameSum = 0.0;                                       /* :766-771 */
  if ((sp->normBandEnergies || sp->sharpness || sp->nRollOff > 0) && srcP)   /* no power spectrum requested (flux only): nothing reads frameSum */
    for (i = loBin; i <= hiBin; i++) frameSum += srcP[i];

  for (i = 0; i < sp->nBands; i++) {                           /* :775-870 */
    long bL = (long)sp->bandLo[i], bH = (long)sp->bandHi[i];
    if (!(bL >= 0 && bH > 0)) continue;
    double idxL, wL, idxR, wR;
    edge_lo(c, (double)bL, &idxL, &wL); if (wL == 0.0) wL = 1.0;
    edge_hi(c, (double)bH, &idxR, &wR); if (wR == 0.0) wR = 1.0;
    long iL = (long)floor(idxL), iR = (long)floor(idxR);
    if (iL >= Nsrc) { iL = iR = Nsrc - 1; wR = 0.0; wL = 0.0; }
    if (iR >= Nsrc) { iR = Nsrc - 1; wR = 1.0; }
    if (iL < 0) iL = 0; if (iR < 0) iR = 0;
    double sum = (double)srcP[iL] * wL;
    for (j = iL + 1; j < iR; j++) sum += (double)srcP[j];
    sum += (double)srcP[iR] * wR;
    if (sp->normBandEnergies) dst[n++] = frameSum > 0.0 ? (float)(sum / frameSum) : 0.0f;
    else if (nBins > 0) dst[n++] = useLog ? (float)(10.0 * log(sum / (double)nBins) / log(10.0)) : (float)(sum / (double)nBins);
    else dst[n++] = 0.0f;
  }
  for (i = 0; i < sp->nSlopes; i++) {                          /* :873-993 */
    long bL = (long)sp->slopeLo[i], bH = (long)sp->slopeHi[i];
    if (!(bL >= 0 && bH > 0)) continue;
    double idxL, wL, idxR, wR;
    edge_lo(c, (double)bL, &idxL, &wL); if (wL == 0.0) wL = 1.0;
    edge_hi(c, (double)bH, &idxR, &wR); if (wR == 0.0) wR = 1.0;
    long iL = (long)floor(idxL), iR = (long)floor(idxR);
    if (iL >= Nsrc) { iL = iR = Nsrc - 1; wR = 0.0; wL = 0.0; }
    if (iR >= Nsrc) { iR = Nsrc - 1; wR = 1.0; }
    if (iL < 0) iL = 0; if (iR < 0) iR = 0;
    double Nind = idxR - idxL;
    double Sf = (double)frq[iL] * wL, S2f = Sf * Sf;
    double sumA = (double)frq[iL] * wL * (double)srcLP[iL], sumB = wL * srcLP[iL];
    for (long ii = iL + 1; ii < iR && ii < Nsrc; ii++) {
      S2f += (double)frq[ii] * (double)frq[ii];
      Sf += (double)frq[ii];
      sumA += (double)frq[ii] * (double)srcLP[ii];
      sumB += (double)srcLP[ii];
    }
    S2f += (double)frq[iR] * wR * (double)frq[iR] * wR;
    Sf += (double)frq[iR] * wR;
    sumA += (double)frq[iR] * wR * (double)srcLP[iR];
    sumB += wR * (double)srcLP[iR];
    double deno = (Nind * S2f - Sf * Sf), slope = 0.0;
    if (deno != 0.0) slope = (Nind * sumA - Sf * sumB) / deno;
    dst[n++] = sp->oldSlopeScale ? (float)(slope * (Nind - 1.0)) : (float)slope;
  }
  if (sp->alphaRatio) {                                        /* :996-1037 */
    float sum01 = 0.0f, sum15 = 0.0f;
    for (j = 0; j < Nsrc; j++) {
      if (frq[j] > 5000.0) break;
      if (frq[j] < 1000.0) sum01 += srcP[j]; else sum15 += srcP[j];
    }
    if (sum01 > 0.0) {
      if (useLog) dst[n++] = (sum15 > specFloor) ? (float)(10.0 * log(sum15 / sum01) / log(10.0))
                                                : (float)(10.0 * (log(specFloor) - log(sum01)) / log(10.0));
      else dst[n++] = sum15 / sum01;
    } else dst[n++] = 0.0f;
  }
  if (sp->hammarbergIndex) {                                   /* :1040-1089 */
    float max02 = 0.0f, max25 = 0.0f;
    for (j = 0; j < Nsrc; j++) {
      if (frq[j] > 5000.0) break;
      if (frq[j] < 2000.0) { if (srcP[j] > max02) max02 = srcP[j]; } else { if (srcP[j] > max25) max25 = srcP[j]; }
    }
    if (max25 > 0.0) {
      if (useLog) dst[n++] = (max02 > specFloor) ? (float)(10.0 * log(max02 / max25) / log(10.0))
                                                : (float)(10.0 * (log(specFloor) - log(max25)) / log(10.0));
      else dst[n++] = max02 / max25;
    } else dst[n++] = 0.0f;
  }
  double sumB = 0.0, sumC = 0.0;                               /* :1092-1099 */
  if (sp->normBandEnergies && !useLog) sumB = frameSum;
  else if (srcLP) for (j = loBin; j <= hiBin; j++) sumB += (double)srcLP[j];   /* (flux only: no log / power spectrum, nothing reads sumB) */
  if (sp->nRollOff > 0) {                                      /* roll-off :1103-1122 */
    float ro[OSM_OR_MAX_LIST];
    for (i = 0; i < sp->nRollOff; i++) ro[i] = 0.0f;
    for (j = loBin; j <= hiBin; j++) {
      sumC += (double)srcP[j];
      for (i = 0; i < sp->nRollOff; i++) {
        if (sp->buggyRollOff == 1 && i > 0) sumC += (double)srcP[j];
        if ((ro[i] == 0.0) && (sumC >= sp->rollOff[i] * frameSum)) ro[i] = (float)frq[j];
      }
    }
    for (i = 0; i < sp->nRollOff; i++) dst[n++] = ro[i];
  }
  if (sp->flux) {                                              /* :1125-1254 */
    if (!c->havePrev) { dst[n++] = 0.0f; c->havePrev = 1; }
    else {
      double myA = 0.0;
      for (j = loBin; j <= hiBin; j++) {
        double myB = ((double)srcM[j] / 1.0 - (double)c->prev[j - loBin] / 1.0);
        myA += myB * myB;
      }
      double fl = nBins > 0 ? myA / (double)nBins : 0.0;
      dst[n++] = fl > 0.0 ? (float)sqrt(fl) : 0.0f;
    }
    for (j = loBin; j <= hiBin; j++) c->prev[j - loBin] = srcM[j];
  }
  float ctr = 0.0f;                                            /* centroid :1257-1312 */
  double sumA = 0.0;
  if (sp->centroid || sp->standardDeviation || sp->variance || sp->skewness || sp->kurtosis || sp->slope) {
    for (j = loBin; j <= hiBin; j++) sumA += (double)frq[j] * (double)srcLP[j];
    if (sumB != 0.0) ctr = (float)(sumA / sumB);
    if (sp->centroid) dst[n++] = ctr;
  }
  if (sp->maxPos || sp->minPos) {                              /* :1314-1330 */
    long maP = loBin, miP = loBin;
    float mx = srcLP[loBin], mn = srcLP[loBin];
    for (j = loBin + 1; j < hiBin; j++) {
      if (srcLP[j] < mn) { mn = srcLP[j]; miP = j; }
      if (srcLP[j] > mx) { mx = srcLP[j]; maP = j; }
    }
    if (sp->maxPos) dst[n++] = (float)frq[maP];
    if (sp->minPos) dst[n++] = (float)frq[miP];
  }
  if (sp->entropy) dst[n++] = stat_entropy(srcLP + loBin, hiBin - loBin + 1);   /* :1333-1336 */
  if (sp->standardDeviation || sp->variance || sp->skewness || sp->kurtosis) { /* :1338-1397 */
    double u = ctr, m2 = 0.0, m3 = 0.0, m4 = 0.0;
    for (i = loBin; i <= hiBin; i++) {
      double t1 = ((double)frq[i] - u);
      double m = t1 * t1 * (double)srcLP[i];
      m2 += m; m *= t1; m3 += m; m4 += m * t1;
    }
    double sigma2 = 0.0;
    if (sumB != 0.0) sigma2 = m2 / sumB;
    if (sp->standardDeviation) dst[n++] = sigma2 > 0.0 ? (float)sqrt(sigma2) : 0.0f;
    if (sp->variance) dst[n++] = (float)sigma2;
    if (sp->skewness) dst[n++] = sigma2 <= 0.0 ? 0.0f : (float)(m3 / (sumB * sigma2 * sqrt(sigma2)));
    if (sp->kurtosis) dst[n++] = sigma2 == 0.0 ? 0.0f : (float)(m4 / (sumB * sigma2 * sigma2));
  }
  if (sp->slope) {                                             /* :1400-1427 */
    double Sf = 0.0, S2f = 0.0, Nind = (double)nBins;
    for (i = loBin; i <= hiBin && i < Nsrc; i++) { S2f += (double)frq[i] * (double)frq[i]; Sf += (double)frq[i]; }
    double deno = (Nind * S2f - Sf * Sf), slope = 0.0;
    if (deno != 0.0) slope = (Nind * sumA - Sf * sumB) / deno;
    dst[n++] = sp->oldSlopeScale ? (float)(slope * (Nind - 1.0)) : (float)slope;
  }
  if (sp->sharpness) {                                         /* :1429-1478 */
    float sumAA = 0.0f, c2 = 0.0f;
    for (j = loBin; j <= hiBin && j < Nsrc; j++) sumAA += (float)(c->sharpW[j - loBin] * (double)srcP[j]);
    if (frameSum != 0.0) c2 = (float)(sumAA / frameSum);
    dst[n++] = (float)(0.11 * c2);
  }
  if (sp->harmonicity) {                                       /* :1484-1513 */
    float ptpSum = 0.0f, lastPeak = -99.0f;
    for (j = loBin + 2; j < hiBin - 1; j++) {
      if ((srcLP[j - 2] < srcLP[j] && srcLP[j - 1] < srcLP[j] && srcLP[j] > srcLP[j + 1] && srcLP[j] > srcLP[j + 2]) ||
          (srcLP[j - 2] > srcLP[j] && srcLP[j - 1] > srcLP[j] && srcLP[j] < srcLP[j + 1] && srcLP[j] < srcLP[j + 2])) {
        if (lastPeak != -99.0) ptpSum += fabs(srcLP[j] - lastPeak);
        lastPeak = srcLP[j];
      }
    }
    ptpSum /= 2.0;
    if (sp->normBandEnergies && sumB != 0.0) {
      if (useLog) ptpSum /= (float)fabs(sumB); else ptpSum /= (float)(frameSum);
    } else ptpSum /= (float)nBins;
    dst[n++] = ptpSum;
  }
  if (sp->flatness) {                                          /* :1515-1544 */
    float sf = 0.0f, gmean = 0.0f;
    int nGm = 0;
    if (sumB != 0.0) {
      for (j = loBin; j <= hiBin; j++) if (srcLP[j] != 0.0) { gmean += log(fabs(srcLP[j])); nGm++; }
      if (nGm > 0) gmean /= (float)nGm;
      gmean = exp(gmean);
      sf = gmean / (float)fabs(sumB / (double)nBins);
    }
    if (sp->logFlatness) dst[n++] = sf > 0.0 ? (float)log(sf) : 0.0f; else dst[n++] = sf;
  }
  free(srcM); free(srcP); free(srcL);
}

static void spec_mag_frame(void *vctx, const float *mag, long nb, float *dst)
{
  (void)nb;
  spectral_frame((spec_ctx *)vctx, mag, dst);
}

/* cSpectral's per-frame context for the geometry of fe (bin frequencies, spectral range, sharpness weights) */
static void spec_ctx_init(spec_ctx *c, const osm_or_frontend *fe, const osm_or_spectral_cfg *sp)
{
  long N = osm_or_frame_size_samples(fe);
  long nfft = osm_or_fft_size(N), Nsrc = nfft / 2 + 1;
  memset(c, 0, sizeof *c);
  c->sp = sp; c->Nsrc = Nsrc; c->fsSec = osm_or_fft_frame_size_sec(fe);
  c->frq = (double *)malloc(sizeof(double) * Nsrc);
  double F0 = (double)(1.0) / (double)c->fsSec;                /* transformFft.cpp:111-115 */
  for (long i = 0; i < Nsrc; i++) c->frq[i] = F0 * (double)i;
  /* spectral range :625-647 */
  long lo = (long)sp->freqRangeLo, hi = (long)sp->freqRangeHi;
  if (lo == hi && hi == 0) { c->loBin = 1; c->hiBin = Nsrc - 1; }
  else {
    c->loBin = -1; c->hiBin = -1;
    for (long i = 0; i < Nsrc; i++) {
      if ((double)lo >= c->frq[i]) c->loBin = i;
      if ((double)hi > c->frq[i]) c->hiBin = i;
    }
    if (c->hiBin == -1 || c->hiBin >= Nsrc) c->hiBin = Nsrc - 1;
    if (c->loBin < 0) c->loBin = 0;
  }
  c->prev = (float *)calloc(Nsrc, sizeof(float));
  c->sharpW = (double *)calloc(Nsrc, sizeof(double));
  for (long j = c->loBin; j <= c->hiBin; j++) {                /* :1443-1453 (linear scale -> bark) */
    double fb = bark_fwd(c->frq[j]);
    c->sharpW[j - c->loBin] = fb * sharp_g(fb);
  }
}

static void spec_ctx_free(spec_ctx *c) { free(c->frq); free(c->prev); free(c->sharpW); }

long osm_or_spectral(const osm_or_frontend *fe, const osm_or_spectral_cfg *sp,
                     const int16_t *pcm, long L, int n_chan, float *out)
{
  long N = osm_or_frame_size_samples(fe), H = osm_or_frame_step_samples(fe);
  long T = osm_or_num_frames(L, N, H);
  if (T <= 0) return 0;
  spec_ctx c;
  spec_ctx_init(&c, fe, sp);
  int K = osm_or_spectral_num_out(sp);
  run_frames(fe, pcm, L, n_chan, spec_mag_frame, &c, K, out, NULL);
  spec_ctx_free(&c);
  return T;
}

long osm_or_spectral_from_mag(const osm_or_frontend *fe, const osm_or_spectral_cfg *sp, const float *mag, long T, float *out)
{
  if (T <= 0) return 0;
  spec_ctx c;
  spec_ctx_init(&c, fe, sp);
  int K = osm_or_spectral_num_out(sp);
  for (long t = 0; t < T; t++) spectral_frame(&c, mag + t * c.Nsrc, out + t * K);
  spec_ctx_free(&c);
  return T;
}


/* ------------------------------------------------------------------ a-10 cAcf + cPitchACF */

int osm_or_pitchacf_num_out(const osm_or_pitchacf_cfg *pc)
{
  return (pc->voiceProb ? 1 : 0) + (pc->HNR ? 1 : 0) + (pc->HNRdB ? 1 : 0) + (pc->linHNR ? 1 : 0) +
         (pc->voiceQual ? 1 : 0) + (pc->F0 ? 1 : 0) + (pc->F0raw ? 1 : 0) + (pc->F0env ? 1 : 0);
}

typedef struct {
  const osm_or_pitchacf_cfg *pc;
  long Nsrc, N;             /* magnitude bins, FFT size */
  double *costab;           /* cos(2 pi i / N) */
  float *acf, *cep;         /* N/2 each, adjacent: acf is the reader's concatenated [acf ; cepstrum] */
  float fsSec;              /* (float) frameSizeSec of the acf level (pitchACF.cpp:107-110) */
  float lastPitch, lastlastPitch, glMeanPitch, pitchEnv;
  int onsFlag;
  float *tap_acf, *tap_cep; long t;
} pacf_ctx;

/* dspcore/acf.cpp:250-345 (non-inverse): inverse rdft of the (power / log) spectrum.
 * Ooura's rdft(n,-1,a): x[j] = (R0 + R_{n/2} (-1)^j)/2 + sum_{k=1}^{n/2-1} R_k cos(2 pi j k/n)
 * (dspcore/fftsg.c:104-122; the imaginary parts are zero here). */
static void acf_level(const pacf_ctx *c, const float *src, int usePower, int cepstrum, int absCeps, float *dst)
{
  long Nsrc = c->Nsrc, N = c->N, Ndst = Nsrc - 1;    /* symmetricData=1: nOutEl = nEl - 1 (acf.cpp:123-128) */
  float *r = (float *)malloc(sizeof(float) * Nsrc);
  const int oldCompat = cepstrum && c->pc->oldCompatCepstrum;
  for (long k = 0; k < Nsrc; k++) {
    float v = usePower ? src[k] * src[k] : src[k];    /* :253-261 */
    if (oldCompat) { if (k > 0 && k < Nsrc - 1) v = (v > 0.0) ? logf(v) : 0.0f; }   /* :276-286: float log, DC / Nyquist as is */
    else if (cepstrum) v = (v > 0.0) ? (float)log(v + 1.0) : 0.0f;   /* :289-305 */
    r[k] = v;
  }
  for (long j = 0; j < Ndst; j++) {
    double x = ((double)r[0] + (double)r[N / 2] * ((j & 1) ? -1.0 : 1.0)) / 2.0;
    for (long k = 1; k < N / 2; k++) x += (double)r[k] * c->costab[(j * k) % N];
    float d = (float)x;
    if (c->pc->acfCepsNormOutput && !oldCompat) d = d / (float)Nsrc;  /* :321-325 (oldCompatCepstrum: acf.cpp:104) */
    if (cepstrum) { if (absCeps || oldCompat) d = fabsf(d); }         /* :327-341 (oldCompatCepstrum: acf.cpp:105) */
    else d = fabsf(d);                                   /* :342-344 */
    dst[j] = d;
  }
  free(r);
}

/* lldcore/pitchACF.cpp:249-284 */
static double voicing_prob(const float *a, int n, int skip, double *Zcr)
{
  int zcr = 0, mcr = 0;
  double mean, max;
  max = a[n - 1];
  mean = a[skip];
  for (int i = 1; i < n; i++) {
    if (a[i - 1] * a[i] < 0) zcr++;
    if (i >= skip) {
      if ((a[i] > max) && (a[i - 1] < a[i])) max = a[i];
      mean += a[i];
    }
  }
  mean /= (double)(n - skip + 1);
  for (int i = 1; i < n; i++) if ((a[i - 1] - mean) * (a[i] - mean) < 0) mcr++;
  if (mcr > zcr) *Zcr = (double)mcr / (double)n; else *Zcr = (double)zcr / (double)n;
  if (a[0] > 0) return max / a[0];
  return 0.0;
}

/* lldcore/pitchACF.cpp:286-310 */
static long pitch_peak(const float *a, long n, long skip)
{
  double max, buf, sum = 0.0;
  max = a[n - 1];
  for (int i = (int)n - 1; i >= 0; i--) {
    buf = a[i];
    sum += fabs(buf);
    if (i >= skip) if (buf > max) max = buf;
  }
  sum /= n;
  for (int i = (int)skip + 1; i < n - 1; i++)
    if (a[i] > (max + sum) * 0.6)
      if ((a[i - 1] < a[i]) && (a[i] > a[i + 1])) return i;
  return 0;
}

/* lldcore/pitchACF.cpp:137-247 */
static void pitchacf_frame(void *vctx, const float *mag, long nb, float *dst)
{
  pacf_ctx *c = (pacf_ctx *)vctx;
  const osm_or_pitchacf_cfg *pc = c->pc;
  (void)nb;
  long N = c->Nsrc - 1;                       /* length of each cAcf level */
  acf_level(c, mag, pc->acfUsePower, 0, 0, c->acf);
  acf_level(c, mag, pc->cepUsePower, 1, pc->absCepstrum, c->cep);
  if (c->tap_acf) memcpy(c->tap_acf + c->t * N, c->acf, sizeof(float) * N);
  if (c->tap_cep) memcpy(c->tap_cep + c->t * N, c->cep, sizeof(float) * N);
  c->t++;
  const float *src = c->acf;                  /* the reader concatenates [acf ; cepstrum], Nsrc = 2N */
  long NsrcCat = 2 * N;
  double Nd = (double)NsrcCat;
  double Tsamp = c->fsSec / Nd;
  double maxPitch = pc->maxPitch < 0.0 ? 0.0 : pc->maxPitch;
  double voicingCutoff = pc->voicingCutoff > 1.0 ? 1.0 : (pc->voicingCutoff < 0.0 ? 0.0 : pc->voicingCutoff);
  int preskip = (maxPitch <= 0.0) ? 0 : (int)(1.0 / (maxPitch * Tsamp));
  double acfZcr = 0.0;
  double voicing = voicing_prob(src, (int)N, preskip, &acfZcr);
  long maxIdx = pitch_peak(c->cep, N, preskip + 1);
  double hnr = 0.0, hnrDB = 0.0, hnrLin = 0.0;
  if (pc->HNR) {                              /* :312-326 */
    double buf = ((src[0] - src[maxIdx]) == 0.0) ? 100000000000000000000.0 : src[maxIdx] / (src[0] - src[maxIdx]);
    hnr = (buf > 0.00000000001) ? 10.0 * log(buf) : 10.0 * log(0.00000000001);
  }
  if (pc->HNRdB) {                            /* :329-343 */
    double buf = src[0] - src[maxIdx];
    buf = (buf == 0.0) ? 10e10 : src[maxIdx] / buf;
    hnrDB = (buf <= 10e-10) ? -100.0 : ((buf >= 10e10) ? +100.0 : 10.0 * log(buf) / log(10.0));
  }
  if (pc->linHNR) {                           /* :346-360 */
    double buf = src[0] - src[maxIdx];
    buf = (buf == 0.0) ? 10e3 : src[maxIdx] / buf;
    hnrLin = (buf <= 10e-3) ? 10e-3 : ((buf >= 10e3) ? 10e3 : buf);
  }
  int n = 0;
  if (pc->voiceProb) dst[n++] = (float)voicing;
  if (pc->HNR) dst[n++] = (float)hnr;
  if (pc->HNRdB) dst[n++] = (float)hnrDB;
  if (pc->linHNR) dst[n++] = (float)hnrLin;
  if (pc->F0 || pc->F0env || pc->voiceQual || pc->F0raw) {   /* :181-245 */
    float vq = ((float)maxPitch - (float)fabs((acfZcr * maxPitch) - ((float)1.0 / ((float)(maxIdx) * (float)Tsamp)))) * (float)voicing;
    if (maxIdx == 0.0) vq = 0.0;
    if (pc->voiceQual) dst[n++] = vq;
    float pitch = 0.0f, rawF0 = 0.0f;
    if (maxIdx > 0) { pitch = (float)1.0 / ((float)(maxIdx) * (float)Tsamp); rawF0 = pitch; }
    if (voicing < voicingCutoff) { maxIdx = 0; pitch = 0.0; }
    if ((c->lastPitch == 0.0) && (pitch > 0.0)) c->onsFlag = 1;
    if ((c->lastPitch > 0.0) && (pitch == 0.0) && (c->onsFlag == 0)) c->onsFlag = -1;
    if ((c->lastPitch > 0.0) && (pitch > 0.0)) c->onsFlag = 0;
    if ((c->lastPitch == 0.0) && (pitch == 0.0)) c->onsFlag = 0;
    if ((pitch == 0.0) && (c->onsFlag == 1)) c->lastPitch = 0.0;
    float oPitch = pitch, tol = (float)0.4, alpha = (float)0.3;
    if (pitch > 0.0) {
      if (c->glMeanPitch == 0.0) c->glMeanPitch = pitch;
      if (!((pitch < ((float)1.0 + tol) * c->glMeanPitch) && (pitch > ((float)1.0 - tol) * c->glMeanPitch))) {
        pitch = c->glMeanPitch;
        alpha /= (float)3.0;
      }
      if (c->onsFlag && (c->lastPitch > pitch)) c->lastPitch *= (float)0.85;
    }
    if ((pitch > 0.0) && (c->onsFlag == -1)) c->lastPitch = pitch;
    if (oPitch > (float)0.0) c->glMeanPitch = ((float)1.0 - alpha) * c->glMeanPitch + alpha * oPitch;
    float out;
    if ((c->lastlastPitch != (float)0.0) && (c->lastPitch != 0.0)) out = (float)0.5 * (c->lastlastPitch + c->lastPitch);
    else out = c->lastPitch;
    if (pc->F0) dst[n++] = out;
    if (pc->F0raw) dst[n++] = rawF0;
    c->lastlastPitch = c->lastPitch;
    c->lastPitch = pitch;
    if (pc->F0env) {
      if (out > 0.0) c->pitchEnv = (float)0.75 * c->pitchEnv + (float)0.25 * out;
      dst[n++] = c->pitchEnv;
    }
  }
}

/* preskip (pitchACF.cpp:155-159) of fe's geometry; the reference reads [acf ; cepstrum][preskip], outside its input from
 * preskip = nfft on: refused (-1) like the plan refuses it */
static int pacf_ctx_init(pacf_ctx *c, const osm_or_frontend *fe, const osm_or_pitchacf_cfg *pc)
{
  long N0 = osm_or_frame_size_samples(fe);
  long nfft = osm_or_fft_size(N0), Nsrc = nfft / 2 + 1;
  memset(c, 0, sizeof *c);
  c->pc = pc; c->Nsrc = Nsrc; c->N = nfft;
  c->fsSec = (float)osm_or_fft_frame_size_sec(fe);     /* cAcf keeps the level's frameSizeSec */
  double maxPitch = pc->maxPitch < 0.0 ? 0.0 : pc->maxPitch;
  int preskip = (maxPitch <= 0.0) ? 0 : (int)(1.0 / (maxPitch * ((double)c->fsSec / (double)nfft)));
  if (preskip >= nfft) return -1;
  c->costab = (double *)malloc(sizeof(double) * nfft);
  for (long i = 0; i < nfft; i++) c->costab[i] = cos(2.0 * M_PI * (double)i / (double)nfft);
  c->acf = (float *)malloc(sizeof(float) * 2 * (Nsrc - 1));
  c->cep = c->acf + (Nsrc - 1);
  return 0;
}

long osm_or_pitchacf(const osm_or_frontend *fe, const osm_or_pitchacf_cfg *pc,
                     const int16_t *pcm, long L, int n_chan, float *out, float *tap_acf, float *tap_cep)
{
  long N0 = osm_or_frame_size_samples(fe), H = osm_or_frame_step_samples(fe);
  long T = osm_or_num_frames(L, N0, H);
  if (T <= 0) return 0;
  pacf_ctx c;
  if (pacf_ctx_init(&c, fe, pc) != 0) return -1;
  c.tap_acf = tap_acf; c.tap_cep = tap_cep;
  int K = osm_or_pitchacf_num_out(pc);
  run_frames(fe, pcm, L, n_chan, pitchacf_frame, &c, K, out, NULL);
  free(c.costab); free(c.acf);
  return T;
}

long osm_or_pitchacf_from_mag(const osm_or_frontend *fe, const osm_or_pitchacf_cfg *pc, const float *mag, long T, float *out,
                              float *tap_acf, float *tap_cep)
{
  if (T <= 0) return 0;
  pacf_ctx c;
  if (pacf_ctx_init(&c, fe, pc) != 0) return -1;
  c.tap_acf = tap_acf; c.tap_cep = tap_cep;
  int K = osm_or_pitchacf_num_out(pc);
  for (long t = 0; t < T; t++) pitchacf_frame(&c, mag + t * c.Nsrc, c.Nsrc, out + t * K);
  free(c.costab); free(c.acf);
  return T;
}
