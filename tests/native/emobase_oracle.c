/*
 * emobase_oracle.c -- plain-C restatement of the pieces of config/emobase/emobase.conf that the project's general oracle
 * (oracle/osm_oracle.c) does not cover (test infrastructure; the product never links it, tests/emobase_oracle.py loads it):
 *   - stand-alone cLpc, method acf, on a frame level: smileDsp_autoCorr + smileDsp_calcLpcAcf (smileutil/smileUtil.c:1560-1627)
 *   - cLsp: cheb_poly_eva, lpc_to_lsp, processVector (lld/lsp.cpp:113-313)
 *   - cAcf (ACF, usePower = 1, acfCepsNormOutput = 0) + cAcf (cepstrum, usePower = 1, oldCompatCepstrum = 1) -> cPitchACF
 *     (dspcore/acf.cpp:103-109,250-345, lldcore/pitchACF.cpp:137-361) with voiceProb, F0 and F0env, on a magnitude level.
 * Written from the reference's statements, independently of the kernel's (opensmile_b200/csrc/lsp_math.cuh); compile without
 * FMA contraction (-ffp-contract=off).  Citations relative to /root/reference/src.
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif

/* smileDsp_autoCorr + smileDsp_calcLpcAcf, float throughout; a[0..p-1], returns the gain (0 when r[0] == 0) */
float emo_lpc(const float *x, long n, int p, float *a)
{
  float r[64];
  int lag = p + 1;
  while (lag) {
    r[--lag] = 0.0f;
    for (long i = lag; i < n; i++) r[lag] += x[i] * x[i - lag];
  }
  if (r[0] == 0.0f) { for (int i = 0; i < p; i++) a[i] = 0.0f; return 0.0f; }
  float e = r[0];
  for (int m = 1; m <= p; m++) {
    float sum = 1.0f * r[m];
    for (int i = 1; i < m; i++) sum += a[i - 1] * r[m - i];
    float k_m = (-1.0f / e) * sum;
    a[m - 1] = k_m;
    for (int i = 1; i <= m / 2; i++) {
      float xx = a[i - 1];
      a[i - 1] += k_m * a[m - i - 1];
      if ((i < (m / 2)) || ((m & 1) == 1)) a[m - i - 1] += k_m * xx;
    }
    e *= (1.0f - k_m * k_m);
    if (e == 0.0f) { for (int i = m; i < p; i++) a[i] = 0.0f; break; }
  }
  return e;
}

/* cLsp::cheb_poly_eva */
static float lsp_cheb(const float *coef, float x, int m)
{
  float b0 = 0, b1 = 0, tmp;
  x *= 2;
  for (int k = m; k > 0; k--) { tmp = b0; b0 = x * b0 - b1 + coef[m - k]; b1 = tmp; }
  return (-b1 + (float)0.5 * x * b0 + coef[m]);
}

/* cLsp::lpc_to_lsp; the reference's C++ build resolves acos(float) to the float overload */
static int lsp_search(const float *a, int lpcrdr, float *freq, int nb, float delta)
{
  float P[17], Q[17];
  int m = lpcrdr / 2, roots = 0;
  P[0] = 1.f; Q[0] = 1.f;
  for (int i = 0; i < m; i++) { P[i + 1] = (a[i] + a[lpcrdr - 1 - i]) - P[i]; Q[i + 1] = (a[i] - a[lpcrdr - 1 - i]) + Q[i]; }
  for (int i = 0; i < m; i++) { P[i] = 2 * P[i]; Q[i] = 2 * Q[i]; }
  float xr = 0, xl = 1.0, xm = 0;
  for (int j = 0; j < lpcrdr; j++) {
    const float *pt = (j & 1) ? Q : P;
    float psuml = lsp_cheb(pt, xl, m), psumr, psumm;
    int flag = 1;
    while (flag && (xr >= -1.0)) {
      float dd = delta * ((float)1.0 - (float)0.9 * xl * xl);
      if (fabsf(psuml) < .2) dd *= (float)0.5;
      xr = xl - dd;
      psumr = lsp_cheb(pt, xr, m);
      float temp_psumr = psumr, temp_xr = xr;
      if ((psumr * psuml) < 0.0) {
        roots++;
        for (int k = 0; k <= nb; k++) {
          xm = (float)0.5 * (xl + xr);
          psumm = lsp_cheb(pt, xm, m);
          if (!((psumm * psuml) < 0.0)) { psuml = psumm; xl = xm; } else { psumr = psumm; xr = xm; }
        }
        if (xm > 1.0) xm = 1.0; else if (xm < -1.0) xm = -1.0;
        freq[j] = acosf(xm);
        xl = xm;
        flag = 0;
      } else { psuml = temp_psumr; xl = temp_xr; }
    }
  }
  return roots;
}

/* cLsp::processVector (nb = 10, grids 0.2 then 0.05, zeros from the last root on); returns the roots of the 0.2 search */
int emo_lsp(const float *a, int p, float *lsf)
{
  int roots = lsp_search(a, p, lsf, 10, (float)0.2), first = roots;
  if (roots != p) {
    roots = lsp_search(a, p, lsf, 10, (float)0.05);
    for (int i = roots; i < p; i++) lsf[i] = 0.0f;
  }
  return first;
}

/* cLpc on every frame of the pre-emphasised (cVectorPreemphasis, dspcore/vectorPreemphasis.cpp:89-108), un-windowed framer level
 * of x[0..L-1] (the wave level as floats), frames of N samples every H; lpc [T x p], gain [T], lsp [T x p], roots1 [T] */
long emo_lpc_frames(const float *x, long L, long N, long H, float k, int p, float *lpc, float *gain, float *lsp, int *roots1)
{
  if (L < N || p < 1 || p > 16) return 0;
  long T = (L - N) / H + 1;
  float *y = (float *)malloc(sizeof(float) * N), a[16], lsf[16];
  for (long t = 0; t < T; t++) {
    const float *fx = x + t * H;
    y[0] = (1 - k) * fx[0];
    for (long n = 1; n < N; n++) y[n] = fx[n] - k * fx[n - 1];
    float g = emo_lpc(y, N, p, a);
    memcpy(lpc + t * p, a, sizeof(float) * p);
    gain[t] = g;
    roots1[t] = emo_lsp(a, p, lsf);
    memcpy(lsp + t * p, lsf, sizeof(float) * p);
  }
  free(y);
  return T;
}

/* dspcore/acf.cpp:250-345 (non-inverse, symmetricData = 1): Ooura's rdft(n, -1) of the real, even input as a cosine sum in double.
 * cepstrum = 0: usePower = 1, acfCepsNormOutput = 0, |.|.  cepstrum = 1 with oldCompatCepstrum = 1 (:103-109, :276-286): log(x) of
 * the float (the float overload), 0 for x <= 0, DC and Nyquist un-logged; acfCepsNormOutput forced 0, absCepstrum forced 1. */
static void acf_level(const float *mag, long Nsrc, const double *costab, int cepstrum, float *r, float *dst)
{
  long N = 2 * (Nsrc - 1), Ndst = Nsrc - 1;
  for (long k = 0; k < Nsrc; k++) {
    float v = mag[k] * mag[k];
    if (cepstrum && k > 0 && k < Nsrc - 1) v = (v > 0.0) ? logf(v) : 0.0f;
    r[k] = v;
  }
  for (long j = 0; j < Ndst; j++) {
    double s = ((double)r[0] + (double)r[N / 2] * ((j & 1) ? -1.0 : 1.0)) / 2.0;
    for (long k = 1; k < N / 2; k++) s += (double)r[k] * costab[(j * k) % N];
    dst[j] = fabsf((float)s);
  }
}

/* lldcore/pitchACF.cpp:249-284 */
static double voicing_prob(const float *a, int n, int skip, double *Zcr)
{
  int zcr = 0, mcr = 0;
  double mean, max = a[n - 1];
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
  *Zcr = (mcr > zcr) ? (double)mcr / (double)n : (double)zcr / (double)n;
  return (a[0] > 0) ? max / a[0] : 0.0;
}

/* lldcore/pitchACF.cpp:286-310 */
static long pitch_peak(const float *a, long n, long skip)
{
  double max = a[n - 1], buf, sum = 0.0;
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

/* mag [T x Nsrc] (the cFFTmagphase level) -> out [T x 3] = voiceProb, F0, F0env (lldcore/pitchACF.cpp:137-247, the F0 state
 * machine carried over the frames of one utterance); cep [T x (Nsrc - 1)] = the cepstrum level (optional).  fsSec = frameSizeSec
 * of the magnitude level (after cTransformFFT's rescale). */
long emo_acf_pitch(const float *mag, long T, long Nsrc, float fsSec, double maxPitch, double voicingCutoff, float *out, float *cep)
{
  long N = Nsrc - 1, nfft = 2 * N;
  double *costab = (double *)malloc(sizeof(double) * nfft);
  for (long i = 0; i < nfft; i++) costab[i] = cos(2.0 * M_PI * (double)i / (double)nfft);
  float *r = (float *)malloc(sizeof(float) * Nsrc), *acf = (float *)malloc(sizeof(float) * N), *cp = (float *)malloc(sizeof(float) * N);
  float lastPitch = 0, lastlastPitch = 0, glMeanPitch = 0, pitchEnv = 0;
  int onsFlag = 0;
  double Tsamp = fsSec / (double)(2 * N);                 /* the reader concatenates [acf ; cepstrum] */
  if (maxPitch < 0.0) maxPitch = 0.0;
  if (voicingCutoff > 1.0) voicingCutoff = 1.0;
  if (voicingCutoff < 0.0) voicingCutoff = 0.0;
  int preskip = (maxPitch <= 0.0) ? 0 : (int)(1.0 / (maxPitch * Tsamp));
  for (long t = 0; t < T; t++) {
    acf_level(mag + t * Nsrc, Nsrc, costab, 0, r, acf);
    acf_level(mag + t * Nsrc, Nsrc, costab, 1, r, cp);
    if (cep) memcpy(cep + t * N, cp, sizeof(float) * N);
    double acfZcr = 0.0;
    double voicing = voicing_prob(acf, (int)N, preskip, &acfZcr);
    long maxIdx = pitch_peak(cp, N, preskip + 1);
    float *dst = out + t * 3;
    dst[0] = (float)voicing;
    float pitch = 0.0f;
    if (maxIdx > 0) pitch = (float)1.0 / ((float)(maxIdx) * (float)Tsamp);
    if (voicing < voicingCutoff) { maxIdx = 0; pitch = 0.0; }
    if ((lastPitch == 0.0) && (pitch > 0.0)) onsFlag = 1;
    if ((lastPitch > 0.0) && (pitch == 0.0) && (onsFlag == 0)) onsFlag = -1;
    if ((lastPitch > 0.0) && (pitch > 0.0)) onsFlag = 0;
    if ((lastPitch == 0.0) && (pitch == 0.0)) onsFlag = 0;
    if ((pitch == 0.0) && (onsFlag == 1)) lastPitch = 0.0;
    float oPitch = pitch, tol = (float)0.4, alpha = (float)0.3;
    if (pitch > 0.0) {
      if (glMeanPitch == 0.0) glMeanPitch = pitch;
      if (!((pitch < ((float)1.0 + tol) * glMeanPitch) && (pitch > ((float)1.0 - tol) * glMeanPitch))) {
        pitch = glMeanPitch;
        alpha /= (float)3.0;
      }
      if (onsFlag && (lastPitch > pitch)) lastPitch *= (float)0.85;
    }
    if ((pitch > 0.0) && (onsFlag == -1)) lastPitch = pitch;
    if (oPitch > (float)0.0) glMeanPitch = ((float)1.0 - alpha) * glMeanPitch + alpha * oPitch;
    float o = ((lastlastPitch != (float)0.0) && (lastPitch != 0.0)) ? (float)0.5 * (lastlastPitch + lastPitch) : lastPitch;
    dst[1] = o;
    lastlastPitch = lastPitch;
    lastPitch = pitch;
    if (o > 0.0) pitchEnv = (float)0.75 * pitchEnv + (float)0.25 * o;
    dst[2] = pitchEnv;
  }
  free(costab); free(r); free(acf); free(cp);
  return T;
}
