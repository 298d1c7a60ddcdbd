/* tonefilt_oracle.c -- literal C restatement of the reference's cTonefilt (lld/tonefilt.cpp:65-134 options and block length,
 * :180-189 tables, :204-226 the per-sample loop with libm sin / cos), test infrastructure.  x = the float wave level, L samples;
 * out = ceil(L / P) rows of nNotes values; the last block is padded with copies of the last sample.  Returns the row count.
 *   gcc -O2 -ffp-contract=off -shared -fPIC -o tonefilt_oracle.so tonefilt_oracle.c -lm */
#include <math.h>
#include <stdlib.h>

long tfo_rows(long L, double fs, double outputPeriod, long *P_out)
{
  const double T = 1.0 / fs;
  if (outputPeriod <= 0.0) outputPeriod = 0.1;
  long P = (long)round(outputPeriod / T);
  if (outputPeriod < T) P = 1;
  if (P_out) *P_out = P;
  return (L + P - 1) / P;
}

long tfo_run(const float *x, long L, double fs, int nNotes, double firstNote, double decayF0, double decayFN, double outputPeriod,
             float *out)
{
  if (decayFN < 0.0) decayFN = 0.0;
  if (decayFN > 1.0) decayFN = 1.0;
  if (decayF0 < decayFN) decayF0 = decayFN;
  if (decayF0 < 0.0) decayF0 = 0.0;
  if (decayF0 > 1.0) decayF0 = 1.0;
  if (firstNote <= 0.0) firstNote = 1.0;
  if (nNotes < 1) nNotes = 1;
  long P;
  const long rows = tfo_rows(L, fs, outputPeriod, &P);
  const double inputPeriod = 1.0 / fs;
  double *freq = malloc(sizeof(double) * nNotes), *decayF = malloc(sizeof(double) * nNotes);
  double *s = calloc(nNotes, sizeof(double)), *c = calloc(nNotes, sizeof(double));
  float *blk = malloc(sizeof(float) * P);
  int n, t;
  for (n = 0; n < nNotes; n++) freq[n] = firstNote * pow(2.0, (double)n / 12.0);
  for (n = 0; n < nNotes; n++) decayF[n] = decayFN + (decayF0 - decayFN) * (freq[n] - freq[0]) / (freq[nNotes - 1]);
  long pos = 0, r, j;
  for (r = 0; r < rows; r++) {
    for (j = 0; j < P; j++) blk[j] = x[(r * P + j < L) ? r * P + j : L - 1];
    for (t = 0; t < nNotes; t++) {
      const double f = freq[t];
      long idx = pos;
      for (n = 0; n < P; n++) {
        double time = (double)(idx + n) * inputPeriod;
        s[t] = decayF[t] * s[t] + (1.0 - decayF[t]) * sin(2.0 * M_PI * f * time) * (double)blk[n];
        c[t] = decayF[t] * c[t] + (1.0 - decayF[t]) * cos(2.0 * M_PI * f * time) * (double)blk[n];
      }
      float y = (float)sqrt(c[t] * c[t] + s[t] * s[t]);
      y *= 10.0;
      out[r * nNotes + t] = y;
    }
    pos += P;
  }
  free(freq); free(decayF); free(s); free(c); free(blk);
  return rows;
}
