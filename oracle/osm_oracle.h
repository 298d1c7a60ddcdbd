/*
 * osm_oracle.h -- CPU restatement of openSMILE's per-frame LLD extraction path.
 *
 * TEST INFRASTRUCTURE ONLY.  This is the checker ("oracle") the CUDA path in
 * opensmile_b200/ is compared against.  Only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline leg may load it; nothing in the product links or imports it.
 *
 * Parity pinning: the reference ships no golden vectors for this path (SURVEY.md 8c), so
 * the restatement is pinned against the UNMODIFIED reference compiled from
 * /root/reference by oracle/Makefile (`make ref` -> oracle/_ref/SMILExtract) and against
 * the fixtures that binary produced (tests/golden/, generator scripts/make_golden.py).
 *
 * Every function cites the reference file:line it restates (paths relative to
 * /root/reference/src).  Types follow the reference: samples and features are float32
 * (FLOAT_DMEM, include/core/smileTypes.h:28); tables are built in double and cast where
 * the reference does so.  The one deliberate difference: the FFT is a textbook double
 * precision transform rounded to float, not Ooura's float32 split-radix (dspcore/fftsg.c)
 * -- the two agree to ~2e-7 of the frame's spectral peak (SURVEY.md H1), far inside the
 * 1e-5-of-scale parity budget.  Compile with -ffp-contract=off (the reference's x86-64
 * Release build has no FMA contraction).
 */
#ifndef OSM_ORACLE_H
#define OSM_ORACLE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { OSM_OR_WIN_RECT = 0, OSM_OR_WIN_HANN = 1, OSM_OR_WIN_HAMM = 2, OSM_OR_WIN_GAUSS = 3,
       OSM_OR_WIN_SINE = 4, OSM_OR_WIN_TRI = 5, OSM_OR_WIN_BARTLETT = 6 };

/* front end shared by every spectral LLD: cFramer -> cVectorPreemphasis -> cWindower ->
 * cTransformFFT -> cFFTmagphase */
typedef struct {
  double sample_rate;      /* Hz; wave level period T = 1/sample_rate (iocore/waveSource.cpp) */
  double frame_size_sec;   /* cFramer.frameSize */
  double frame_step_sec;   /* cFramer.frameStep */
  int    preemph_on;       /* 1 if a cVectorPreemphasis instance is in the chain */
  double preemph_k;        /* cVectorPreemphasis.k (cast to float like the reference) */
  int    win_func;         /* OSM_OR_WIN_* */
  double win_sigma;        /* cWindower.sigma (Gauss) */
  double win_gain;         /* cWindower.gain */
  double win_offset;       /* cWindower.offset */
  int    zero_pad_symmetric; /* cTransformFFT.zeroPadSymmetric */
} osm_or_frontend;

typedef struct {
  int    n_bands;          /* cMelspec.nBands */
  double lofreq, hifreq;   /* cMelspec.lofreq / hifreq */
  int    use_power;        /* cMelspec.usePower */
  int    htkcompatible;    /* cMelspec.htkcompatible */
  int    spec_scale;       /* cMelspec.specScale when htkcompatible = 0: 0 mel, 1 bark, 2 bark_speex, 3 bark_schroed, 4 semitone, 5 linear, 6 log */
  double scale_param;      /* firstNote (semitone) / logScaleBase (log) */
} osm_or_melspec;

typedef struct {
  int    first_mfcc, last_mfcc; /* cMfcc.firstMfcc / lastMfcc */
  double cep_lifter;       /* cMfcc.cepLifter */
  double melfloor;         /* cMfcc.melfloor (forced to 1.0 when htkcompatible) */
  int    htkcompatible;    /* cMfcc.htkcompatible */
} osm_or_mfcc;

typedef struct {
  int    lp_order;         /* cPlp.lpOrder */
  int    first_cc, last_cc;/* cPlp.firstCC / lastCC (resolved: -1 -> lpOrder) */
  int    do_log, do_aud, do_inv_log, do_idft, do_lp, do_lp_to_ceps;
  int    rasta, new_rasta;
  double rasta_upper, rasta_lower;
  double cep_lifter;
  double compression;      /* cPlp.compression */
  double melfloor;
  int    htkcompatible;
} osm_or_plp;

#define OSM_OR_MAX_LIST 16
typedef struct {            /* cSpectral (lldcore/spectral.cpp), same fields as osm_b200_spectral */
  int squareInput;
  int nBands;  double bandLo[OSM_OR_MAX_LIST], bandHi[OSM_OR_MAX_LIST];
  int nSlopes; double slopeLo[OSM_OR_MAX_LIST], slopeHi[OSM_OR_MAX_LIST];
  int nRollOff; double rollOff[OSM_OR_MAX_LIST];
  int flux, centroid, maxPos, minPos, entropy, standardDeviation, variance, skewness,
      kurtosis, slope, alphaRatio, hammarbergIndex, sharpness, harmonicity, flatness;
  int normBandEnergies, buggyRollOff, oldSlopeScale, useLogSpectrum;
  double freqRangeLo, freqRangeHi;
  double specFloor;
  int logFlatness;
} osm_or_spectral_cfg;

typedef struct {            /* cEnergy (lldcore/energy.cpp) */
  int htkcompatible, rms, energy2, log;
  double escaleLog, escaleRms, escaleSquare, ebiasLog, ebiasRms, ebiasSquare;
} osm_or_energy_cfg;

typedef struct { int zcr, mcr, amax, maxmin, dc; } osm_or_mzcr_cfg;   /* cMZcr (lldcore/mzcr.cpp) */
typedef struct { int intensity, loudness; } osm_or_intensity_cfg;        /* cIntensity (lldcore/intensity.cpp) */

typedef struct {            /* cAcf x2 + cPitchACF (dspcore/acf.cpp, lldcore/pitchACF.cpp) */
  int acfUsePower;          /* [acf] usePower (1) */
  int cepUsePower;          /* [cep] usePower (0 when cepstrum=1 and not set) */
  int absCepstrum;          /* [cep] absCepstrum (0) */
  int acfCepsNormOutput;    /* 1 */
  double maxPitch;          /* 500 */
  int voiceProb, voiceQual, HNR, HNRdB, linHNR, F0, F0raw, F0env;
  double voicingCutoff;     /* 0.55 */
  int oldCompatCepstrum;    /* [cep] oldCompatCepstrum (0): log(x) without +1, DC / Nyquist un-logged; forces absCepstrum = 1
                               and acfCepsNormOutput = 0 on the cepstrum (dspcore/acf.cpp:103-109,276-286) */
} osm_or_pitchacf_cfg;

/* ---- geometry (integer work, must be bit exact) ---- */
long osm_or_frame_size_samples(const osm_or_frontend *fe);
long osm_or_frame_step_samples(const osm_or_frontend *fe);
long osm_or_fft_size(long frame_size_samples);
long osm_or_num_frames(long n_samples, long frame_size, long frame_step);

/* ---- stage by stage ---- */
void osm_or_pcm16_to_float(const int16_t *pcm, long n_samples, int n_chan, float *out);
void osm_or_pcm_to_float(const void *buf, int format, long n_samples, int n_chan, float *out);
void osm_or_window_table(int win_func, long n, double sigma, double gain, double *w);
/* one frame: raw float samples (frame_size) -> magnitude spectrum (nfft/2+1) */
void osm_or_frame_to_mag(const osm_or_frontend *fe, const float *x, long frame_size,
                         long nfft, const double *win, float *fft_packed, float *mag);
/* frameSizeSec seen by cMelspec after cTransformFFT rescaled it (H2 quirk) */
double osm_or_fft_frame_size_sec(const osm_or_frontend *fe);

/* whole chains on one utterance (mono float or int16 PCM) -------------------------------
 * out must hold n_frames * n_out floats; functions return the number of frames written
 * (or <0 on error).  tap_* pointers are optional (NULL) intermediate dumps. */
long osm_or_mfcc_d_a(const osm_or_frontend *fe, const osm_or_melspec *ms, const osm_or_mfcc *mf,
                     int delta_win, int accel_win,
                     const int16_t *pcm, long n_samples, int n_chan,
                     float *out, float *tap_mag, float *tap_mel);

long osm_or_plp_d_a(const osm_or_frontend *fe, const osm_or_melspec *ms, const osm_or_plp *pl,
                    int delta_win, int accel_win,
                    const int16_t *pcm, long n_samples, int n_chan,
                    float *out, float *tap_mel);

int osm_or_plp_num_out(const osm_or_plp *pl, int n_bands);
/* cPlp static level only, with RASTA / newRASTA if configured: out = [T][num_out] */
long osm_or_plp_static(const osm_or_frontend *fe, const osm_or_melspec *ms, const osm_or_plp *pl,
                       const int16_t *pcm, long n_samples, int n_chan, float *out);
/* cFullinputMean (default mode): per-column mean over all T frames subtracted (dspcore/fullinputMean.cpp:484-548) */
void osm_or_cms(const float *x, long T, int K, float *out);
/* cVectorOperation operation=ll1: per-row sum / K (other/vectorOperation.cpp:475-481) */
void osm_or_ll1(const float *x, long T, int K, float *out);

/* static (per-frame) LLDs other than the cepstral chains.  `windowed` selects whether the
 * time-domain component reads the framer level (0) or the windower level (1). */
int  osm_or_spectral_num_out(const osm_or_spectral_cfg *sp);
long osm_or_spectral(const osm_or_frontend *fe, const osm_or_spectral_cfg *sp,
                     const int16_t *pcm, long n_samples, int n_chan, float *out);
/* the same on given magnitudes: mag = [T][nfft/2+1] (the FFT size and bin frequencies of fe's geometry) -> out = [T][num_out];
 * osm_or_spectral is the oracle's own FFT front end followed by this */
long osm_or_spectral_from_mag(const osm_or_frontend *fe, const osm_or_spectral_cfg *sp, const float *mag, long T, float *out);
int  osm_or_energy_num_out(const osm_or_energy_cfg *en);
long osm_or_energy(const osm_or_frontend *fe, const osm_or_energy_cfg *en, int windowed,
                   const int16_t *pcm, long n_samples, int n_chan, float *out);
int  osm_or_pitchacf_num_out(const osm_or_pitchacf_cfg *pc);
/* fftmag -> cAcf (ACF) + cAcf (cepstrum) -> cPitchACF, including its per-utterance smoothing
 * state.  tap_acf / tap_cep (optional): [T x nfft/2] dumps of the two cAcf levels. */
long osm_or_pitchacf(const osm_or_frontend *fe, const osm_or_pitchacf_cfg *pc,
                     const int16_t *pcm, long n_samples, int n_chan, float *out,
                     float *tap_acf, float *tap_cep);
/* the same on given magnitudes [T][nfft/2+1] of one utterance (the smoothing state starts at its frame 0) */
long osm_or_pitchacf_from_mag(const osm_or_frontend *fe, const osm_or_pitchacf_cfg *pc, const float *mag, long T, float *out,
                              float *tap_acf, float *tap_cep);
int  osm_or_mzcr_num_out(const osm_or_mzcr_cfg *mz);
int  osm_or_intensity_num_out(const osm_or_intensity_cfg *in);
/* cIntensity on the framer level: out = [T][num_out] (lldcore/intensity.cpp:86-146) */
long osm_or_intensity(const osm_or_frontend *fe, const osm_or_intensity_cfg *in, int windowed,
                      const int16_t *pcm, long n_samples, int n_chan, float *out);
long osm_or_mzcr(const osm_or_frontend *fe, const osm_or_mzcr_cfg *mz, int windowed,
                 const int16_t *pcm, long n_samples, int n_chan, float *out);

/* cDeltaRegression with the reference's edge/phantom-frame semantics.
 * in: T x K ; out: (T + win) x K.  Returns T + win. */
long osm_or_delta(const float *in, long T, int K, int win, float *out);
long osm_or_delta_variant(const float *in, long T, int K, int W, int relative, int abs_output, int half_wave, float *out);
/* cContourSmoother: in T x K ; out (T + (smaWin-1)/2) x K */
long osm_or_sma(const float *in, long T, int K, int sma_win, int no_zero_sma, float *out);
/* chained variants: `n0` = frames of the input level already written when EOI is raised
 * (tick-order model, see osm_oracle.c); *c0_out = the same quantity for the output level */
long osm_or_delta_chained(const float *in, long T, long n0, int K, int win, float *out, long *c0_out);
long osm_or_sma_chained(const float *in, long T, long n0, int K, int sma_win, int no_zero_sma, float *out, long *c0_out);

#ifdef __cplusplus
}
#endif
#endif
