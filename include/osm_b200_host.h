/*
 * osm_b200_host.h -- host-side front end of libosm_b200.so: reads the reference's own .conf
 * files, resolves the LLD sub-graph into an osm_b200_plan (include/osm_b200.h) and moves
 * utterances between WAV files / PCM buffers and HTK / CSV files / row buffers.
 *
 * It mirrors, for the LLD path only, what SMILExtract / SMILEapi do around the component graph
 * (reference: progsrc/smilextract/SMILExtract.cpp:42-174, progsrc/include/smileapi/SMILEapi.h):
 *
 *   osm_b200_session_open          ~ smile_new + smile_initialize(configFile, options...)
 *                                    (cConfigManager: ini sections, \{include}, \cm[opt(short){dflt}:help],
 *                                     src/core/configManager.cpp:1632-1645,1747-2146; unknown fields are an
 *                                     error like CONF_PARSER_ERR, :2599)
 *   osm_b200_session_extract_files ~ one SMILExtract run per input file (-I wav -O htk -csvoutput csv),
 *                                    all files of the call batched through ONE plan run
 *   osm_b200_session_extract_pcm   ~ smile_extaudiosource_write_data + smile_run + cExternalSink rows
 *   osm_b200_session_num_elements / element_name ~ smile_extsink_get_num_elements / _get_element_name
 *
 * Component types understood in a .conf: the LLD components of include/osm_b200.h (incl. cFullinputMean,
 * cIntensity and cVectorOperation ll1) plus the host
 * edges cDataMemory, cWaveSource / cExternalAudioSource, cHtkSink, cCsvSink, cArffSink (parsed,
 * ARFF output not written) and cExternalSink.  Anything else on the path to the sink's level
 * makes session_open fail with OSM_B200_ERR_UNSUPPORTED; there is no CPU fallback.
 */
#ifndef OSM_B200_HOST_H
#define OSM_B200_HOST_H

#include "osm_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct osm_b200_session osm_b200_session;

/* conf_path: an openSMILE configuration file.  opt_names/opt_values: command line options the
 * config declares through \cm[...] (e.g. "csvoutput" -> "x.csv"; names without the leading '-').
 * output_level: level to extract, NULL = the level the active file sinks read (normally "lld").
 * device: CUDA device, < 0 = description only (parsing / validation without a GPU). */
OSM_B200_API osm_b200_status osm_b200_session_open(const char *conf_path, int32_t n_opts,
                                                   const char *const *opt_names, const char *const *opt_values,
                                                   const char *output_level, int32_t device,
                                                   osm_b200_session **session);
OSM_B200_API void osm_b200_session_close(osm_b200_session *session);

/* number / names of the elements of the output level for the given input format (compiles the
 * plan for that format on first use) */
OSM_B200_API int32_t osm_b200_session_num_elements(osm_b200_session *session, double sample_rate, int32_t n_channels);
OSM_B200_API const char *osm_b200_session_element_name(osm_b200_session *session, int32_t idx);

/* Extract n WAV files (16-bit PCM) in one batch.  htk_paths / csv_paths may be NULL or hold NULL
 * entries; files are written in the reference's formats (src/iocore/htkSink.cpp:90-106,183-206,
 * src/iocore/csvSink.cpp:150-235).  frames_out (optional): rows written per file. */
OSM_B200_API osm_b200_status osm_b200_session_extract_files(osm_b200_session *session, int32_t n,
                                                            const char *const *wav_paths,
                                                            const char *const *htk_paths,
                                                            const char *const *csv_paths,
                                                            int64_t *frames_out);

/* same, additionally writing WEKA ARFF files like cArffSink (src/iocore/arffSink.cpp:225-440) with the options of the
 * configuration's active ARFF sink (relation, instance name, class[] / target[].all from the included targets file) */
OSM_B200_API osm_b200_status osm_b200_session_extract_files_arff(osm_b200_session *session, int32_t n,
                                                                 const char *const *wav_paths,
                                                                 const char *const *htk_paths,
                                                                 const char *const *csv_paths,
                                                                 const char *const *arff_paths,
                                                                 int64_t *frames_out);

/* The sink half of osm_b200_session_extract_files_arff for rows the caller already holds (osm_b200_session_extract_pcm):
 * file i gets rows [frame_offsets[i], frame_offsets[i+1]) of `rows`; n_samples[i] = sample frames of utterance i (time stamps
 * of the rows a window processor appends at the end of input), may be NULL.  Files are formatted on host threads in parallel
 * (OSM_B200_IO_THREADS overrides the count).  Replaces cHtkSink / cCsvSink / cArffSink (src/iocore/htkSink.cpp:120-190,
 * csvSink.cpp:150-235, arffSink.cpp:225-440); needs no device. */
OSM_B200_API osm_b200_status osm_b200_session_write_files(osm_b200_session *session, double sample_rate, int32_t n_channels,
                                                          int32_t n, const int64_t *frame_offsets, const int64_t *n_samples,
                                                          const float *rows, const char *const *htk_paths,
                                                          const char *const *csv_paths, const char *const *arff_paths);

/* the sink formatting options taken from the configuration (active CSV / HTK / ARFF sinks), as text; for bindings
 * and tests.  The string is owned by the library (thread-local). */
OSM_B200_API const char *osm_b200_session_sink_options(osm_b200_session *session);

/* Extract from packed PCM (layout of osm_b200_plan_run_host).  frame_offsets_out: n_utt+1 entries;
 * out: caller buffer of at least max_rows * num_elements floats, or NULL to only get the offsets. */
OSM_B200_API osm_b200_status osm_b200_session_extract_pcm(osm_b200_session *session, const int16_t *pcm,
                                                          const int64_t *utt_offsets, int32_t n_utt,
                                                          double sample_rate, int32_t n_channels,
                                                          int64_t *frame_offsets_out, float *out, int64_t max_rows);

/* Extract from audio already in device memory: a padded batch [n_utt][n_channels][stride] (channel-planar, the layout of a
 * contiguous torch tensor [B, C, L]; mono is n_channels = 1) of int16 (pcm_format = OSM_B200_PCM_S16) or float32
 * (OSM_B200_PCM_F32) samples; lengths: HOST array of n_utt sample-frame counts <= stride (the padding is never read).  int16 samples
 * are those of a 16-bit WAV file; float32 samples are taken as a 32-bit float WAV file holds them, without a full-scale division
 * (e.g. values in [-1, 1]).  The rows are those osm_b200_session_extract_pcm / _extract_files give for the same samples.
 * Same two-call protocol: d_out = NULL only fills frame_offsets_out (which needs a device exactly where extract_pcm's query does);
 * otherwise d_out is a DEVICE buffer of at least max_rows * num_elements floats.  All work is enqueued on `stream` (cudaStream_t,
 * NULL = default stream) and the call never synchronises the device: the host waits on `stream` only for the Viterbi lags of
 * summary configurations with the SHS pitch chain, the cFunctionals row counts, and the cPitchJitter condition flag (reported as
 * OSM_B200_ERR_UNSUPPORTED like extract_pcm).  An LLD configuration without cPitchJitter returns once its work is enqueued.
 * The next call on the session, on any stream, starts after this call's work. */
OSM_B200_API osm_b200_status osm_b200_session_extract_device(osm_b200_session *session, const void *d_pcm, int32_t pcm_format,
                                                             int64_t stride, const int64_t *lengths, int32_t n_utt,
                                                             double sample_rate, int32_t n_channels,
                                                             int64_t *frame_offsets_out, float *d_out, int64_t max_rows,
                                                             void *stream);

/* the component list the session resolved (for diagnostics / tests): number of osm_b200_component
 * entries and a pointer to them (owned by the session, valid until close) */
OSM_B200_API int32_t osm_b200_session_components(osm_b200_session *session, double sample_rate, int32_t n_channels,
                                                 const osm_b200_component **comps, const char **output_level);

/* the plan the session compiled for this input format (owned by the session, valid until close): geometry / row-count /
 * time-stamp queries of include/osm_b200.h for callers that embed the session in a host runtime (plugin/lldBlockB200.cpp) */
OSM_B200_API osm_b200_status osm_b200_session_plan(osm_b200_session *session, double sample_rate, int32_t n_channels,
                                                   osm_b200_plan **plan);

/* message of the last failed osm_b200_session_* call on this thread (falls back to osm_b200_last_error) */
OSM_B200_API const char *osm_b200_host_last_error(void);

/* the file writers on their own (rows -> file), 0 on success.  HTK: 12-byte big-endian header
 * {nSamples, samplePeriod = round(period * 1e7), sampleSize = 4 * n_elements, parmKind} followed by
 * big-endian float32 rows (src/iocore/htkSink.cpp:90-106,183-206).  CSV: cCsvSink's format --
 * header "[name;][frameIndex;][frameTime;]<elements>", rows "['<instance>';][<index>;][<%f time>;]<values>"
 * with integer-valued floats printed as %.0f and the rest as %e, ';' as delimiter
 * (src/iocore/csvSink.cpp:150-235); instance_name NULL = no name column. */
OSM_B200_API int32_t osm_b200_write_htk(const char *path, const float *rows, int64_t n_rows, int32_t n_elements,
                                        double period, int32_t parm_kind);
OSM_B200_API int32_t osm_b200_write_csv(const char *path, const float *rows, int64_t n_rows, int32_t n_elements,
                                        const char *const *names, double period, const char *instance_name,
                                        int32_t frame_index, int32_t frame_time);

/* same, with the time stamp of row r = min(r, n_time_frames - 1) * period (osm_b200_plan_num_time_frames);
 * n_time_frames <= 0: every row has its own time stamp */
OSM_B200_API int32_t osm_b200_write_csv_timed(const char *path, const float *rows, int64_t n_rows, int32_t n_elements,
                                              const char *const *names, double period, const char *instance_name,
                                              int32_t frame_index, int32_t frame_time, int64_t n_time_frames);

/* ---- the value formatting of the sinks on the device (sinks.cu; SURVEY.md 8f-4) ------------------------------------------------
 * Rows a plan run left in HBM become file bytes there; osm_b200_session_extract_files* use these unless OSM_B200_DEVICE_SINKS=0.
 *   osm_b200_device_format_csv : every value of every row as cCsvSink prints it ("%.0f" integer valued, "%e" otherwise,
 *       iocore/csvSink.cpp:216-233), followed by `delim` (newline after the last value of a row), rows at d_text + r * slot_bytes
 *       (slot_bytes >= osm_b200_device_csv_slot_bytes(K)), d_row_len[r] = bytes of row r, d_row_host[r] = 1 when the row holds a value
 *       the device leaves to the host formatter (non-finite, |x| >= 1e15, an undecidable rounding: about 1e-7 of the values)
 *   osm_b200_device_format_rows: the same with always_e = 1 for cArffSink, which prints every value with "%e"
 *       (iocore/arffSink.cpp:300-312; delim ','); integer values >= 1e7 are then left to the host as well
 *   osm_b200_device_pack_htk   : cHtkSink's payload, float32 big endian (iocore/htkSink.cpp:183-206)
 * Asynchronous on `stream` (cudaStream_t); return 0 on success. */
OSM_B200_API int64_t osm_b200_device_csv_slot_bytes(int32_t n_elements);
OSM_B200_API int32_t osm_b200_device_format_csv(const float *d_rows, int64_t n_rows, int32_t n_elements, char delim, char *d_text,
                                                int64_t slot_bytes, int32_t *d_row_len, uint8_t *d_row_host, void *stream);
OSM_B200_API int32_t osm_b200_device_format_rows(const float *d_rows, int64_t n_rows, int32_t n_elements, char delim, int32_t always_e,
                                                 char *d_text, int64_t slot_bytes, int32_t *d_row_len, uint8_t *d_row_host, void *stream);
OSM_B200_API int32_t osm_b200_device_pack_htk(const float *d_rows, int64_t n_values, uint32_t *d_out, void *stream);
/* whole files from device rows (format on the device, copy, write): byte-identical to osm_b200_write_csv_timed / osm_b200_write_htk */
OSM_B200_API int32_t osm_b200_write_csv_device(const char *path, const float *d_rows, int64_t n_rows, int32_t n_elements,
                                               const char *const *names, double period, const char *instance_name,
                                               int32_t frame_index, int32_t frame_time, int64_t n_time_frames);
OSM_B200_API int32_t osm_b200_write_htk_device(const char *path, const float *d_rows, int64_t n_rows, int32_t n_elements, double period,
                                               int32_t parm_kind);

/* cArffSink's file format for rows already in host memory; targets[c] = value of class attribute c for every row
 * ("?" = unknown); append: add rows to an existing file without repeating the header */
OSM_B200_API int32_t osm_b200_write_arff(const char *path, const float *rows, int64_t n_rows, int32_t n_elements,
                                         const char *const *names, double period, const char *relation,
                                         const char *instance_name, int32_t frame_index, int32_t frame_time,
                                         int32_t n_classes, const char *const *class_names, const char *const *class_types,
                                         const char *const *targets, int32_t append, int64_t n_time_frames);

#ifdef __cplusplus
}
#endif
#endif
