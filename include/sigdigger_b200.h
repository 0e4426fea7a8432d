/*
 * sigdigger_b200.h -- C-ABI of libsigdigger_b200.so: the H100-native replacement of the suscan /
 * sigutils analyzer hot path that BatchDrake/SigDigger drives (SURVEY.md section 8).
 *
 * Plain C, plain pointers and sizes, no CUDA or torch types.  Every entry point names the reference
 * interface it replaces (file:line in the SigDigger sources).  `const sdb_complex *` has the layout of
 * SUCOMPLEX (interleaved float32 re, im).  Functions return 0 / a non-negative value on success and -1
 * on failure (SUBOOL-style callers map that to SU_FALSE; message via sdb_last_error(), which plays
 * the role of the sigutils log sink, include/Suscan/Logger.h:55).  There is NO CPU fallback: without a
 * CUDA device sdb_engine_new() fails.
 */
#ifndef SIGDIGGER_B200_H
#define SIGDIGGER_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct { float re, im; } sdb_complex;      /* SUCOMPLEX */
typedef struct sdb_engine sdb_engine_t;             /* one analyzer batch on one GPU */

/* SU_CHANNEL_DETECTOR_WINDOW_* (include/Suscan/AnalyzerParams.h:37-43) */
enum { SDB_WINDOW_NONE = 0, SDB_WINDOW_HAMMING, SDB_WINDOW_HANN, SDB_WINDOW_FLAT_TOP,
       SDB_WINDOW_BLACKMANN_HARRIS };

/* inspector classes: "psk" / "fsk" / "ask" (Default/Inspection/InspToolWidget.cpp:932,938,944),
 * "audio" (Default/Audio/AudioProcessor.cpp:153), "raw" (InspToolWidget.cpp:612), "power" (InspToolWidget.cpp:950,
 * the RMS tool: one mean channel power (re, 0) per power_integrate_samples channel samples, SPEC PW in
 * oracle/SPEC_PW.md) */
enum { SDB_INSP_PSK = 0, SDB_INSP_FSK = 1, SDB_INSP_ASK = 2, SDB_INSP_AUDIO = 3, SDB_INSP_RAW = 4, SDB_INSP_POWER = 5 };

/* SigDigger's AudioDemod enum + 1 as it goes on the wire (include/SigDiggerHelpers.h:39-45,
 * Default/Audio/AudioProcessor.cpp:261) */
enum { SDB_AUDIO_DISABLED = 0, SDB_AUDIO_AM, SDB_AUDIO_FM, SDB_AUDIO_USB, SDB_AUDIO_LSB };

#define SDB_FLAG_PSD_SHIFT_DB 1u  /* fold the GUI's fft-shift + SU_POWER_DB pass
                                     (Suscan/Messages/PSDMessage.cpp:32-38) into the PSD kernel */
#define SDB_FLAG_IQ_REVERSE   2u  /* suscan_analyzer_set_iq_reverse (Suscan/Analyzer.cpp:238-244): the source delivers
                                     (Q, I); swapped inside the first load of the path, any sample format */
#define SDB_FLAG_DC_REMOVE    4u  /* suscan_analyzer_set_dc_remove (Suscan/Analyzer.cpp:229-236): block-wise single-pole
                                     DC estimate subtracted from every sample before the PSD and the channeliser
                                     see it (SPEC R: c += alpha (mean(block) - c), alpha = 1 - exp(-n / (fs 0.1 s)));
                                     one extra pass that also converts native formats to float32 */

/* Replaces struct suscan_analyzer_params.detector_params.{window_size, window}
 * (Suscan/AnalyzerParams.cpp:56-66) + the specttuner's sigutils_specttuner_params.window_size
 * (Tasks/LPFTask.cpp:52). n_streams > 1 batches independent sources through the same plan. */
typedef struct {
  uint32_t n_streams;
  uint32_t psd_size;        /* power of two, 512 .. 2^20 (Default/FFT/FFTWidget.cpp:350-351); 0 = no PSD */
  int32_t  psd_window;
  uint32_t st_window_size;  /* channeliser FFT size; 0 = psd_size */
  uint32_t max_feed;        /* largest per-stream feed, samples */
  int32_t  device;          /* CUDA ordinal */
  uint32_t flags;
  int32_t  input_format;    /* SDB_FORMAT_*: layout of the IQ the feed calls receive */
  /* Frame-averaged main PSD (SPEC A, oracle/SPEC_A.md): 0 or 1 = off; A in [2, SDB_PSD_AVERAGE_MAX] emits the mean of
   * every A consecutive frames of each stream (the partial group carries across feeds; sdb_engine_read_psd_average).
   * With averaging on, SDB_FLAG_PSD_SHIFT_DB applies to the means only and the per-frame PSD stays linear. */
  uint32_t psd_average;
  /* Peak detectors of the main PSD (SPEC PK, oracle/SPEC_PK.md): 0 or 1 = off; P in [2, SDB_PSD_PEAK_MAX] emits the
   * per-bin maximum and minimum of every P consecutive frames of each stream (the partial group carries across feeds;
   * sdb_engine_read_psd_peak).  With peak detection on, SDB_FLAG_PSD_SHIFT_DB applies to the extremes (and to the means
   * when averaging is on as well) and the per-frame PSD stays linear. */
  uint32_t psd_peak;
} sdb_engine_params;
#define SDB_PSD_AVERAGE_MAX 65536u
#define SDB_PSD_PEAK_MAX 65536u

/* SUSCAN_SOURCE_FORMAT_RAW_{FLOAT32, UNSIGNED8, SIGNED8, SIGNED16} (Default/SourceConfig/FileSourcePage.cpp:80-104):
 * interleaved I,Q pairs; 8/16-bit samples are converted inside the first load of the path (u8: (v-128)/128,
 * s8: v/128, s16: v/32768), so an 8-bit source moves 4x fewer bytes over PCIe and HBM than float32. */
enum { SDB_FORMAT_FLOAT32 = 0, SDB_FORMAT_UNSIGNED8 = 1, SDB_FORMAT_SIGNED8 = 2, SDB_FORMAT_SIGNED16 = 3 };

/* Replaces struct sigutils_specttuner_channel_params {f0, bw, guard, precise}
 * (Tasks/LPFTask.cpp:63-67); angular units (rad/sample). */
typedef struct {
  float   f0, bw, guard;
  int32_t precise;
} sdb_channel_params;

typedef struct {
  uint32_t center, size, width;
  float    decimation;      /* st_window_size / size */
} sdb_channel_info;

/* Typed image of the inspector's suscan_config_t key/value bag.  Field <-> key:
 * agc.enabled, agc.gain (GainControl.cpp:51-60); afc.costas-order, afc.bits-per-symbol, afc.loop-bw,
 * afc.offset (AfcControl.cpp:54-83); fsk.bits-per-symbol, fsk.phase, fsk.quad-demod
 * (ToneControl.cpp:59-81); ask.bits-per-symbol, ask.use-pll, ask.loop-bw, ask.offset, ask.channel
 * (AskControl.cpp:53-77); mf.type, mf.roll-off (MfControl.cpp:56-78); clock.type, clock.baud,
 * clock.gain, clock.phase, clock.running (ClockRecovery.cpp:59-93); equalizer.type, equalizer.rate,
 * equalizer.locked (EqualizerControl.cpp:47-75); audio.* and agc.ts
 * (Default/Audio/AudioProcessor.cpp:257-265).  All under Default/GenericInspector/InspectorCtl/, except
 * power.integrate-samples (Default/RMSInspector/RMSInspector.cpp:404-416, 438-439). */
typedef struct {
  int32_t  insp_class;
  float    fs;              /* filled by the engine: equivalent channel rate in Hz (= samp_rate / decimation) */
  int32_t  agc_enabled;
  float    agc_gain_db;
  uint32_t costas_order;    /* 0 manual, 1 BPSK, 2 QPSK, 3 8PSK */
  uint32_t bits_per_symbol;
  float    loop_bw;         /* Hz */
  float    offset;          /* Hz */
  float    fsk_phase;
  int32_t  fsk_quad_demod;
  int32_t  ask_use_pll;
  uint32_t ask_channel;
  uint32_t mf_type;         /* SUSCAN_INSPECTOR_MATCHED_FILTER_{BYPASS=0, MANUAL=1} */
  float    mf_rolloff;
  uint32_t clock_type;      /* SUSCAN_INSPECTOR_BAUDRATE_CONTROL_{MANUAL=0, GARDNER=1} */
  float    baud, clock_gain, clock_phase;
  int32_t  clock_running;
  float    audio_cutoff, audio_volume, audio_squelch_level, agc_ts;
  uint32_t audio_sample_rate, audio_demod;
  int32_t  audio_squelch;
  uint32_t eq_type;         /* equalizer.type: SUSCAN_INSPECTOR_EQUALIZER_{BYPASS=0, CMA=1} (EqualizerControl.cpp:56-75) */
  float    eq_rate;         /* equalizer.rate */
  int32_t  eq_locked;       /* equalizer.locked */
  /* power.integrate-samples: channel samples per mean of the "power" class (0 is read as 1); the default is
   * max(1, llround(0.1 fs)), a tenth of a second of channel samples */
  uint64_t power_integrate_samples;
} sdb_inspector_config;

const char *sdb_last_error(void);
int         sdb_device_count(void);

/* suscan_analyzer_new / suscan_analyzer_destroy (Suscan/Analyzer.cpp:608, :636) */
sdb_engine_t *sdb_engine_new(const sdb_engine_params *params, double samp_rate);
void          sdb_engine_destroy(sdb_engine_t *e);

/* su_specttuner_open_channel (Tasks/LPFTask.cpp:69) / suscan_analyzer_open_ex_async
 * (Suscan/Analyzer.cpp:459-484).  Returns the channel handle (SUHANDLE). */
int sdb_engine_open_channel(sdb_engine_t *e, const sdb_channel_params *p, sdb_channel_info *info);
/* the same geometry without an engine (su_specttuner_open_channel reports it before any data flows) */
int sdb_channel_geometry(uint32_t window_size, const sdb_channel_params *p, sdb_channel_info *info);
/* suscan_analyzer_set_inspector_config_async (Suscan/Analyzer.cpp:486-495) */
int sdb_engine_set_inspector(sdb_engine_t *e, int handle, const sdb_inspector_config *cfg);
/* fills cfg with the class defaults the OPEN message would carry
 * (Suscan/Messages/InspectorMessage.cpp:28-71 `config`) */
int sdb_inspector_config_default(sdb_inspector_config *cfg, int insp_class, float fs);
/* freezes the channel plan and allocates device buffers; required before the first feed */
int sdb_engine_commit(sdb_engine_t *e);
/* Live re-plan: `dst` (committed, not yet fed) takes over the running state of `src` (same streams / window /
 * device): input history, the partial group of the frame-averaged PSD and of the peak detectors, each when psd_size,
 * psd_window and its group size (psd_average, psd_peak) match (otherwise `dst` starts an empty group), and per channel
 * with identical parameters the cross-fade tail, the LO phase
 * and -- if the inspector class and the sizes of its state lines are unchanged -- the loop state of every chain; a power
 * inspector that stays one with the same power_integrate_samples keeps its partial group (SPEC PW).  This is how an
 * analyzer opens, closes, retunes or reconfigures ONE inspector at a block boundary while the others keep running
 * (suscan_analyzer_open_ex_async / close_async / set_inspector_config_async / set_inspector_freq_overridable,
 * Suscan/Analyzer.cpp:459-526).  `src` is synchronised and left intact.  The channel detector's state (SPEC K) is not
 * carried: `dst`'s detector starts afresh, and so does its channel tracking (oracle/SPEC_KT.md), with track ids
 * beginning again at 1. */
int sdb_engine_migrate(sdb_engine_t *dst, sdb_engine_t *src);
/* the same with the caller saying which old channel each new one continues: old_of_new[new handle] = old handle or
 * -1 (a retuned inspector keeps its loops even though its channel moved; only the cross-fade tail restarts) */
int sdb_engine_migrate_map(sdb_engine_t *dst, sdb_engine_t *src, const int32_t *old_of_new, size_t n);
int sdb_engine_same_geometry(const sdb_engine_t *a, const sdb_engine_t *b);   /* 1: migrate would accept the pair */

/* One pass of the hot path over `n` new samples of every stream (the body of suscan's source-worker
 * loop, SURVEY.md 3.2 HOT LOOP #1 + 3.3 HOT LOOP #2).  n must be a multiple of the PSD size and of
 * half the channeliser window.  x: stream s starts at x + s * stream_stride.
 *   _device: x is a device pointer (IQ already resident in HBM); asynchronous.
 *   _host:   x is host memory (pinned for full speed); copies H2D inside the call; asynchronous. */
int sdb_engine_feed_device(sdb_engine_t *e, const sdb_complex *x, size_t stream_stride, size_t n);
int sdb_engine_feed_host(sdb_engine_t *e, const sdb_complex *x, size_t stream_stride, size_t n);
int sdb_engine_sync(sdb_engine_t *e);
/* The inspector kernels run on a second CUDA stream so that the next feed's FFT kernels overlap them.
 * sdb_engine_join() makes work queued afterwards on the engine stream wait for all of them (call it
 * before recording a CUDA event that must cover whole feeds); sdb_engine_sync() joins and blocks. */
int sdb_engine_join(sdb_engine_t *e);

/* Results of the last feed.  PSD = payload of suscan_analyzer_psd_msg (psd_size, psd_data;
 * Suscan/Messages/PSDMessage.cpp:26-39): [stream][frame][psd_size] float32, linear power, DC at 0
 * unless SDB_FLAG_PSD_SHIFT_DB. */
size_t       sdb_engine_psd_frames(const sdb_engine_t *e);
const float *sdb_engine_psd_device(const sdb_engine_t *e);
int          sdb_engine_read_psd(sdb_engine_t *e, float *dst, size_t cap_floats);
/* Frame-averaged PSD of the last feed (sdb_engine_params.psd_average >= 2): [stream][mean][psd_size] float32, the means
 * of the groups the feed completed, linear with DC at 0 unless SDB_FLAG_PSD_SHIFT_DB.  _frames: means per stream (0
 * when averaging is off); _device: the engine's buffer, valid until the feed after next; read: blocking copy, fenced
 * like sdb_engine_read_psd. */
size_t       sdb_engine_psd_average_frames(const sdb_engine_t *e);
const float *sdb_engine_psd_average_device(const sdb_engine_t *e);
int          sdb_engine_read_psd_average(sdb_engine_t *e, float *dst, size_t cap_floats);
/* Peak detectors of the last feed (sdb_engine_params.psd_peak >= 2): two [stream][group][psd_size] float32 arrays, the
 * per-bin maxima and minima of the groups the feed completed, linear with DC at 0 unless SDB_FLAG_PSD_SHIFT_DB.
 * _groups: groups per stream (0 when peak detection is off); _device: the engine's buffer of the maxima (which = 0) or
 * the minima (which = 1), valid until the feed after next; read: blocking copy of both, fenced like sdb_engine_read_psd,
 * either destination may be NULL and cap_floats applies to each. */
size_t       sdb_engine_psd_peak_groups(const sdb_engine_t *e);
const float *sdb_engine_psd_peak_device(const sdb_engine_t *e, int which);
int          sdb_engine_read_psd_peak(sdb_engine_t *e, float *max_dst, float *min_dst, size_t cap_floats);
/* channel-rate output of the channeliser (what on_data delivers, Tasks/LPFTask.cpp:28-42) */
long         sdb_engine_read_channel(sdb_engine_t *e, uint32_t stream, int handle, sdb_complex *dst,
                                     size_t cap);
/* inspector output: suscan_analyzer_sample_batch_msg.samples
 * (include/Suscan/Messages/SamplesMessage.h:33-59) + the GUI's Decider output
 * (Default/GenericInspector/InspectorUI.cpp:836-846).  Either dst may be NULL. */
long         sdb_engine_read_symbols(sdb_engine_t *e, uint32_t stream, int handle, sdb_complex *soft,
                                     uint8_t *hard, size_t cap);
/* all streams, all channels at once: counts[S*K], soft/hard laid out [S][K][cap] */
int          sdb_engine_read_all_symbols(sdb_engine_t *e, uint32_t *counts, sdb_complex *soft,
                                         uint8_t *hard, size_t cap);
/* Asynchronous reads: queued on the engine's D2H stream behind the kernels that produce the data, so the
 * next feed can be submitted at once (H2D of feed i+1, kernels of feed i and D2H of feed i-1 overlap;
 * results are double-buffered by feed parity).  Destinations should be pinned host memory and stay valid
 * until sdb_engine_sync(). */
int          sdb_engine_read_psd_async(sdb_engine_t *e, float *dst, size_t cap_floats);
int          sdb_engine_read_all_symbols_async(sdb_engine_t *e, uint32_t *counts, sdb_complex *soft,
                                               uint8_t *hard, size_t cap);
/* Packed read of the last feed's symbols (the batch counterpart of suscan's per-inspector SAMPLES messages,
 * Suscan/Messages/SamplesMessage.cpp): chain c = stream * n_channels + channel has counts[c] symbols at
 * soft[offsets[c] ...] / hard[offsets[c] ...]; every start is a multiple of 16 symbols (the gap is zero-filled) and
 * offsets[chains] is the total extent.  A chain whose row would pass cap_total is skipped (offsets[chains] >
 * cap_total tells).  The GPU writes soft / hard directly: they must be 16-byte-aligned PINNED host memory
 * (cudaHostAlloc / cudaHostRegister) or device memory, anything else is refused; counts and offsets (chains and
 * chains + 1 entries) are ordinary async copies.  PCIe carries ~9 bytes per symbol instead of 9 bytes per channel
 * sample. */
int          sdb_engine_read_symbols_packed_async(sdb_engine_t *e, uint32_t *counts, uint64_t *offsets,
                                                  sdb_complex *soft, uint8_t *hard, size_t cap_total);
int          sdb_engine_read_symbols_packed(sdb_engine_t *e, uint32_t *counts, uint64_t *offsets,
                                            sdb_complex *soft, uint8_t *hard, size_t cap_total);
/* ---- inspector spectrum sources and parameter estimators (SURVEY.md 8(f) rank 1; SPEC.md section U) ----
 * suscan_analyzer_inspector_set_spectrum_async(analyzer, handle, spectsrc_id, req_id) (Suscan/Analyzer.cpp:539-548)
 * and suscan_analyzer_inspector_estimator_cmd_async(analyzer, handle, estimator_id, enabled, req_id)
 * (Suscan/Analyzer.cpp:550-565).  Index 0 of the GUI's source combo is "none"; the OPEN message lists the
 * sources / estimators below in this order (Suscan/Messages/InspectorMessage.cpp:40-61).  Every feed that
 * produced more than `size` channel-rate samples emits one spectrum of the last `size` samples (linear power,
 * DC at index 0: the GUI converts to dB and swaps halves itself, GenericInspector.cpp:232-250) and one value
 * per enabled estimator.  Both calls must precede sdb_engine_commit(). */
enum { SDB_SPECTSRC_NONE = 0, SDB_SPECTSRC_PSD, SDB_SPECTSRC_CYCLO, SDB_SPECTSRC_FMSPECT, SDB_SPECTSRC_TIMEDIFF,
       SDB_SPECTSRC_ABSTIMEDIFF, SDB_SPECTSRC_EXP_2, SDB_SPECTSRC_EXP_4, SDB_SPECTSRC_EXP_8, SDB_SPECTSRC_FAC,
       SDB_SPECTSRC_COUNT };
enum { SDB_ESTIMATOR_BAUD_FAC = 0, SDB_ESTIMATOR_BAUD_NONLINEAR = 1, SDB_ESTIMATOR_COUNT };
/* name / description strings of the registries (suscan_spectsrc_class_lookup, suscan_estimator_class_lookup) */
const char *sdb_spectsrc_name(int spectsrc_id);
const char *sdb_estimator_name(int estimator_id);
int sdb_engine_set_spectrum_source(sdb_engine_t *e, int handle, int spectsrc_id, uint32_t size /* 64..4096, 2^k */);
int sdb_engine_set_estimator(sdb_engine_t *e, int handle, int estimator_id, int enabled);
/* latest spectra of one channel, all streams: out[n_streams][size] (FAC fills size/2), sizes[n_streams] = floats
 * emitted per stream (0 = nothing this feed).  Waits for the feed's kernels. */
int sdb_engine_read_spectrum(sdb_engine_t *e, int handle, float *out, uint32_t *sizes);
/* latest estimates of one channel, all streams: values[n_streams], valid[n_streams] */
int sdb_engine_read_estimate(sdb_engine_t *e, int handle, int estimator_id, float *values, int32_t *valid);
/* Scheduled spectra and estimates (oracle/SPEC_US.md): with an interval I >= 1, the channel emits at every t_j = j I
 * channel samples since it started (from t_j >= size + 1 on) over the frame c[t_j - size - 1 .. t_j - 1], carried
 * across feeds, so that narrow channels emit and wide ones emit at a fixed rate whatever the feed size.  I = 0 (the
 * default) keeps one emission per feed as above.  Call before sdb_engine_commit() on a channel with a spectrum
 * source or an estimator.  A feed emits at most ceil(max_feed channel samples / I) <= SDB_SPECTRUM_EMITS_MAX times;
 * commit refuses a larger count.  The ring of the last size + 1 samples costs n_streams (size + 1) 8 bytes. */
#define SDB_SPECTRUM_EMITS_MAX 256
#define SDB_SPECTRUM_INTERVAL_MAX (1ull << 62)   /* larger intervals are refused */
int  sdb_engine_set_spectrum_interval(sdb_engine_t *e, int handle, uint64_t interval);
/* every emission of the last feed, all streams: out[n_streams][cap][out_size] (out_size = size, or size / 2 for
 * "fac"), ends[cap] = t_j of each emission (the same in every stream).  Returns the emission count (<= cap; the same
 * for every stream), -1 on error.  On a scheduled channel sdb_engine_read_spectrum / _read_estimate give the last
 * emission of the feed, or size 0 / invalid when it had none. */
long sdb_engine_read_spectra(sdb_engine_t *e, int handle, float *out, uint64_t *ends, size_t cap);
/* values[n_streams][cap], valid[n_streams][cap] of every emission of the last feed; returns the emission count */
long sdb_engine_read_estimates(sdb_engine_t *e, int handle, int estimator_id, float *values, int32_t *valid, size_t cap);

/* ---- the inspector's FAC tab (Default/GenericInspector/FACTab.cpp; oracle/SPEC_FC.md) ----
 * The averaged, peak-marked autocorrelation of a psk / fsk / ask inspector's soft symbols, per stream.  Symbols fill
 * blocks of `size` = 2^9 .. 2^19 (the tab's 65536 by default) across feeds; each completed block gives
 * v[l] = |autocorrelation| at lag l < size / 2 (unnormalised), and fac[l] += alpha (v[l] / max - fac[l]) with max the
 * running maximum of v over the lag window [lag_lo, lag_hi) since the channel started (lag_lo = lag_hi = 0: [0, size/2),
 * the tab's default view).  alpha = 1 - averaging slider / 100.  Per feed, over the blocks it completed: the first
 * lag of the largest v in the window (peak_lag), sigmas = that v / sqrt(mean v^2 of the window's values that set no
 * running maximum), and marker = sigmas > sigma (the tab's peak detector; 5 by default).  sigmas and marker are 0
 * when the feed completed no block, no value counted or the peak is infinite.  An all-zero input gives max = 0 and a
 * NaN fac, as in the tab.
 * set_fac: before commit; NULL turns the FAC off.  Device memory: n_streams (8 L + 2 L + slots 4 L, plus slots 8 L
 * for L >= 8192) bytes per FAC channel, slots = the blocks one feed can complete, (L - 1 + n) / L with n the channel
 * samples of a max_feed feed.
 * read_fac: fac[n_streams][size / 2] and st[n_streams] after the latest feed (waits for it); either may be NULL.
 * _fac_device: the engine's fac of stream 0 of the channel (the streams follow, size / 2 floats apart), or NULL.
 * Migration keeps a channel's block, fill, max, min and fac when it continues with the same class, size and channel
 * rate (alpha, the window and sigma may change); anything else restarts as after a resize. */
typedef struct { uint32_t size; float alpha; uint32_t lag_lo, lag_hi; double sigma; } sdb_fac_params;
typedef struct { uint32_t blocks, peak_lag; float max, min, sigmas; int32_t marker; } sdb_fac_status;
int  sdb_engine_set_fac(sdb_engine_t *e, int handle, const sdb_fac_params *p);
int  sdb_engine_read_fac(sdb_engine_t *e, int handle, float *fac, sdb_fac_status *st);
const float *sdb_engine_fac_device(const sdb_engine_t *e, int handle);

/* ---- the inspector's SNR meter (InspectorUI::feed, Default/GenericInspector/InspectorUI.cpp:807-833; Misc/
 * SNREstimator.cpp; oracle/SPEC_SN.md) ----
 * Per stream of a psk / fsk / ask inspector: every feed's soft symbols (what SAMPLES carries) are binned into a
 * decision-space histogram h[bins] (the argument on [-pi, pi] for psk and fsk, the modulus on [0, 1) for ask, where
 * values at or above 1 are not counted), and every feed that brought at least one symbol runs one gradient step of the
 * comb fit (SPEC Y.7) with K = 2^bits_per_symbol (0 read as 1) Gaussians of width sigma: sigma -= alpha delta.
 * SNR = 1 / (K sigma).  When a bin reaches 2^31, every bin is halved.
 * set_snr: before commit; NULL turns the meter off.  bins 16 .. 1024 (the GUI's 256), sigma and alpha finite and > 0
 * (the GUI's toggle: sigma 1, alpha 1 / K).  Device memory: n_streams (8 bins + 32) bytes per channel.
 * reset_snr: between feeds, sets sigma of every stream of the channel from the next feed on; h is kept (the GUI's
 * reset button).
 * read_snr: hist[n_streams][bins], model[n_streams][bins] (the fitted comb, normalised to a maximum of 1) and
 * st[n_streams] after the latest feed (waits for it); any of them may be NULL.
 * Migration (SPEC SN.4): a channel that keeps its inspector class and bins keeps h, the model, sigma and the step count
 * when its inspector configuration is unchanged; any other configuration clears h and keeps sigma, which restarts at
 * 1/8 when bits_per_symbol changed.  Anything else starts afresh.  alpha always comes from the new parameters. */
typedef struct { uint32_t bins; float sigma, alpha; } sdb_snr_params;
/* counted = sum of h; steps = gradient steps so far; stepped = 1 when the latest feed ran one; delta = its gradient */
typedef struct { uint64_t counted; uint32_t steps, stepped; float sigma, snr, delta; } sdb_snr_status;
int  sdb_engine_set_snr(sdb_engine_t *e, int handle, const sdb_snr_params *p);
int  sdb_engine_reset_snr(sdb_engine_t *e, int handle, float sigma);
int  sdb_engine_read_snr(sdb_engine_t *e, int handle, uint32_t *hist, float *model, sdb_snr_status *st);

/* ---- channel detector on the main PSD (SURVEY.md 8(f) rank 3; SPEC.md section K) ----
 * struct suscan_analyzer_params.detector_params.{alpha, beta, gamma, snr} + channel_update_int
 * (Suscan/AnalyzerParams.cpp:27-66) -> SUSCAN_ANALYZER_MESSAGE_TYPE_CHANNEL lists of struct sigutils_channel
 * (Suscan/Messages/ChannelMessage.cpp:25-70; include/Suscan/Channel.h:26-32).  alpha = spectrum averaging,
 * gamma = noise-floor averaging, snr = linear power ratio over the floor; beta (signal-level averaging) is used only
 * by channel tracking (sdb_engine_set_channel_tracking): the detector reports levels per update.  One update per
 * feed. */
typedef struct {
  double   fc, f_lo, f_hi, bw;      /* Hz (sigutils_channel.fc / f_lo / f_hi / bw) */
  float    snr, S0, N0;             /* linear power: peak averaged level, noise floor, S0 / N0 */
  uint32_t bin_lo, bin_hi;          /* [lo, hi) in ascending-frequency bin order */
} sdb_detected_channel;
/* engine-integrated: enable before sdb_engine_commit(); needs a linear per-frame PSD (no SDB_FLAG_PSD_SHIFT_DB, unless
 * psd_average >= 2 or psd_peak >= 2 confines the flag to the group outputs) */
int  sdb_engine_set_channel_detector(sdb_engine_t *e, float alpha, float beta, float gamma, float snr,
                                     uint32_t min_bins);
/* channels of one stream after the latest feed (ascending frequency); *total = channels found before the
 * 256-entry cap.  center_freq shifts the reported frequencies (source tuner frequency, sigutils_channel.ft). */
long sdb_engine_read_channels(sdb_engine_t *e, uint32_t stream, double center_freq, sdb_detected_channel *out,
                              size_t cap, uint32_t *total);
/* the lists of all streams in one read: centers[n_streams] (host), out[n_streams][cap], counts[n_streams] */
int  sdb_engine_read_all_channels(sdb_engine_t *e, const double *centers, sdb_detected_channel *out, size_t cap,
                                  uint32_t *counts);
/* ---- channel tracking across detector updates (oracle/SPEC_KT.md) ----
 * Follows each detected channel from one update to the next: a detection continues the live track it overlaps most,
 * whose peak level S0 is then smoothed by the detector's beta; a track no detection continues is kept for `hold`
 * further updates (its range and S0 unchanged) and then removed; a detection no track continues opens a new track.
 * At most 256 tracks per stream.  Enable with sdb_engine_set_channel_tracking() before sdb_engine_commit(), after
 * sdb_engine_set_channel_detector(); beta must then be in (0, 1] (checked at commit).  Without it the engine issues
 * the same launches as before and beta stays unused. */
#define SDB_CHTRACK_HOLD_MAX 65535u
typedef struct {
  double   fc, f_lo, f_hi, bw;      /* Hz, as sdb_detected_channel, over the track's latest range */
  float    snr, S0, N0;             /* beta-smoothed peak level, the detector's current floor, S0 / N0 */
  uint32_t bin_lo, bin_hi;          /* [lo, hi) in ascending-frequency bin order */
  uint32_t id;                      /* per stream, from 1 in order of opening */
  uint32_t age, present, misses;    /* updates since opening, updates detected (sigutils_channel.age / .present),
                                       updates missed in a row (> 0: in hold) */
} sdb_tracked_channel;
int  sdb_engine_set_channel_tracking(sdb_engine_t *e, uint32_t hold);
/* live tracks of one stream after the latest feed, ascending (bin_lo, id); *total = live tracks before the cap,
 * *dropped = detections not tracked because 256 tracks were live, since commit (either pointer may be NULL) */
long sdb_engine_read_tracked_channels(sdb_engine_t *e, uint32_t stream, double center_freq, sdb_tracked_channel *out,
                                      size_t cap, uint32_t *total, uint64_t *dropped);
/* all streams in one read: centers[n_streams] (host), out[n_streams][cap], counts[n_streams], dropped[n_streams]
 * (may be NULL) */
int  sdb_engine_read_all_tracked_channels(sdb_engine_t *e, const double *centers, sdb_tracked_channel *out, size_t cap,
                                          uint32_t *counts, uint64_t *dropped);
/* stand-alone detector on any device-resident linear PSD (e.g. the stitched SpectrumView of the panoramic
 * scanner, BASELINE config 5 "per-GPU channel detector"): psd_dev[stream][frame][n_bins], DC at index 0 */
typedef struct sdb_chdet sdb_chdet_t;
sdb_chdet_t *sdb_chdet_new(int device, uint32_t n_bins, uint32_t n_streams, float alpha, float gamma, float snr,
                           uint32_t min_bins);
void sdb_chdet_destroy(sdb_chdet_t *d);
int  sdb_chdet_feed_device(sdb_chdet_t *d, const float *psd_dev, uint32_t frames, size_t stream_stride);
long sdb_chdet_read(sdb_chdet_t *d, uint32_t stream, double samp_rate, double center_freq,
                    sdb_detected_channel *out, size_t cap, uint32_t *total);
int  sdb_chdet_read_all(sdb_chdet_t *d, double samp_rate, const double *centers, sdb_detected_channel *out, size_t cap,
                        uint32_t *counts);

/* device-side views for zero-copy consumers / benchmarks */
const uint32_t *sdb_engine_symbol_counts_device(const sdb_engine_t *e);
size_t          sdb_engine_symbol_capacity(const sdb_engine_t *e);

/* CUDA stream the engine launches on (cudaStream_t as void*), for event timing by the caller */
void    *sdb_engine_stream(const sdb_engine_t *e);
/* kernels launched since engine creation (for bench.py's gpu_launches) */
uint64_t sdb_engine_launch_count(const sdb_engine_t *e);
/* average device time (ms) of the named kernel family over the launches since the last reset, measured
 * with CUDA events on the engine stream; families: "fft_cols", "fft_rows_psd", "fft_rows_chan",
 * "chan_ifft", "inspector", "psd_average", "power", "psd_peak", "spectsrc_sched".  A 65536-point plan's fused forward transform counts as
 * "fft_cols"; its "fft_rows_psd" / "fft_rows_chan" stay at zero launches; "psd_average" (the group means) records none
 * while averaging is off, "power" (the power inspectors' integration) none while no channel has a power inspector,
 * "psd_peak" (the group extremes) none while peak detection is off, "spectsrc_sched" (the scheduled spectra: frame
 * gather, transforms and ring update) none in a feed that neither emits nor keeps samples, "fac" (the FAC tab's
 * launches, sdb_engine_set_fac) none while no channel has the FAC on, "snr" (the SNR meter's k_snr, sdb_engine_set_snr)
 * none while no channel has the meter on */
int      sdb_engine_kernel_time(sdb_engine_t *e, const char *family, double *avg_ms, uint64_t *launches);
void     sdb_engine_timing(sdb_engine_t *e, int enable);
/* inspector-kernel stage balance since the last reset: out[0..3] = busy SM cycles of the gain / carrier /
 * filter / clock stage warps summed over CTAs, out[4] = chunk-samples processed (profiling aid) */
int      sdb_debug_stage_cycles(uint64_t out[8], int reset);
/* instrumented twin only (zeros otherwise), per inspector class c = 0..4 (SDB_INSP_*): out[c] = sum of CTA lifetimes
 * in SM cycles, out[5 + c] = CTAs, out[10 + c] = longest CTA, out[15 + c] = latest CTA end and out[20] = earliest CTA
 * start (ns, global timer); out[24 + 8 c + r] = busy cycles of role r (0 track, 1 carrier, 2 filter, 3 clock,
 * 5 pre, 6 post) and [24 + 8 c + 4] = chunk samples, in CTAs of class c */
int      sdb_debug_cta_cycles(uint64_t out[64], int reset);

/* ------------------------------------------------------------------------------------------------
 * Offline Tasks/ primitives over a whole capture buffer (host pointers; one GPU chain each; the
 * batched forms take `batch` independent buffers of n samples, contiguous).
 * ---------------------------------------------------------------------------------------------- */
/* CarrierXlator: su_ncqo_init(-relFreq), su_ncqo_set_phase(-phase), dst = src * su_ncqo_read()
 * (Tasks/CarrierXlator.cpp:36-37,57-60) */
int sdb_task_carrier_xlate(const sdb_complex *src, sdb_complex *dst, size_t n, size_t batch,
                           float rel_freq, float phase);
/* QuadDemodTask (Tasks/QuadDemodTask.cpp:44-60) */
int sdb_task_quad_demod(const sdb_complex *src, sdb_complex *dst, size_t n, size_t batch);
/* CostasRecoveryTask: su_costas_init(kind, 0, 1/tau, 3, loopbw) + su_costas_feed loop
 * (Tasks/CostasRecoveryTask.cpp:36-41,58-61) */
int sdb_task_costas(const sdb_complex *src, sdb_complex *dst, size_t n, size_t batch, int kind,
                    float tau, float loop_bw);
/* PLLSyncTask: su_pll_init(0, bw) + su_pll_track loop (Tasks/PLLSyncTask.cpp:36,53-56) */
int sdb_task_pll(const sdb_complex *src, sdb_complex *dst, size_t n, size_t batch, float bw);
/* Bulk twins of the per-sample su_costas_feed / su_pll_track of the sigutils-named shim (include/sigutils/pll.h): one
 * buffer, the loop continues from the caller's state and the final state is written back, so consecutive work()
 * blocks of a Tasks/ object (Tasks/CostasRecoveryTask.cpp:49-61) chain exactly.  k / s: the configuration and state
 * members of su_costas_t (sizes checked); state[2] = {phi, omega}. */
int sdb_task_costas_state(const sdb_complex *src, sdb_complex *dst, size_t n, const void *k, size_t k_bytes,
                          void *s, size_t s_bytes);
int sdb_task_pll_state(const sdb_complex *src, sdb_complex *dst, size_t n, float alpha, float beta, float state[2]);
/* AGCTask: su_agc_init with tau fractions + su_agc_feed loop (Tasks/AGCTask.cpp:41-53,70-73) */
int sdb_task_agc(const sdb_complex *src, sdb_complex *dst, size_t n, size_t batch, float tau);
/* LPFTask: su_specttuner low-pass with guard = 2 pi / bw, output length == input length
 * (Tasks/LPFTask.cpp:52-69,83-87,104-107) */
int sdb_task_lpf(const sdb_complex *src, sdb_complex *dst, size_t n, size_t batch, float bw);

/* Decision spaces of the TimeWindow samplers (enum SamplingSpace, include/SamplingProperties.h:27-31) */
enum { SDB_SPACE_AMPLITUDE = 0, SDB_SPACE_PHASE = 1, SDB_SPACE_FREQUENCY = 2 };
/* DelayedConjTask: dst[p] = 0 for p < delay, else x[p] conj(x[p-delay]) / (|x[p-delay]| + 1e-3)
 * (Tasks/DelayedConjTask.cpp:58-100); delay == 0 is an error as in the constructor (:36-37) */
int  sdb_task_delayed_conj(const sdb_complex *src, sdb_complex *dst, size_t n, size_t batch, size_t delay);
/* HistogramFeeder: the decision variable of every sample -- |x|, arg x, or arg(x[p] conj(x[p-1])) for p >= 1
 * (Tasks/HistogramFeeder.cpp:35-87).  out: [batch][count]; returns count (n, or n - 1 for FREQUENCY) */
long sdb_task_histogram_feed(const sdb_complex *src, float *out, size_t n, size_t batch, int space);
/* WaveSampler, sync = MANUAL: box-car average over each of (long) symbol_count symbol periods of
 * n / symbol_count samples with fractional edge weights; PHASE / FREQUENCY accumulate x conj(prev),
 * AMPLITUDE the RMS (Tasks/WaveSampler.cpp:28-46, 96-175).  out: [batch][count]; returns count */
long sdb_task_sample_manual(const sdb_complex *src, size_t n, size_t batch, int space, size_t symbol_sync,
                            double symbol_count, sdb_complex *out);
/* WaveSampler, sync = ZERO_CROSSING (Tasks/WaveSampler.cpp:222-292): run lengths between sign changes of
 * the decision variable, rounded to symbols with bnor = min(rate / fs, 1) symbols per sample; sym:
 * [batch][cap] bits (var > 0), counts[batch] = symbols produced (may exceed cap; the excess is dropped) */
int  sdb_task_sample_zero_crossing(const sdb_complex *src, size_t n, size_t batch, int space, int amplitude,
                                   float threshold_re, float threshold_im, float zc_angle_re, float zc_angle_im,
                                   float bnor, uint8_t *sym, uint32_t *counts, size_t cap);
/* CarrierDetector: Blackman-Harris, zero-padded power spectrum, strongest bin outside the DC notch, centroid
 * over avg_rel_bw of the band (Tasks/CarrierDetector.cpp:49-147).  peak[batch]: rad / sample in (-pi, pi];
 * n <= 2^20 */
int  sdb_task_carrier_detect(const sdb_complex *src, size_t n, size_t batch, double avg_rel_bw,
                             double dc_notch_rel_bw, float *peak);
/* SNR estimator the inspector tab runs on its decision-space histogram (Misc/SNREstimator.cpp:30-169,
 * include/SNREstimator.h; fed at Default/GenericInspector/InspectorUI.cpp:822-836): a comb of 2^bps Gaussians of
 * width sigma fitted to the normalised histogram, one gradient step per feed.  A batch of estimators (one per
 * inspector), histories of `length` bins each. */
typedef struct sdb_snr_estimator sdb_snr_estimator_t;
sdb_snr_estimator_t *sdb_snr_estimator_new(uint32_t n_estimators, uint32_t length, int device);
void sdb_snr_estimator_destroy(sdb_snr_estimator_t *e);
int  sdb_snr_estimator_set_bps(sdb_snr_estimator_t *e, uint32_t index, uint32_t bps);     /* restarts sigma at 1/8 */
int  sdb_snr_estimator_set_alpha(sdb_snr_estimator_t *e, uint32_t index, float alpha);
int  sdb_snr_estimator_set_sigma(sdb_snr_estimator_t *e, uint32_t index, float sigma);
int  sdb_snr_estimator_feed(sdb_snr_estimator_t *e, const uint32_t *histories /* host, [n][length] */);
/* sigma[n], snr[n] = 1 / (2^bps sigma), model[n][length]; any of them may be NULL */
int  sdb_snr_estimator_read(sdb_snr_estimator_t *e, float *sigma, float *snr, float *model);

/* Decider over sampler output (Default/GenericInspector/InspectorUI.cpp:836-846; Tasks/WaveSampler.cpp:316-317):
 * mode 0 = argument on [min, max), 1 = modulus; sym[i] in [0, 2^bps) */
int  sdb_task_decide(const sdb_complex *soft, uint8_t *sym, size_t n, int mode, unsigned bps, float min, float max);

/* ------------------------------------------------------------------------------------------------
 * Capture files (SURVEY.md 8(f) rank 2): the file source of Default/SourceConfig/FileSourcePage.cpp:68-140
 * (SUSCAN_SOURCE_FORMAT_{AUTO, RAW_*, WAV, SIGMF} + metadata guessed from the file name; SigDigger's own
 * recordings are "sigdigger_%Y%m%d_%H%M%SZ_<rate>_<freq>_float32_iq.raw", Default/Source/SourceWidget.cpp:1092-1100).
 * The file is mapped read-only; samples stay in their native format and are converted inside the first load of the
 * transforms (sdb_engine_params.input_format / sdb_source_config.input_format).  Host-only: works without a GPU.
 * ---------------------------------------------------------------------------------------------- */
enum { SDB_CONTAINER_AUTO = -1, SDB_CONTAINER_RAW = 0, SDB_CONTAINER_WAV = 1, SDB_CONTAINER_SIGMF = 2 };
#define SDB_CAPTURE_GUESS_START_TIME 1u   /* SUSCAN_SOURCE_CONFIG_GUESS_START_TIME */
#define SDB_CAPTURE_GUESS_SAMP_RATE  2u   /* ..._GUESS_SAMP_RATE */
#define SDB_CAPTURE_GUESS_FREQ       4u   /* ..._GUESS_FREQ */
#define SDB_CAPTURE_GUESS_FORMAT     8u
typedef struct {
  int32_t  container, sample_format;      /* SDB_CONTAINER_*, SDB_FORMAT_* */
  double   samp_rate, frequency;          /* 0 when the container does not say */
  uint64_t data_offset, n_samples;        /* byte offset of the first IQ pair, number of IQ pairs */
  uint32_t guessed;                       /* SDB_CAPTURE_GUESS_* bits filled from the file name (raw files) */
  int64_t  start_time;                    /* UTC seconds */
} sdb_capture_info;
typedef struct sdb_capture sdb_capture_t;
/* container = SDB_CONTAINER_AUTO picks by extension (.wav, .sigmf-meta / .sigmf-data, anything else raw);
 * sample_format < 0 = from the container or the file name (raw default: float32) */
sdb_capture_t *sdb_capture_open(const char *path, int32_t container, int32_t sample_format, sdb_capture_info *info);
const void    *sdb_capture_data(const sdb_capture_t *c);
void           sdb_capture_close(sdb_capture_t *c);
const char    *sdb_capture_last_error(void);

/* Recording side.  Host-only as well.
 *  - baseband capture: what the GUI's baseband-filter hook writes (Default/Source/SourceWidget.cpp:1078-1100,
 *    1156-1171; Misc/FileDataSaver.cpp:68-82): complex float32 blocks appended to
 *    "sigdigger_%Y%m%d_%H%M%SZ_<rate>_<freq>_float32_iq.raw".  The recorder also stores u8 / s8 / s16 (inverse of
 *    the loader's scaling, round to nearest, saturating) and the WAV / SigMF containers sdb_capture_open() reads.
 *  - audio: mono PCM16 WAV of Re{x} named "audio-<AM|FM|USB|LSB|RAW>-<freq>-<rate>-<NNNN>.wav", first free index
 *    (Audio/AudioFileSaver.cpp:57-107,131-152).
 * Errors: NULL / -1 with the text in sdb_capture_last_error(). */
typedef struct {
  int32_t container, sample_format;       /* SDB_CONTAINER_RAW / WAV / SIGMF; SDB_FORMAT_* as stored */
  double  samp_rate, frequency;
  int64_t start_time;                     /* UTC seconds; 0 = now */
} sdb_recorder_params;
typedef struct sdb_recorder sdb_recorder_t;
/* auto_name != 0: `path` is a directory and the file gets SigDigger's capture name */
sdb_recorder_t *sdb_recorder_open(const char *path, int32_t auto_name, const sdb_recorder_params *p);
sdb_recorder_t *sdb_audio_recorder_open(const char *dir, int32_t demod, double frequency, uint32_t samp_rate);
const char     *sdb_recorder_path(const sdb_recorder_t *r);
uint64_t        sdb_recorder_samples(const sdb_recorder_t *r);
long            sdb_recorder_write(sdb_recorder_t *r, const sdb_complex *x, size_t n);   /* returns n or -1 */
int             sdb_recorder_close(sdb_recorder_t *r);                                    /* patches WAV sizes */
int             sdb_capture_file_name(char *dst, size_t cap, int64_t utc_seconds, int32_t sample_format,
                                      double samp_rate, double frequency);
/* The audio inspector's caller (Default/Audio/AudioProcessor.cpp): which channel it opens, where LO and bandwidth
 * really go for the side-band modes, and what it writes into the audio.* keys.  demod = SigDigger's AudioDemod
 * (0 AM, 1 FM, 2 USB, 3 LSB, 4 RAW; include/SigDiggerHelpers.h:39-45).  Host-only parameter arithmetic. */
typedef struct {
  double   max_audio_bw;                     /* min(fs / 2, 2e5)                      (AudioProcessor.cpp:118-121) */
  uint32_t sample_rate;                      /* requested rate floored to it          (:123-125) */
  double   true_bw, true_lo;                 /* calcTrueBandwidth / calcTrueLoFreq    (:200-228) */
  double   ch_fc, ch_ft, ch_bw, ch_f_lo, ch_f_hi;   /* channel of requestOpen("audio", ch)   (:143-151) */
} sdb_audio_plan;
int sdb_audio_plan_make(double analyzer_samp_rate, uint32_t requested_rate, int32_t demod, double lo, double bw,
                        sdb_audio_plan *out);
/* setParams() (:250-269): fills audio_cutoff / volume (1) / sample_rate / demod (+1 on the wire) / squelch / agc */
int sdb_audio_plan_config(const sdb_audio_plan *plan, int32_t demod, float cutoff, int32_t squelch, float squelch_level,
                          int32_t agc, float agc_ts, sdb_inspector_config *cfg);
/* Inspector recording / forwarding formats (Default/GenericInspector/InspectorUI.cpp:860-930): the bytes the data
 * saver receives for each data variable.  decision_mode: 0 argument (arg(i x) / pi), 1 modulus.  Returns bytes. */
enum { SDB_DATAVAR_DECISION_SPACE = 0, SDB_DATAVAR_SOFT_BITS, SDB_DATAVAR_SOFT_BITS_I, SDB_DATAVAR_SOFT_BITS_Q,
       SDB_DATAVAR_SYMBOLS };
long            sdb_inspector_forward(int32_t data_var, int32_t decision_mode, const sdb_complex *soft,
                                      const uint8_t *hard, size_t n, void *dst);

/* ------------------------------------------------------------------------------------------------
 * suscan-style asynchronous analyzer (SURVEY.md 8(a) a18, 8(b)): a worker thread reads the source, runs the
 * engine block by block and posts messages; requests are answered in order with messages carrying req_id.
 * Field names follow the structs the reference dereferences (Suscan/Messages/PSDMessage.cpp:30-112,
 * include/Suscan/Messages/SamplesMessage.h:33-59, Suscan/Messages/InspectorMessage.cpp:28-252,
 * Suscan/Messages/StatusMessage.cpp:33-45, include/Suscan/Analyzer.h:113-254).
 * ---------------------------------------------------------------------------------------------- */
#include <sys/time.h>

enum {   /* SUSCAN_ANALYZER_MESSAGE_TYPE_* as dispatched at Suscan/Analyzer.cpp:75-98 */
  SDB_ANALYZER_MESSAGE_TYPE_SOURCE_INFO = 0, SDB_ANALYZER_MESSAGE_TYPE_SOURCE_INIT, SDB_ANALYZER_MESSAGE_TYPE_CHANNEL,
  SDB_ANALYZER_MESSAGE_TYPE_EOS, SDB_ANALYZER_MESSAGE_TYPE_READ_ERROR, SDB_ANALYZER_MESSAGE_TYPE_INTERNAL,
  SDB_ANALYZER_MESSAGE_TYPE_SAMPLES, SDB_ANALYZER_MESSAGE_TYPE_INSPECTOR, SDB_ANALYZER_MESSAGE_TYPE_PSD,
  SDB_ANALYZER_MESSAGE_TYPE_PARAMS
};
#define SDB_WORKER_MSG_TYPE_HALT   0xffffffffu      /* SUSCAN_WORKER_MSG_TYPE_HALT */
#define SDB_ANALYZER_INIT_FAILURE  (-1)             /* SUSCAN_ANALYZER_INIT_FAILURE, App/Application.cpp:529 */
enum {   /* SUSCAN_ANALYZER_INSPECTOR_MSGKIND_* (Suscan/AnalyzerRequestTracker.cpp:138-177) */
  SDB_INSPECTOR_MSGKIND_OPEN = 0, SDB_INSPECTOR_MSGKIND_SET_ID, SDB_INSPECTOR_MSGKIND_GET_CONFIG,
  SDB_INSPECTOR_MSGKIND_SET_CONFIG, SDB_INSPECTOR_MSGKIND_ESTIMATOR, SDB_INSPECTOR_MSGKIND_SPECTRUM,
  SDB_INSPECTOR_MSGKIND_CLOSE, SDB_INSPECTOR_MSGKIND_INVALID_CHANNEL, SDB_INSPECTOR_MSGKIND_WRONG_HANDLE,
  SDB_INSPECTOR_MSGKIND_WRONG_OBJECT, SDB_INSPECTOR_MSGKIND_WRONG_KIND,
  SDB_INSPECTOR_MSGKIND_FAC,         /* this project's: the FAC tab (oracle/SPEC_FC.md); suscan has no such kind */
  SDB_INSPECTOR_MSGKIND_SNR          /* this project's: the SNR meter (oracle/SPEC_SN.md); suscan has no such kind */
};
enum { SDB_ANALYZER_MODE_CHANNEL = 0, SDB_ANALYZER_MODE_WIDE_SPECTRUM = 1 };

/* struct sigutils_channel {fc, ft, f_lo, f_hi, bw} (Suscan/Analyzer.cpp:417-424); Hz, fc relative to the tuner */
typedef struct { double fc, ft, f_lo, f_hi; float bw; } sdb_sigutils_channel;

/* struct suscan_analyzer_params (Suscan/AnalyzerParams.cpp:27-68) */
typedef struct {
  int32_t mode;
  struct { uint64_t window_size; int32_t window; float alpha, beta, gamma, snr; } detector_params;
  float   channel_update_int, psd_update_int;       /* seconds */
  double  min_freq, max_freq;
  /* Channel mode: non-zero posts, instead of one frame per psd_update_int, the mean of every
   * A = clamp(llround(psd_update_int * rate / window_size), 1, SDB_PSD_AVERAGE_MAX) frames (SPEC A), time-stamped at
   * its first sample; 0 = one frame per interval.  Wide-spectrum sweeps ignore it. */
  int32_t psd_average;
  /* Channel mode: SDB_PSD_DETECTOR_POS_PEAK / _NEG_PEAK post, instead, the per-bin maximum / minimum of every
   * P = clamp(llround(psd_update_int * rate / window_size), 1, SDB_PSD_PEAK_MAX) frames (SPEC PK), time-stamped at the
   * first sample of the group; a detector takes precedence over psd_average.  SDB_PSD_DETECTOR_DEFAULT = one frame per
   * interval, or the mean with psd_average.  sdb_analyzer_new and _set_params_async refuse other values; wide-spectrum
   * sweeps ignore it. */
  int32_t psd_detector;
  /* Seconds between inspector spectra and baud estimates.  > 0: every inspector with a spectrum source or an
   * estimator takes 4096-point frames from a window carried across blocks and emits every
   * I = max(1, llround(spectrum_update_int * channel rate)) channel samples (oracle/SPEC_US.md), one SPECTRUM message
   * and one ESTIMATOR message per valid estimate each time, in order, after the block's SAMPLES.  An I that would
   * allow more than SDB_SPECTRUM_EMITS_MAX emissions in one block is raised to ceil(channel samples per block /
   * SDB_SPECTRUM_EMITS_MAX).  0 = one emission per block that fills a frame, of the largest power of two <= 4096 the
   * block fills.  sdb_analyzer_new and _set_params_async refuse negative values, infinities and NaN. */
  float   spectrum_update_int;
  /* Channel tracking (oracle/SPEC_KT.md), seconds.  0 (the default): none, and CHANNEL messages carry each update's
   * detector list as before.  > 0: the detector follows channels across updates with
   * hold = ceil(channel_hold_int / block duration) updates (at most SDB_CHTRACK_HOLD_MAX), and CHANNEL messages carry
   * the tracked list: a channel that drops out for less than the hold stays one entry, S0 is smoothed by
   * detector_params.beta (which must then be in (0, 1]), and tracked_list adds ids, age and present.  The detector
   * runs only when channel_update_int > 0, so without it this has no effect.  Any re-plan restarts the tracks, as it
   * restarts the detector.  Negative, NaN and infinite values are refused. */
  float   channel_hold_int;
} sdb_analyzer_params;
enum { SDB_PSD_DETECTOR_DEFAULT = 0, SDB_PSD_DETECTOR_POS_PEAK = 1, SDB_PSD_DETECTOR_NEG_PEAK = 2 };

/* the part of suscan_source_config_t this path needs: a callback source (role of file / stdin / SoapySDR
 * back-ends) or an in-memory capture */
typedef long (*sdb_source_read_fn)(void *priv, sdb_complex *dst, size_t max_samples);   /* 0 = EOS, < 0 = error */
typedef struct {
  double  samp_rate, freq;
  size_t  read_size;              /* samples per block (rounded to a multiple of window_size; 0 = 8 windows) */
  sdb_source_read_fn read; void *priv;
  const sdb_complex *data; size_t length; int32_t loop;
  int32_t device;
  int32_t input_format;           /* SDB_FORMAT_* of `data` (length counts IQ pairs); callback sources deliver float32 */
  int (*set_frequency)(void *priv, double freq);   /* tuner of the source; used by the wide-spectrum mode (may be NULL) */
  /* suscan_source_config_set_average (Suscan/Source.cpp:195-201): source decimation D (0 or 1 = none, at most
   * SDB_DECIMATION_MAX; channel mode only).  Every block reads D x read_size source samples, the FIR decimator
   * (SPEC L) brings them to samp_rate / D, and everything downstream -- PSD, inspectors, channel detector, baseband
   * filters, history -- runs at samp_rate / D.  Source time, seek and the throttle stay in source samples. */
  uint32_t decimation;
} sdb_source_config;

/* Wide-spectrum (panoramic) mode, sdb_analyzer_params.mode = SDB_ANALYZER_MODE_WIDE_SPECTRUM
 * (Panoramic/Scanner.cpp:296-372): the worker retunes the source, drops `buffering_size` samples, takes one window and
 * posts its PSD with the hop centre in psd_msg.fc; the hop plan follows min_freq / max_freq (set_hop_range),
 * rel_bandwidth, the sweep strategy and the partitioning (Panoramic/Scanner.cpp:396-431, 452-503;
 * include/Suscan/Analyzer.h:263-271, 321-333). */
enum { SDB_SWEEP_STRATEGY_STOCHASTIC = 0, SDB_SWEEP_STRATEGY_PROGRESSIVE = 1 };
enum { SDB_SPECTRUM_PARTITIONING_DISCRETE = 0, SDB_SPECTRUM_PARTITIONING_CONTINUOUS = 1 };

typedef struct {                  /* suscan_analyzer_psd_msg */
  int64_t fc; uint32_t inspector_id; struct timeval timestamp, rt_time; int32_t looped; uint64_t history_size;
  float samp_rate, measured_samp_rate; uint64_t psd_size; float *psd_data;
} sdb_analyzer_psd_msg;
typedef struct {                  /* suscan_analyzer_sample_batch_msg (+ the GUI Decider's output) */
  uint32_t inspector_id; sdb_complex *samples; uint64_t sample_count; uint8_t *symbols;
} sdb_analyzer_sample_batch_msg;
typedef struct {                  /* suscan_analyzer_inspector_msg, fields this path fills */
  int32_t kind; uint32_t inspector_id, req_id; int32_t handle; char *class_name; sdb_sigutils_channel channel;
  sdb_inspector_config config; float fs, equiv_fs, bandwidth, lo;
  /* kind = OPEN: sizes of the spectrum-source / estimator lists (names: sdb_spectsrc_name(1..), sdb_estimator_name)
   * (spectsrc_count / estimator_count, Suscan/Messages/InspectorMessage.cpp:40-61).
   * kind = SPECTRUM: spectsrc_id, spectrum_data[spectrum_size] (linear power, DC at 0), samp_rate
   * (InspectorMessage.cpp:75-100); kind = ESTIMATOR: estimator_id, enabled, value (:120-135). */
  uint32_t spectsrc_count, estimator_count;
  uint32_t spectsrc_id; float *spectrum_data; uint64_t spectrum_size; uint64_t samp_rate;
  uint32_t estimator_id; int32_t enabled; float value;
  /* kind = FAC: the acknowledgement of sdb_analyzer_inspector_set_fac_async (no data), or, after the SAMPLES of every
   * block that completed at least one FAC block, fac[size / 2] in spectrum_data / spectrum_size and the block's status
   * here (sdb_engine_read_fac) */
  sdb_fac_status fac;
  /* kind = SNR: the acknowledgement of sdb_analyzer_inspector_set_snr_async / _reset_snr_async (no data), or, after the
   * SAMPLES of every block in which the meter stepped, the model[bins] in spectrum_data / spectrum_size, the status here
   * and h[bins] in snr_histogram (freed with the message) (sdb_engine_read_snr) */
  sdb_snr_status snr;
  uint32_t *snr_histogram;
} sdb_analyzer_inspector_msg;
/* suscan_analyzer_channel_msg (Suscan/Messages/ChannelMessage.cpp:25-70): posted every channel_update_int seconds
 * of signal time when channel_update_int > 0 */
typedef struct {
  const void *source; uint32_t channel_count; sdb_detected_channel *channel_list;
  /* with channel_hold_int > 0: the same channel_count tracks in full, in the order of channel_list; otherwise NULL */
  sdb_tracked_channel *tracked_list;
} sdb_analyzer_channel_msg;
typedef struct { int32_t code; char *err_msg; } sdb_analyzer_status_msg;   /* suscan_analyzer_status_msg */
typedef struct {                  /* suscan_source_info, fields this path fills */
  uint64_t permissions, source_samp_rate, effective_samp_rate; float measured_samp_rate; double frequency;
  int32_t seekable;
} sdb_source_info;

typedef struct sdb_analyzer sdb_analyzer_t;
sdb_analyzer_t *sdb_analyzer_new(const sdb_analyzer_params *params, const sdb_source_config *src);  /* Analyzer.cpp:608 */
void  *sdb_analyzer_read(sdb_analyzer_t *a, uint32_t *type);                 /* blocking; Analyzer.cpp:111-115 */
void  *sdb_analyzer_read_timeout(sdb_analyzer_t *a, uint32_t *type, unsigned timeout_ms);
void   sdb_analyzer_dispose_message(uint32_t type, void *ptr);               /* Suscan/Message.cpp:43-48 */
void   sdb_analyzer_req_halt(sdb_analyzer_t *a);                             /* Analyzer.cpp:321 */
void   sdb_analyzer_destroy(sdb_analyzer_t *a);                              /* Analyzer.cpp:625-638 */
int    sdb_analyzer_open_ex_async(sdb_analyzer_t *a, const char *class_name, const sdb_sigutils_channel *ch,
                                  int precise, int32_t parent, uint32_t req_id);        /* Analyzer.cpp:459-484 */
int    sdb_analyzer_set_inspector_id_async(sdb_analyzer_t *a, int32_t handle, uint32_t inspector_id, uint32_t req_id);
int    sdb_analyzer_set_inspector_config_async(sdb_analyzer_t *a, int32_t handle, const sdb_inspector_config *cfg,
                                               uint32_t req_id);
int    sdb_analyzer_close_async(sdb_analyzer_t *a, int32_t handle, uint32_t req_id);
/* suscan_analyzer_set_inspector_watermark_async (Suscan/Analyzer.cpp:527-537; Default/Audio/AudioProcessor.cpp:745-747):
 * SAMPLES batches of this inspector are held back until they contain `watermark` samples (0 = one batch per block) */
int    sdb_analyzer_set_inspector_watermark_async(sdb_analyzer_t *a, int32_t handle, uint64_t watermark, uint32_t req_id);
/* suscan_analyzer_set_inspector_freq_overridable / _bandwidth_overridable (Suscan/Analyzer.cpp:509-526): no reply, the
 * latest value wins; freq in Hz relative to the tuner (or to the parent's centre), bw in Hz */
int    sdb_analyzer_set_inspector_freq_overridable(sdb_analyzer_t *a, int32_t handle, double freq);
int    sdb_analyzer_set_inspector_bandwidth_overridable(sdb_analyzer_t *a, int32_t handle, double bw);
/* suscan_analyzer_inspector_set_spectrum_async / _estimator_cmd_async (Suscan/Analyzer.cpp:539-565) */
int    sdb_analyzer_inspector_set_spectrum_async(sdb_analyzer_t *a, int32_t handle, uint32_t spectsrc_id, uint32_t req_id);
/* the FAC tab of a psk / fsk / ask inspector (sdb_engine_set_fac; p NULL = off), from the next block on, through the
 * re-plan: the FAC state carries over as sdb_engine_migrate says.  Acknowledged by an INSPECTOR message of kind FAC;
 * WRONG_HANDLE, WRONG_KIND (another class) or WRONG_OBJECT (parameters sdb_engine_set_fac refuses) otherwise. */
int    sdb_analyzer_inspector_set_fac_async(sdb_analyzer_t *a, int32_t handle, const sdb_fac_params *p, uint32_t req_id);
/* the SNR meter of a psk / fsk / ask inspector (sdb_engine_set_snr; p NULL = off), from the next block on, through the
 * re-plan: its state carries over as SPEC SN.4 says.  The meter steps once per block, not once per SAMPLES batch.
 * reset_snr sets sigma (sdb_engine_reset_snr) at the next block boundary, without a re-plan.  Both are acknowledged
 * by an INSPECTOR message of kind SNR; WRONG_HANDLE, WRONG_KIND (another class) or WRONG_OBJECT (parameters
 * sdb_engine_set_snr refuses, or a reset with the meter off or a sigma that is not finite and positive) otherwise. */
int    sdb_analyzer_inspector_set_snr_async(sdb_analyzer_t *a, int32_t handle, const sdb_snr_params *p, uint32_t req_id);
int    sdb_analyzer_inspector_reset_snr_async(sdb_analyzer_t *a, int32_t handle, float sigma, uint32_t req_id);
int    sdb_analyzer_inspector_estimator_cmd_async(sdb_analyzer_t *a, int32_t handle, uint32_t estimator_id,
                                                  int enabled, uint32_t req_id);
int    sdb_analyzer_set_params_async(sdb_analyzer_t *a, const sdb_analyzer_params *p, uint32_t req_id);
/* source-side options of the worker loop: suscan_analyzer_set_iq_reverse (Suscan/Analyzer.cpp:238-244; applied at
 * the next block boundary, swap done inside the first load on the GPU), suscan_analyzer_set_throttle_async
 * (Suscan/Analyzer.cpp:117-123; 0 = unthrottled) and suscan_analyzer_register_baseband_filter
 * (Suscan/Analyzer.cpp:126-130; SUBOOL f(privdata, analyzer, samples, length, offset) as used by the GUI's baseband
 * recorder, Default/Source/SourceWidget.cpp:1156-1184): called on the worker thread with every float32 block before
 * it is analysed; it may rewrite the samples. */
typedef int (*sdb_baseband_filter_fn)(void *privdata, sdb_analyzer_t *a, sdb_complex *samples, uint64_t length,
                                      uint64_t offset);
/* suscan_analyzer_seek (Suscan/Analyzer.cpp:151-155): position (signal time) in a seekable source, i.e. an in-memory
 * / mapped capture; applied at the next block boundary; -1 for callback sources */
int    sdb_analyzer_seek(sdb_analyzer_t *a, const struct timeval *pos);
/* suscan_analyzer_set_history_size / suscan_analyzer_replay (Suscan/Analyzer.cpp:157-167; GUI: Default/Source/
 * SourceWidget.cpp:1070-1073, 1206, 1508): keep the last `samples` float32 baseband samples in a ring; replay pauses
 * the source and plays the ring in a loop (psd_msg.looped / .history_size report it) */
int    sdb_analyzer_set_history_size(sdb_analyzer_t *a, uint64_t samples);
int    sdb_analyzer_replay(sdb_analyzer_t *a, int enabled);
int    sdb_analyzer_set_hop_range(sdb_analyzer_t *a, double min_freq, double max_freq);   /* Analyzer.cpp:255-260 */
int    sdb_analyzer_set_rel_bandwidth(sdb_analyzer_t *a, float rel_bw);
int    sdb_analyzer_set_buffering_size(sdb_analyzer_t *a, uint64_t samples);
int    sdb_analyzer_set_sweep_strategy(sdb_analyzer_t *a, int strategy);
int    sdb_analyzer_set_spectrum_partitioning(sdb_analyzer_t *a, int partitioning);
int    sdb_analyzer_set_iq_reverse(sdb_analyzer_t *a, int enabled);
int    sdb_analyzer_set_dc_remove(sdb_analyzer_t *a, int enabled);        /* Suscan/Analyzer.cpp:229-236; SPEC R */
int    sdb_analyzer_set_throttle_async(sdb_analyzer_t *a, uint64_t samp_rate, uint32_t req_id);
int    sdb_analyzer_register_baseband_filter(sdb_analyzer_t *a, sdb_baseband_filter_fn fn, void *privdata);
/* suscan_analyzer_register_baseband_filter_with_prio (Suscan/Analyzer.cpp:137-143): ascending priority value */
int    sdb_analyzer_register_baseband_filter_prio(sdb_analyzer_t *a, sdb_baseband_filter_fn fn, void *privdata,
                                                  int64_t prio);
/* suscan_analyzer_get_source_time (Suscan/Analyzer.cpp:145-149): signal time since the start of the source, seconds */
double sdb_analyzer_get_source_time(const sdb_analyzer_t *a);
/* configuration an open inspector currently runs with (the payload of a GET_CONFIG reply); -1: not open */
int    sdb_analyzer_get_inspector_config(sdb_analyzer_t *a, int32_t handle, sdb_inspector_config *cfg);
uint64_t sdb_analyzer_get_samp_rate(const sdb_analyzer_t *a);
float    sdb_analyzer_get_measured_samp_rate(const sdb_analyzer_t *a);

/* ------------------------------------------------------------------------------------------------
 * Panoramic scanner: SpectrumView (Panoramic/Scanner.cpp:36-293, constants include/Scanner.h:26-32).
 * The reference does view.feed(psd, nullptr, fftSize, fc) per PSD message on the GUI thread
 * (Panoramic/Scanner.cpp:503-523).  Here the per-hop projection (the O(psd_size) part) is separate from
 * the order-dependent per-bin accumulation so that hops can be spread over GPUs: project on every rank,
 * gather the small contribution lists (NCCL), accumulate on rank 0.  project + accumulate of the same
 * hops in the same order == the reference's feed() sequence, value by value.
 * ---------------------------------------------------------------------------------------------- */
typedef struct sdb_sview sdb_sview_t;
sdb_sview_t *sdb_sview_new(int device);
void         sdb_sview_destroy(sdb_sview_t *v);
/* SpectrumView::setRange + fftBandwidth / fftRelBw members; resets the view */
int      sdb_sview_set_range(sdb_sview_t *v, double freq_min, double freq_max, double fft_bandwidth, float rel_bw);
int      sdb_sview_reset(sdb_sview_t *v);                         /* SpectrumView::reset */
uint32_t sdb_sview_size(const sdb_sview_t *v);                    /* spectrumSize */
uint32_t sdb_sview_max_bins(const sdb_sview_t *v);                /* row pitch of the contribution lists */
/* psd_dev: device pointer [n_hops][psd_size], PSDMessage layout (shifted, dB); centers: host doubles */
int      sdb_sview_project(sdb_sview_t *v, const float *psd_dev, size_t psd_size, const double *centers,
                           size_t n_hops, int adjust_sides);
/* PSDMessage post-processing as a separate pass (Suscan/Messages/PSDMessage.cpp:32-38: swap halves,
 * SU_POWER_DB) for engines that keep the linear PSD for the channel detector: db[f][(k+n/2)%n] =
 * 10 log10(lin[f][k] + 1e-8), bit-identical to SDB_FLAG_PSD_SHIFT_DB.  Device pointers, out of place. */
int      sdb_psd_shift_db_device(const float *lin_dev, float *db_dev, size_t n_frames, uint32_t psd_size);
/* Spectrum averager the GUI runs on every PSD message (Misc/Averager.cpp:25-60; fed at
 * UIMediator/SpectrumMediator.cpp:128): per bin last += alpha (x - last), first frame (and alpha >= 1) copied.
 * One state row of psd_size bins per stream, on the device; frames of a feed are applied in order.
 * psd_dev: [n_streams] rows of `frames` frames, `stream_stride` floats apart (e.g. sdb_engine_psd_device).
 * Both passes run on the default stream: the producer of psd_dev must have completed (sdb_engine_sync). */
typedef struct sdb_averager sdb_averager_t;
sdb_averager_t *sdb_averager_new(uint32_t psd_size, uint32_t n_streams, float alpha, int device);
void         sdb_averager_destroy(sdb_averager_t *a);
int          sdb_averager_set_alpha(sdb_averager_t *a, float alpha);      /* Averager::setAlpha */
int          sdb_averager_reset(sdb_averager_t *a);                       /* Averager::reset: next frame is copied */
int          sdb_averager_feed_device(sdb_averager_t *a, const float *psd_dev, size_t frames, size_t stream_stride);
const float *sdb_averager_device(const sdb_averager_t *a);                /* [n_streams][psd_size] */
int          sdb_averager_read(sdb_averager_t *a, float *dst, size_t cap);
/* Source decimator (SPEC L, oracle/SPEC_L.md; the source config's `average`, Suscan/Source.cpp:195-201): anti-aliased FIR decimation
 * by D in [1, SDB_DECIMATION_MAX] with the brick-wall low-pass of 16 D + 1 taps at fc = 1/D (SPEC I.3), over
 * n_streams streams fed together.  Output k of a stream is sum_i h_i x[kD - i]; the last 16 D input samples and the
 * input phase are carried per stream on the device, so the outputs do not depend on how the input is split into
 * feeds (a feed of m D samples yields m outputs).  Input: [n_streams] rows of n samples in input_format, stream_stride
 * samples apart.  A device feed must be readable by the time the decimator's stream runs (synchronise its producer
 * first).  Each feed returns its outputs per stream and overwrites the previous feed's output: [n_streams] rows,
 * sdb_decimator_output_stride() complex samples apart, valid after sdb_decimator_sync. */
#define SDB_DECIMATION_MAX 256
typedef struct sdb_decimator sdb_decimator_t;
sdb_decimator_t *sdb_decimator_new(int device, uint32_t n_streams, uint32_t decimation, int32_t input_format,
                                   size_t max_feed);
void     sdb_decimator_destroy(sdb_decimator_t *d);
long     sdb_decimator_feed_device(sdb_decimator_t *d, const void *x, size_t stream_stride, size_t n);
long     sdb_decimator_feed_host(sdb_decimator_t *d, const void *x, size_t stream_stride, size_t n);
const sdb_complex *sdb_decimator_output_device(const sdb_decimator_t *d);
size_t   sdb_decimator_output_stride(const sdb_decimator_t *d);
void    *sdb_decimator_stream(const sdb_decimator_t *d);                          /* cudaStream_t of the feeds */
int      sdb_decimator_sync(sdb_decimator_t *d);
int      sdb_decimator_read(sdb_decimator_t *d, sdb_complex *dst, size_t cap);   /* [n_streams][outputs of last feed] */
int      sdb_decimator_reset(sdb_decimator_t *d);                                 /* zero carry, phase 0 */
/* device pointers of the last projection: j0[n_hops], nb[n_hops], va/vc[n_hops][max_bins] */
int      sdb_sview_contrib(sdb_sview_t *v, int32_t **j0, int32_t **nb, float **va, float **vc);
/* copy them into caller-owned device buffers (e.g. the send buffers of the NCCL gather) */
int      sdb_sview_contrib_copy(sdb_sview_t *v, int32_t *j0, int32_t *nb, float *va, float *vc, size_t n_hops);
/* apply contribution lists (device pointers; own or gathered from peers) in hop order, then fill gaps */
int      sdb_sview_accumulate(sdb_sview_t *v, const int32_t *j0, const int32_t *nb, const float *va,
                              const float *vc, size_t n_hops);
int      sdb_sview_read(sdb_sview_t *v, float *psd, float *accum, float *count, size_t cap);

/* ------------------------------------------------------------------------------------------------
 * Panoramic sweep over the GPUs of one node (BASELINE.json configs[4]: tuner hops x PSD stitched over NVLink, per-GPU
 * channel detector, gather to rank 0).  One process per GPU; rank r owns a contiguous shard of the hop list
 * (sdb_panoramic_shard), computes its hop PSDs, projects them onto the SpectrumView grid (and detects channels per
 * hop), and the packed contribution lists are gathered on rank 0 with NCCL -- the one collective of the path -- where
 * they are applied in global hop order: the result equals the reference's sequential view.feed(psd, nullptr, fftSize,
 * fc) series (Panoramic/Scanner.cpp:503-523) value by value.  world = 1 needs no NCCL.
 * The 128-byte NCCL id comes from sdb_panoramic_unique_id() on rank 0 and reaches the peers by whatever the launcher
 * offers (torch.distributed broadcast, MPI, a file); NCCL itself is bound at run time (dlopen "libnccl.so.2").
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  uint32_t psd_size; int32_t psd_window;      /* points per hop, SDB_WINDOW_* */
  double   fft_bandwidth;                     /* sample rate of a hop (Hz) */
  float    rel_bw;                            /* kept fraction of a hop, include/Scanner.h:70 (0 -> 0.5) */
  double   freq_min, freq_max;                /* view range (Hz) */
  int32_t  device;
  int32_t  detect;                            /* per-hop channel detector (SPEC K) on the owning rank */
  float    det_alpha, det_gamma, det_snr; uint32_t det_min_bins, channel_cap;
  uint32_t frames_per_hop;                    /* windows per hop (0 = 1): the detector averages them, the view takes the last */
} sdb_panoramic_params;
typedef struct {
  float    psd_project_ms, gather_ms, accumulate_ms;   /* device time of the three phases of the last sweep */
  uint64_t gather_bytes;                               /* bytes rank 0 received (0 on one GPU) */
  uint64_t n_hops_local;
} sdb_panoramic_timing;
typedef struct sdb_panoramic sdb_panoramic_t;
int              sdb_panoramic_unique_id(void *id128);
sdb_panoramic_t *sdb_panoramic_new(const sdb_panoramic_params *p, int rank, int world, const void *id128);
void             sdb_panoramic_destroy(sdb_panoramic_t *s);
void             sdb_panoramic_shard(size_t n_hops, int world, int rank, size_t *lo, size_t *hi);
/* hops_local: this rank's shard [hi - lo][psd_size] complex64, one window per hop (device / host pointer);
 * centers_all: host, all n_hops hop centres in sweep order.  Collective: every rank calls it. */
int      sdb_panoramic_sweep_device(sdb_panoramic_t *s, const sdb_complex *hops_local_dev, const double *centers_all,
                                    size_t n_hops);
int      sdb_panoramic_sweep_host(sdb_panoramic_t *s, const sdb_complex *hops_local, const double *centers_all,
                                  size_t n_hops);
int      sdb_panoramic_reset(sdb_panoramic_t *s);                       /* SpectrumView::reset */
uint32_t sdb_panoramic_size(const sdb_panoramic_t *s);
int      sdb_panoramic_read(sdb_panoramic_t *s, float *psd, float *accum, float *count, size_t cap);   /* rank 0 */
/* channels the detector found in hop `hop` of the LAST sweep (rank 0, detector enabled; valid until the next sweep).
 * The sweep reads the lists back packed behind an event; a sweep with more than ~8 channels per hop on average is
 * served from the full device array on the first call. */
long     sdb_panoramic_read_channels(sdb_panoramic_t *s, size_t hop, sdb_detected_channel *out, size_t cap);
int      sdb_panoramic_last_timing(const sdb_panoramic_t *s, sdb_panoramic_timing *t);
const char *sdb_panoramic_last_error(void);

/* SpectrumView::feed(SpectrumView const &detail) (Panoramic/Scanner.cpp:276-286): seed / refine a view with another
 * one's accumulators weighted by its counts -- what Scanner::setViewRange does on zoom (:471-479: flip, setRange,
 * feed(previous)).  Both views on the same device. */
int      sdb_sview_feed_view(sdb_sview_t *v, const sdb_sview_t *detail);

/* ------------------------------------------------------------------------------------------------
 * Analog-TV processor of the inspector's TV tab (SURVEY.md 8(f) rank 4; SPEC.md section TV), a batch of processors,
 * one warp each.  sdb_tv_params has the fields of struct sigutils_tv_processor_params as the reference fills them
 * (Default/GenericInspector/TVProcessorTab.cpp:549-597; lengths in samples, time constants in their own units).
 * The input is the TV tab's real-valued signal with the sync tips HIGH (TVProcessorTab::feed, :601-620:
 * sdb_tv_feed_transform).  The sigutils-named per-sample interface (su_tv_processor_feed ...) is <sigutils/tvproc.h>.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int32_t  enable_sync, reverse, interlace, enable_agc;
  float    x_off;
  int32_t  dominance;
  uint32_t frame_lines;
  float    frame_spacing;                     /* fractional lines per frame beyond frame_lines (TVProcessorTab.cpp:559) */
  int32_t  enable_comb, comb_reverse;
  float    hsync_len, vsync_len, line_len;    /* samples */
  uint32_t vsync_odd_trigger;                 /* equalising pulses that end a field */
  float    t_tol, l_tol, g_tol;
  float    hsync_huge_err, hsync_max_err, hsync_min_err;
  float    hsync_len_tau, line_len_tau, agc_tau, hsync_fast_track_tau, hsync_slow_track_tau;
} sdb_tv_params;
typedef struct sdb_tv_processor sdb_tv_processor_t;
/* su_tv_processor_params_pal / _ntsc (TVProcessorTab.cpp:629,633) */
void sdb_tv_params_pal(sdb_tv_params *p, float samp_rate);
void sdb_tv_params_ntsc(sdb_tv_params *p, float samp_rate);
/* su_tv_processor_new / _destroy / _set_params (TVProcessorWorker.cpp:204, :175, :222) */
sdb_tv_processor_t *sdb_tv_processor_new(const sdb_tv_params *p, uint32_t batch, int device);
void sdb_tv_processor_destroy(sdb_tv_processor_t *t);
int  sdb_tv_processor_set_params(sdb_tv_processor_t *t, const sdb_tv_params *p);
int  sdb_tv_processor_geometry(const sdb_tv_processor_t *t, uint32_t *width, uint32_t *height);
/* TVProcessorWorker::work (TVProcessorWorker.cpp:120-151) over the batch: x[batch][stride], n <= stride samples each
 * (host or device memory); frames_done[batch]; returns the frames completed in this call (-1 on error) */
long sdb_tv_processor_feed(sdb_tv_processor_t *t, const float *x, size_t stride, size_t n, uint32_t *frames_done);
long sdb_tv_processor_feed_device(sdb_tv_processor_t *t, const float *x_dev, size_t stride, size_t n, uint32_t *frames_done);
int  sdb_tv_processor_frames(sdb_tv_processor_t *t, uint64_t *counts);
/* su_tv_processor_take_frame (TVProcessorWorker.cpp:143): completed frame `frame_no` of processor `which`,
 * [height][width] floats (0 = black ... 1 = white before contrast / brightness) */
int  sdb_tv_processor_read_frame(sdb_tv_processor_t *t, uint32_t which, uint64_t frame_no, float *out, size_t cap);
int  sdb_tv_processor_estimates(sdb_tv_processor_t *t, uint32_t which, float *line_len, float *hsync_len, float *gain);
/* TVProcessorTab::feed (TVProcessorTab.cpp:601-620): mode 0 = k |x| + dc, 1 = k arg(x) / pi + dc */
int  sdb_tv_feed_transform(const sdb_complex *x, size_t n, int mode, float k, float dc, float *out);

/* Offline inspector over captured channel-rate buffers (the block-wise CPU loops the GUI's TimeWindow
 * launches, Components/TimeWindow.cpp:1571-2183; sampler + decider of Tasks/WaveSampler.cpp:188-205,
 * 316-317): `batch` buffers of n samples -> soft [batch][cap], hard [batch][cap], counts [batch].
 * cfg->fs must be the buffers' sample rate. */
long sdb_task_inspector(const sdb_inspector_config *cfg, const sdb_complex *src, size_t n, size_t batch,
                        sdb_complex *soft, uint8_t *hard, uint32_t *counts, size_t cap);
/* Offline power inspector (SPEC PW) over captured channel-rate buffers, what the RMS tab's raw mode computes over a
 * capture: `batch` buffers of n samples, each integrated from an empty group with `integrate_samples` samples per
 * mean (0 is read as 1) -> means [batch][cap] as (mean, 0), counts [batch]; cap must be >= n / integrate_samples */
long sdb_task_power(const sdb_complex *src, size_t n, size_t batch, uint64_t integrate_samples, sdb_complex *means,
                    uint32_t *counts, size_t cap);

#ifdef __cplusplus
}
#endif
#endif
