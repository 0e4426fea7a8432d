/* analyzer/msg.h -- message payloads, the typed config bag and the analyzer params of the suscan-named shim.  Field
 * names are the ones the reference dereferences (SURVEY.md 8(b) "Struct fields dereferenced directly by callers"):
 * Suscan/Messages/PSDMessage.cpp:30-112, Suscan/Messages/InspectorMessage.cpp:28-252,
 * include/Suscan/Messages/SamplesMessage.h:33-59, Suscan/Messages/StatusMessage.cpp:33-45,
 * include/Suscan/Analyzer.h:113-254, include/Suscan/Config.h:36-76, Suscan/AnalyzerParams.cpp:27-68. */
#ifndef _SUSCAN_MSG_H
#define _SUSCAN_MSG_H
#include <sigutils/types.h>
#include <sigutils/softtune.h>
#include <analyzer/source/info.h>
#include <sys/time.h>
#ifdef __cplusplus
extern "C" {
#endif

/* released exactly once per payload, from any thread (Suscan/Message.cpp:43-48) */
void   suscan_analyzer_dispose_message(uint32_t type, void *ptr);

/* ---- message types (Suscan/Analyzer.cpp:75-98) */
#define SUSCAN_ANALYZER_MESSAGE_TYPE_SOURCE_INFO 0
#define SUSCAN_ANALYZER_MESSAGE_TYPE_SOURCE_INIT 1
#define SUSCAN_ANALYZER_MESSAGE_TYPE_CHANNEL     2
#define SUSCAN_ANALYZER_MESSAGE_TYPE_EOS         3
#define SUSCAN_ANALYZER_MESSAGE_TYPE_READ_ERROR  4
#define SUSCAN_ANALYZER_MESSAGE_TYPE_INTERNAL    5
#define SUSCAN_ANALYZER_MESSAGE_TYPE_SAMPLES     6
#define SUSCAN_ANALYZER_MESSAGE_TYPE_INSPECTOR   7
#define SUSCAN_ANALYZER_MESSAGE_TYPE_PSD         8
#define SUSCAN_ANALYZER_MESSAGE_TYPE_PARAMS      9
#define SUSCAN_WORKER_MSG_TYPE_HALT              0xffffffffu
#define SUSCAN_ANALYZER_INIT_FAILURE             (-1)
#define SUSCAN_ANALYZER_INIT_SUCCESS             0

enum suscan_analyzer_inspector_msgkind {
  SUSCAN_ANALYZER_INSPECTOR_MSGKIND_OPEN = 0,
  SUSCAN_ANALYZER_INSPECTOR_MSGKIND_SET_ID,
  SUSCAN_ANALYZER_INSPECTOR_MSGKIND_GET_CONFIG,
  SUSCAN_ANALYZER_INSPECTOR_MSGKIND_SET_CONFIG,
  SUSCAN_ANALYZER_INSPECTOR_MSGKIND_ESTIMATOR,
  SUSCAN_ANALYZER_INSPECTOR_MSGKIND_SPECTRUM,
  SUSCAN_ANALYZER_INSPECTOR_MSGKIND_CLOSE,
  SUSCAN_ANALYZER_INSPECTOR_MSGKIND_INVALID_CHANNEL,
  SUSCAN_ANALYZER_INSPECTOR_MSGKIND_WRONG_HANDLE,
  SUSCAN_ANALYZER_INSPECTOR_MSGKIND_WRONG_OBJECT,
  SUSCAN_ANALYZER_INSPECTOR_MSGKIND_WRONG_KIND,
  SUSCAN_ANALYZER_INSPECTOR_MSGKIND_SET_TLE,
  SUSCAN_ANALYZER_INSPECTOR_MSGKIND_ORBIT_REPORT
};

/* ---- struct sigutils_channel: <sigutils/softtune.h> */

/* ---- typed key / value bag (include/Suscan/Config.h:36-76, Suscan/Config.cpp:72-73) */
enum suscan_field_type {
  SUSCAN_FIELD_TYPE_STRING, SUSCAN_FIELD_TYPE_INTEGER, SUSCAN_FIELD_TYPE_FLOAT, SUSCAN_FIELD_TYPE_FILE,
  SUSCAN_FIELD_TYPE_BOOLEAN
};
struct suscan_field { enum suscan_field_type type; SUBOOL optional; char *name; char *desc; };
struct suscan_field_value {
  SUBOOL set;
  const struct suscan_field *field;
  union { uint64_t as_int; SUFLOAT as_float; SUBOOL as_bool; };
  char as_string[64];
};
typedef struct suscan_config_desc {
  char *global_name;
  struct suscan_field **field_list;
  unsigned int field_count;
} suscan_config_desc_t;
typedef struct suscan_config {
  const suscan_config_desc_t *desc;
  struct suscan_field_value **values;
} suscan_config_t;

suscan_config_t *suscan_config_new(const suscan_config_desc_t *desc);
suscan_config_t *suscan_config_dup(const suscan_config_t *config);
void             suscan_config_destroy(suscan_config_t *config);
struct suscan_field_value *suscan_config_get_value(const suscan_config_t *cfg, const char *name);
SUBOOL suscan_config_set_integer(suscan_config_t *cfg, const char *name, uint64_t value);
SUBOOL suscan_config_set_float(suscan_config_t *cfg, const char *name, SUFLOAT value);
SUBOOL suscan_config_set_bool(suscan_config_t *cfg, const char *name, SUBOOL value);
SUBOOL suscan_config_set_string(suscan_config_t *cfg, const char *name, const char *value);
SUBOOL suscan_config_desc_has_prefix(const suscan_config_desc_t *desc, const char *prefix);
SUBOOL suscan_config_str_to_bool(const char *str, SUBOOL deflt);
/* the bag of an inspector class ("psk", "fsk", "ask", "audio", "raw", "power") with its default values for a channel rate */
suscan_config_t *suscan_inspector_config_new(const char *class_name, SUFLOAT equiv_fs);

/* enum values of the config vocabulary (InspectorCtl/ClockRecovery.cpp:59-93, MfControl.cpp:56-78,
 * EqualizerControl.cpp:56-75) */
enum { SUSCAN_INSPECTOR_BAUDRATE_CONTROL_MANUAL = 0, SUSCAN_INSPECTOR_BAUDRATE_CONTROL_GARDNER = 1 };
enum { SUSCAN_INSPECTOR_MATCHED_FILTER_BYPASS = 0, SUSCAN_INSPECTOR_MATCHED_FILTER_MANUAL = 1 };
enum { SUSCAN_INSPECTOR_EQUALIZER_BYPASS = 0, SUSCAN_INSPECTOR_EQUALIZER_CMA = 1 };
enum { SUSCAN_INSPECTOR_CARRIER_CONTROL_MANUAL = 0, SUSCAN_INSPECTOR_CARRIER_CONTROL_COSTAS_2 = 1,
       SUSCAN_INSPECTOR_CARRIER_CONTROL_COSTAS_4 = 2, SUSCAN_INSPECTOR_CARRIER_CONTROL_COSTAS_8 = 3 };

/* ---- spectrum-source / estimator registries (looked up by name, InspectorMessage.cpp:46,55) */
struct suscan_spectsrc_class { const char *name; const char *desc; };
struct suscan_estimator_class { const char *name; const char *desc; const char *field; };
const struct suscan_spectsrc_class  *suscan_spectsrc_class_lookup(const char *name);
const struct suscan_estimator_class *suscan_estimator_class_lookup(const char *name);

/* ---- analyzer params (Suscan/AnalyzerParams.cpp:27-68, include/Suscan/AnalyzerParams.h:31-48) */
enum sigutils_channel_detector_window {
  SU_CHANNEL_DETECTOR_WINDOW_NONE = 0, SU_CHANNEL_DETECTOR_WINDOW_HAMMING, SU_CHANNEL_DETECTOR_WINDOW_HANN,
  SU_CHANNEL_DETECTOR_WINDOW_FLAT_TOP, SU_CHANNEL_DETECTOR_WINDOW_BLACKMANN_HARRIS
};
enum suscan_analyzer_mode { SUSCAN_ANALYZER_MODE_CHANNEL = 0, SUSCAN_ANALYZER_MODE_WIDE_SPECTRUM = 1 };
struct sigutils_channel_detector_params {
  SUSCOUNT samp_rate;
  SUSCOUNT window_size;
  SUFLOAT  fc;
  SUSCOUNT decimation;
  SUFLOAT  bw;
  SUSCOUNT max_order;
  SUBOOL   tune;
  enum sigutils_channel_detector_window window;
  SUFLOAT  alpha, beta, gamma, snr;
  SUSCOUNT max_age, pd_size;
  SUFLOAT  pd_thres, pd_signif;
};
struct suscan_analyzer_params {
  enum suscan_analyzer_mode mode;
  struct sigutils_channel_detector_params detector_params;
  SUFLOAT channel_update_int, psd_update_int;
  SUFREQ  min_freq, max_freq;
};
#define suscan_analyzer_params_INITIALIZER                                                                          \
  { SUSCAN_ANALYZER_MODE_CHANNEL,                                                                                   \
    { 8000, 8192, 0, 1, 0, 8, SU_TRUE, SU_CHANNEL_DETECTOR_WINDOW_BLACKMANN_HARRIS, 1e-2f, 1e-3f, .5f, 6, 40, 10,   \
      2, 10 },                                                                                                     \
    .1f, .04f, -1, -1 }

/* ---- message payloads */
struct suscan_analyzer_status_msg { int code; char *err_msg; const void *sender; };

struct suscan_analyzer_psd_msg {
  int64_t  fc;
  uint32_t inspector_id;
  struct timeval timestamp, rt_time;
  SUBOOL   looped;
  SUSCOUNT history_size;
  SUFLOAT  samp_rate, measured_samp_rate, N0;
  SUSCOUNT psd_size;
  SUFLOAT *psd_data;
};

struct suscan_analyzer_sample_batch_msg {
  uint32_t   inspector_id;
  SUCOMPLEX *samples;
  SUSCOUNT   sample_count;
  uint8_t   *symbols;        /* extension: hard decisions (the GUI's Decider output), same count; may be NULL */
};

struct suscan_orbit_report { struct timeval rx_time; SUFLOAT freq_corr; SUDOUBLE vlos_vel; };

struct suscan_analyzer_inspector_msg {
  enum suscan_analyzer_inspector_msgkind kind;
  uint32_t inspector_id, req_id;
  SUHANDLE handle;
  int      status;
  char    *class_name;
  struct sigutils_channel channel;
  suscan_config_t *config;
  SUBOOL   precise;
  unsigned int fs;
  SUFLOAT  equiv_fs, bandwidth, lo;
  SUHANDLE parent;
  char   **spectsrc_list;  unsigned int spectsrc_count;
  char   **estimator_list; unsigned int estimator_count;
  uint32_t estimator_id; SUBOOL enabled; SUFLOAT value;
  uint32_t spectsrc_id;
  SUFLOAT *spectrum_data; SUSCOUNT spectrum_size; SUSCOUNT samp_rate;
  SUFREQ   fc;
  SUFLOAT  N0;
  SUSCOUNT watermark;
  SUBOOL   tle_enable;
  struct suscan_orbit_report orbit_report;
  char    *signal_name; SUDOUBLE signal_value;
};

struct suscan_analyzer_channel_msg {
  const void *source;
  struct sigutils_channel **channel_list;
  unsigned int channel_count;
};

/* struct suscan_source_info: <analyzer/source/info.h> */
/* permissions (include/Suscan/Analyzer.h:113-123) */
#define SUSCAN_ANALYZER_PERM_HALT            (1ull << 0)
#define SUSCAN_ANALYZER_PERM_SET_FREQ        (1ull << 1)
#define SUSCAN_ANALYZER_PERM_SET_GAIN        (1ull << 2)
#define SUSCAN_ANALYZER_PERM_SET_ANTENNA     (1ull << 3)
#define SUSCAN_ANALYZER_PERM_SET_BW          (1ull << 4)
#define SUSCAN_ANALYZER_PERM_SET_PPM         (1ull << 5)
#define SUSCAN_ANALYZER_PERM_SET_DC_REMOVE   (1ull << 6)
#define SUSCAN_ANALYZER_PERM_SET_IQ_REVERSE  (1ull << 7)
#define SUSCAN_ANALYZER_PERM_SET_AGC         (1ull << 8)
#define SUSCAN_ANALYZER_PERM_OPEN_AUDIO      (1ull << 9)
#define SUSCAN_ANALYZER_PERM_OPEN_RAW        (1ull << 10)
#define SUSCAN_ANALYZER_PERM_OPEN_INSPECTOR  (1ull << 11)
#define SUSCAN_ANALYZER_PERM_SET_FFT_SIZE    (1ull << 12)
#define SUSCAN_ANALYZER_PERM_SET_FFT_FPS     (1ull << 13)
#define SUSCAN_ANALYZER_PERM_SET_FFT_WINDOW  (1ull << 14)
#define SUSCAN_ANALYZER_PERM_SEEK            (1ull << 15)
#define SUSCAN_ANALYZER_PERM_THROTTLE        (1ull << 16)
#define SUSCAN_ANALYZER_PERM_SET_BB_FILTER   (1ull << 17)
#define SUSCAN_ANALYZER_PERM_ALL             0xffffffffffffffffull

#ifdef __cplusplus
}
#endif
#endif
