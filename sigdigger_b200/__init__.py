"""sigdigger_b200 -- Python host mirror of the C-ABI in include/sigdigger_b200.h.

The product is libsigdigger_b200.so (hand-written CUDA for sm_90a + a C++ host runtime); this module
is a thin ctypes binding used by the tests and the benchmark.  It fails loudly when the native library
is missing or no CUDA device is present: there is no CPU path.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsigdigger_b200.so")

WINDOW = {"none": 0, "hamming": 1, "hann": 2, "flat_top": 3, "blackmann_harris": 4}
INSP = {"psk": 0, "fsk": 1, "ask": 2, "audio": 3, "raw": 4, "power": 5}
AUDIO = {"disabled": 0, "am": 1, "fm": 2, "usb": 3, "lsb": 4}
FLAG_PSD_SHIFT_DB = 1
FLAG_IQ_REVERSE = 2
FLAG_DC_REMOVE = 4
SPECTSRC = {"none": 0, "psd": 1, "cyclo": 2, "fmspect": 3, "timediff": 4, "abstimediff": 5, "exp_2": 6,
            "exp_4": 7, "exp_8": 8, "fac": 9}
ESTIMATOR = {"baud-fac": 0, "baud-nonlinear": 1}


class EngineParams(C.Structure):
    _fields_ = [("n_streams", C.c_uint32), ("psd_size", C.c_uint32), ("psd_window", C.c_int32),
                ("st_window_size", C.c_uint32), ("max_feed", C.c_uint32), ("device", C.c_int32),
                ("flags", C.c_uint32), ("input_format", C.c_int32), ("psd_average", C.c_uint32),
                ("psd_peak", C.c_uint32)]


FORMAT = {"f32": 0, "u8": 1, "s8": 2, "s16": 3}
FORMAT_DTYPE = {0: np.complex64, 1: np.uint8, 2: np.int8, 3: np.int16}


class DetectedChannel(C.Structure):
    """sdb_detected_channel (struct sigutils_channel)."""
    _fields_ = [("fc", C.c_double), ("f_lo", C.c_double), ("f_hi", C.c_double), ("bw", C.c_double),
                ("snr", C.c_float), ("S0", C.c_float), ("N0", C.c_float), ("bin_lo", C.c_uint32),
                ("bin_hi", C.c_uint32)]


class TrackedChannel(C.Structure):
    """sdb_tracked_channel: a detected channel followed across updates (oracle/SPEC_KT.md)."""
    _fields_ = [("fc", C.c_double), ("f_lo", C.c_double), ("f_hi", C.c_double), ("bw", C.c_double),
                ("snr", C.c_float), ("S0", C.c_float), ("N0", C.c_float), ("bin_lo", C.c_uint32),
                ("bin_hi", C.c_uint32), ("id", C.c_uint32), ("age", C.c_uint32), ("present", C.c_uint32),
                ("misses", C.c_uint32)]


class FacParams(C.Structure):
    """sdb_fac_params: the FAC tab of one inspector (oracle/SPEC_FC.md)."""
    _fields_ = [("size", C.c_uint32), ("alpha", C.c_float), ("lag_lo", C.c_uint32), ("lag_hi", C.c_uint32),
                ("sigma", C.c_double)]


class FacStatus(C.Structure):
    """sdb_fac_status: the FAC tab's outputs of one stream's latest feed."""
    _fields_ = [("blocks", C.c_uint32), ("peak_lag", C.c_uint32), ("max", C.c_float), ("min", C.c_float),
                ("sigmas", C.c_float), ("marker", C.c_int32)]


class SnrParams(C.Structure):
    """sdb_snr_params: the SNR meter of one inspector (oracle/SPEC_SN.md)."""
    _fields_ = [("bins", C.c_uint32), ("sigma", C.c_float), ("alpha", C.c_float)]


class SnrStatus(C.Structure):
    """sdb_snr_status: the SNR meter's state after one stream's latest feed."""
    _fields_ = [("counted", C.c_uint64), ("steps", C.c_uint32), ("stepped", C.c_uint32), ("sigma", C.c_float),
                ("snr", C.c_float), ("delta", C.c_float)]


class CaptureInfo(C.Structure):
    """sdb_capture_info"""
    _fields_ = [("container", C.c_int32), ("sample_format", C.c_int32), ("samp_rate", C.c_double),
                ("frequency", C.c_double), ("data_offset", C.c_uint64), ("n_samples", C.c_uint64),
                ("guessed", C.c_uint32), ("start_time", C.c_int64)]


CONTAINER = {"auto": -1, "raw": 0, "wav": 1, "sigmf": 2}


class Capture:
    """Capture file (raw / WAV / SigMF) mapped read-only; `.samples` is a numpy view in the native sample format
    (complex64, or interleaved I,Q of uint8 / int8 / int16).  Host-only: needs no GPU."""

    def __init__(self, path, container="auto", sample_format=None):
        self._L = load_library()
        self.info = CaptureInfo()
        fmt = -1 if sample_format is None else (FORMAT[sample_format] if isinstance(sample_format, str) else sample_format)
        self._h = self._L.sdb_capture_open(os.fsencode(path), CONTAINER[container], fmt, C.byref(self.info))
        if not self._h:
            raise SdbError((self._L.sdb_capture_last_error() or b"sdb_capture_open failed").decode())
        dt = FORMAT_DTYPE[self.info.sample_format]
        n = self.info.n_samples * (1 if dt is np.complex64 else 2)
        buf = (C.c_char * (n * np.dtype(dt).itemsize)).from_address(self._L.sdb_capture_data(self._h))
        self.samples = np.frombuffer(buf, dtype=dt, count=n)

    def close(self):
        if getattr(self, "_h", None):
            self.samples = None
            self._L.sdb_capture_close(self._h)
            self._h = None

    __del__ = close


class RecorderParams(C.Structure):
    """sdb_recorder_params"""
    _fields_ = [("container", C.c_int32), ("sample_format", C.c_int32), ("samp_rate", C.c_double),
                ("frequency", C.c_double), ("start_time", C.c_int64)]


AUDIO_DEMOD = {"am": 0, "fm": 1, "usb": 2, "lsb": 3, "raw": 4}
DATAVAR = {"decision_space": 0, "soft_bits": 1, "soft_bits_i": 2, "soft_bits_q": 3, "symbols": 4}


def _cap_err(L, what):
    return SdbError((L.sdb_capture_last_error() or what.encode()).decode())


class Recorder:
    """Capture writer (raw / WAV / SigMF; float32 / u8 / s8 / s16), or with `audio=` the mono PCM16 audio saver.
    Host-only.  write() takes complex64 blocks -- the body of the GUI's baseband-filter hook."""

    def __init__(self, path, samp_rate=0.0, frequency=0.0, container="raw", sample_format="f32", start_time=0,
                 auto_name=False, audio=None):
        self._L = L = load_library()
        if audio is not None:
            self._h = L.sdb_audio_recorder_open(os.fsencode(path), AUDIO_DEMOD[audio], frequency, int(samp_rate))
        else:
            p = RecorderParams(CONTAINER[container], FORMAT[sample_format], samp_rate, frequency, start_time)
            self._h = L.sdb_recorder_open(os.fsencode(path), int(auto_name), C.byref(p))
        if not self._h:
            raise _cap_err(L, "recorder open failed")
        self.path = os.fsdecode(L.sdb_recorder_path(self._h))

    def write(self, x):
        x = np.ascontiguousarray(x, dtype=np.complex64)
        n = self._L.sdb_recorder_write(self._h, x.ctypes.data, x.size)
        if n < 0:
            raise _cap_err(self._L, "write failed")
        return n

    @property
    def samples(self):
        return self._L.sdb_recorder_samples(self._h)

    def close(self):
        if getattr(self, "_h", None):
            h, self._h = self._h, None
            if self._L.sdb_recorder_close(h) != 0:
                raise _cap_err(self._L, "close failed")

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class AudioPlan(C.Structure):
    """sdb_audio_plan"""
    _fields_ = [("max_audio_bw", C.c_double), ("sample_rate", C.c_uint32), ("true_bw", C.c_double),
                ("true_lo", C.c_double), ("ch_fc", C.c_double), ("ch_ft", C.c_double), ("ch_bw", C.c_double),
                ("ch_f_lo", C.c_double), ("ch_f_hi", C.c_double)]


def audio_plan(analyzer_samp_rate, requested_rate, demod, lo, bw):
    """AudioProcessor's open / LO / bandwidth rules -> AudioPlan"""
    L = load_library()
    p = AudioPlan()
    d = AUDIO_DEMOD[demod] if isinstance(demod, str) else int(demod)
    if L.sdb_audio_plan_make(analyzer_samp_rate, int(requested_rate), d, lo, bw, C.byref(p)) != 0:
        raise _cap_err(L, "audio plan failed")
    return p


def audio_plan_config(plan, demod, cutoff, squelch=False, squelch_level=0.0, agc=True, agc_ts=0.2, fs=None):
    """AudioProcessor::setParams -> InspectorConfig of class "audio" """
    L = load_library()
    cfg = InspectorConfig()
    _check(L.sdb_inspector_config_default(C.byref(cfg), INSP["audio"], fs if fs is not None else plan.max_audio_bw))
    d = AUDIO_DEMOD[demod] if isinstance(demod, str) else int(demod)
    if L.sdb_audio_plan_config(C.byref(plan), d, cutoff, int(squelch), squelch_level, int(agc), agc_ts,
                               C.byref(cfg)) != 0:
        raise _cap_err(L, "audio config failed")
    return cfg


def capture_file_name(utc_seconds, samp_rate, frequency, sample_format="f32"):
    buf = C.create_string_buffer(128)
    L = load_library()
    if L.sdb_capture_file_name(buf, 128, int(utc_seconds), FORMAT[sample_format], samp_rate, frequency) < 0:
        raise _cap_err(L, "file name failed")
    return buf.value.decode()


def inspector_forward(data_var, soft, hard=None, decision_mode="argument"):
    """InspectorUI recording formats -> numpy array of what the data saver would receive"""
    L = load_library()
    soft = np.ascontiguousarray(soft, dtype=np.complex64)
    n = soft.size
    dv = DATAVAR[data_var]
    out = np.empty(n, np.complex64 if dv == 1 else np.uint8 if dv == 4 else np.float32)
    if hard is not None:
        hard = np.ascontiguousarray(hard, dtype=np.uint8)
    r = L.sdb_inspector_forward(dv, {"argument": 0, "modulus": 1}[decision_mode], soft.ctypes.data,
                                hard.ctypes.data if hard is not None else None, n, out.ctypes.data)
    if r < 0:
        raise _cap_err(L, "forward failed")
    assert r == out.nbytes
    return out


class ChannelDetector:
    """Stand-alone SPEC K detector on device-resident linear PSDs (e.g. a stitched SpectrumView)."""

    def __init__(self, n_bins, n_streams=1, alpha=0.01, gamma=0.5, snr=4.0, min_bins=2, device=0):
        self._L = load_library()
        self._h = self._L.sdb_chdet_new(device, n_bins, n_streams, alpha, gamma, snr, min_bins)
        if not self._h:
            raise RuntimeError("sdb_chdet_new failed (no CUDA device or bad parameters)")
        self.n_bins, self.n_streams = n_bins, n_streams

    def close(self):
        if self._h:
            self._L.sdb_chdet_destroy(self._h)
            self._h = None

    __del__ = close

    def feed(self, psd):
        """psd: CUDA float32 tensor [n_streams, frames, n_bins] (linear power, DC at index 0)."""
        assert psd.is_cuda and psd.dim() == 3 and psd.shape[0] == self.n_streams and psd.shape[2] == self.n_bins
        psd = psd.contiguous()
        _check(self._L.sdb_chdet_feed_device(self._h, psd.data_ptr(), psd.shape[1], psd.shape[1] * psd.shape[2]))

    def read(self, stream=0, samp_rate=1.0, center_freq=0.0, cap=256):
        out = (DetectedChannel * cap)()
        tot = C.c_uint32()
        n = _check(self._L.sdb_chdet_read(self._h, stream, samp_rate, center_freq, out, cap, C.byref(tot)))
        return [out[i] for i in range(n)], tot.value


class ChannelParams(C.Structure):
    _fields_ = [("f0", C.c_float), ("bw", C.c_float), ("guard", C.c_float), ("precise", C.c_int32)]


class ChannelInfo(C.Structure):
    _fields_ = [("center", C.c_uint32), ("size", C.c_uint32), ("width", C.c_uint32),
                ("decimation", C.c_float)]


class InspectorConfig(C.Structure):
    _fields_ = [("insp_class", C.c_int32), ("fs", C.c_float), ("agc_enabled", C.c_int32),
                ("agc_gain_db", C.c_float), ("costas_order", C.c_uint32), ("bits_per_symbol", C.c_uint32),
                ("loop_bw", C.c_float), ("offset", C.c_float), ("fsk_phase", C.c_float),
                ("fsk_quad_demod", C.c_int32), ("ask_use_pll", C.c_int32), ("ask_channel", C.c_uint32),
                ("mf_type", C.c_uint32), ("mf_rolloff", C.c_float), ("clock_type", C.c_uint32),
                ("baud", C.c_float), ("clock_gain", C.c_float), ("clock_phase", C.c_float),
                ("clock_running", C.c_int32), ("audio_cutoff", C.c_float), ("audio_volume", C.c_float),
                ("audio_squelch_level", C.c_float), ("agc_ts", C.c_float),
                ("audio_sample_rate", C.c_uint32), ("audio_demod", C.c_uint32), ("audio_squelch", C.c_int32),
                ("eq_type", C.c_uint32), ("eq_rate", C.c_float), ("eq_locked", C.c_int32),
                ("power_integrate_samples", C.c_uint64)]


_lib = None

_PROTOS = {
    "sdb_last_error": (C.c_char_p, []),
    "sdb_device_count": (C.c_int, []),
    "sdb_engine_new": (C.c_void_p, [C.c_void_p, C.c_double]),
    "sdb_engine_destroy": (None, [C.c_void_p]),
    "sdb_engine_open_channel": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "sdb_engine_set_inspector": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    "sdb_inspector_config_default": (C.c_int, [C.c_void_p, C.c_int, C.c_float]),
    "sdb_engine_commit": (C.c_int, [C.c_void_p]),
    "sdb_panoramic_unique_id": (C.c_int, [C.c_void_p]),
    "sdb_panoramic_new": (C.c_void_p, [C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "sdb_panoramic_destroy": (None, [C.c_void_p]),
    "sdb_panoramic_shard": (None, [C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "sdb_panoramic_sweep_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "sdb_panoramic_sweep_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "sdb_panoramic_reset": (C.c_int, [C.c_void_p]),
    "sdb_panoramic_size": (C.c_uint32, [C.c_void_p]),
    "sdb_panoramic_read": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "sdb_panoramic_read_channels": (C.c_long, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]),
    "sdb_panoramic_last_timing": (C.c_int, [C.c_void_p, C.c_void_p]),
    "sdb_panoramic_last_error": (C.c_char_p, []),
    "sdb_engine_read_all_channels": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "sdb_chdet_read_all": (C.c_int, [C.c_void_p, C.c_double, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "sdb_engine_migrate": (C.c_int, [C.c_void_p, C.c_void_p]),
    "sdb_engine_migrate_map": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "sdb_engine_same_geometry": (C.c_int, [C.c_void_p, C.c_void_p]),
    "sdb_channel_geometry": (C.c_int, [C.c_uint32, C.c_void_p, C.c_void_p]),
    "sdb_engine_feed_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t]),
    "sdb_engine_feed_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t]),
    "sdb_engine_sync": (C.c_int, [C.c_void_p]),
    "sdb_engine_join": (C.c_int, [C.c_void_p]),
    "sdb_engine_psd_frames": (C.c_size_t, [C.c_void_p]),
    "sdb_engine_psd_device": (C.c_void_p, [C.c_void_p]),
    "sdb_engine_read_psd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "sdb_engine_psd_average_frames": (C.c_size_t, [C.c_void_p]),
    "sdb_engine_psd_average_device": (C.c_void_p, [C.c_void_p]),
    "sdb_engine_read_psd_average": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "sdb_engine_psd_peak_groups": (C.c_size_t, [C.c_void_p]),
    "sdb_engine_psd_peak_device": (C.c_void_p, [C.c_void_p, C.c_int]),
    "sdb_engine_read_psd_peak": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "sdb_engine_read_channel": (C.c_long, [C.c_void_p, C.c_uint32, C.c_int, C.c_void_p, C.c_size_t]),
    "sdb_engine_read_symbols": (C.c_long, [C.c_void_p, C.c_uint32, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t]),
    "sdb_engine_read_all_symbols": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "sdb_engine_read_psd_async": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "sdb_engine_read_all_symbols_async": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "sdb_engine_read_symbols_packed_async": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                       C.c_size_t]),
    "sdb_engine_read_symbols_packed": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                 C.c_size_t]),
    "sdb_engine_symbol_counts_device": (C.c_void_p, [C.c_void_p]),
    "sdb_engine_symbol_capacity": (C.c_size_t, [C.c_void_p]),
    "sdb_spectsrc_name": (C.c_char_p, [C.c_int]),
    "sdb_estimator_name": (C.c_char_p, [C.c_int]),
    "sdb_engine_set_spectrum_source": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_uint32]),
    "sdb_engine_set_estimator": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int]),
    "sdb_engine_set_fac": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    "sdb_engine_read_fac": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "sdb_engine_fac_device": (C.c_void_p, [C.c_void_p, C.c_int]),
    "sdb_engine_set_snr": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    "sdb_engine_reset_snr": (C.c_int, [C.c_void_p, C.c_int, C.c_float]),
    "sdb_engine_read_snr": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sdb_engine_set_tv": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    "sdb_engine_set_tv_params": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    "sdb_engine_read_tv": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "sdb_engine_read_spectrum": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "sdb_engine_read_estimate": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "sdb_engine_set_spectrum_interval": (C.c_int, [C.c_void_p, C.c_int, C.c_uint64]),
    "sdb_engine_read_spectra": (C.c_long, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t]),
    "sdb_engine_read_estimates": (C.c_long, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t]),
    "sdb_engine_set_channel_detector": (C.c_int, [C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_float, C.c_uint32]),
    "sdb_engine_read_channels": (C.c_long, [C.c_void_p, C.c_uint32, C.c_double, C.c_void_p, C.c_size_t, C.c_void_p]),
    "sdb_engine_set_channel_tracking": (C.c_int, [C.c_void_p, C.c_uint32]),
    "sdb_engine_read_tracked_channels": (C.c_long, [C.c_void_p, C.c_uint32, C.c_double, C.c_void_p, C.c_size_t,
                                                    C.c_void_p, C.c_void_p]),
    "sdb_engine_read_all_tracked_channels": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                                        C.c_void_p]),
    "sdb_chdet_new": (C.c_void_p, [C.c_int, C.c_uint32, C.c_uint32, C.c_float, C.c_float, C.c_float, C.c_uint32]),
    "sdb_chdet_destroy": (None, [C.c_void_p]),
    "sdb_chdet_feed_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_size_t]),
    "sdb_chdet_read": (C.c_long, [C.c_void_p, C.c_uint32, C.c_double, C.c_double, C.c_void_p, C.c_size_t, C.c_void_p]),
    "sdb_capture_open": (C.c_void_p, [C.c_char_p, C.c_int32, C.c_int32, C.c_void_p]),
    "sdb_capture_data": (C.c_void_p, [C.c_void_p]),
    "sdb_capture_close": (None, [C.c_void_p]),
    "sdb_capture_last_error": (C.c_char_p, []),
    "sdb_engine_stream": (C.c_void_p, [C.c_void_p]),
    "sdb_engine_launch_count": (C.c_uint64, [C.c_void_p]),
    "sdb_engine_kernel_time": (C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(C.c_double), C.POINTER(C.c_uint64)]),
    "sdb_engine_timing": (None, [C.c_void_p, C.c_int]),
    "sdb_debug_stage_cycles": (C.c_int, [C.POINTER(C.c_uint64), C.c_int]),
    "sdb_debug_cta_cycles": (C.c_int, [C.POINTER(C.c_uint64), C.c_int]),
    "sdb_task_carrier_xlate": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_float, C.c_float]),
    "sdb_task_quad_demod": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t]),
    "sdb_task_costas": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_float, C.c_float]),
    "sdb_task_pll": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_float]),
    "sdb_task_agc": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_float]),
    "sdb_task_costas_state": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]),
    "sdb_task_pll_state": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_float, C.c_float, C.c_void_p]),
    "sdb_task_lpf": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_float]),
    "sdb_task_delayed_conj": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t]),
    "sdb_task_histogram_feed": (C.c_long, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int]),
    "sdb_task_sample_manual": (C.c_long, [C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_size_t, C.c_double,
                                          C.c_void_p]),
    "sdb_task_sample_zero_crossing": (C.c_int, [C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_int, C.c_float,
                                                C.c_float, C.c_float, C.c_float, C.c_float, C.c_void_p, C.c_void_p,
                                                C.c_size_t]),
    "sdb_task_carrier_detect": (C.c_int, [C.c_void_p, C.c_size_t, C.c_size_t, C.c_double, C.c_double, C.c_void_p]),
    "sdb_task_decide": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_uint, C.c_float, C.c_float]),
    "sdb_analyzer_new": (C.c_void_p, [C.c_void_p, C.c_void_p]),
    "sdb_analyzer_read": (C.c_void_p, [C.c_void_p, C.POINTER(C.c_uint32)]),
    "sdb_analyzer_read_timeout": (C.c_void_p, [C.c_void_p, C.POINTER(C.c_uint32), C.c_uint]),
    "sdb_analyzer_dispose_message": (None, [C.c_uint32, C.c_void_p]),
    "sdb_analyzer_req_halt": (None, [C.c_void_p]),
    "sdb_analyzer_destroy": (None, [C.c_void_p]),
    "sdb_analyzer_open_ex_async": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int, C.c_int32, C.c_uint32]),
    "sdb_analyzer_set_inspector_id_async": (C.c_int, [C.c_void_p, C.c_int32, C.c_uint32, C.c_uint32]),
    "sdb_analyzer_set_inspector_config_async": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_uint32]),
    "sdb_analyzer_close_async": (C.c_int, [C.c_void_p, C.c_int32, C.c_uint32]),
    "sdb_analyzer_set_params_async": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32]),
    "sdb_analyzer_set_inspector_watermark_async": (C.c_int, [C.c_void_p, C.c_int32, C.c_uint64, C.c_uint32]),
    "sdb_analyzer_set_inspector_freq_overridable": (C.c_int, [C.c_void_p, C.c_int32, C.c_double]),
    "sdb_analyzer_set_inspector_bandwidth_overridable": (C.c_int, [C.c_void_p, C.c_int32, C.c_double]),
    "sdb_analyzer_seek": (C.c_int, [C.c_void_p, C.c_void_p]),
    "sdb_analyzer_set_history_size": (C.c_int, [C.c_void_p, C.c_uint64]),
    "sdb_analyzer_replay": (C.c_int, [C.c_void_p, C.c_int]),
    "sdb_analyzer_set_hop_range": (C.c_int, [C.c_void_p, C.c_double, C.c_double]),
    "sdb_analyzer_set_rel_bandwidth": (C.c_int, [C.c_void_p, C.c_float]),
    "sdb_analyzer_set_buffering_size": (C.c_int, [C.c_void_p, C.c_uint64]),
    "sdb_analyzer_set_sweep_strategy": (C.c_int, [C.c_void_p, C.c_int]),
    "sdb_analyzer_set_spectrum_partitioning": (C.c_int, [C.c_void_p, C.c_int]),
    "sdb_analyzer_set_iq_reverse": (C.c_int, [C.c_void_p, C.c_int]),
    "sdb_analyzer_set_dc_remove": (C.c_int, [C.c_void_p, C.c_int]),
    "sdb_analyzer_register_baseband_filter_prio": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]),
    "sdb_analyzer_get_source_time": (C.c_double, [C.c_void_p]),
    "sdb_analyzer_get_inspector_config": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p]),
    "sdb_analyzer_set_throttle_async": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint32]),
    "sdb_analyzer_register_baseband_filter": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "sdb_analyzer_inspector_set_spectrum_async": (C.c_int, [C.c_void_p, C.c_int32, C.c_uint32, C.c_uint32]),
    "sdb_analyzer_inspector_set_fac_async": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_uint32]),
    "sdb_analyzer_inspector_set_snr_async": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_uint32]),
    "sdb_analyzer_inspector_reset_snr_async": (C.c_int, [C.c_void_p, C.c_int32, C.c_float, C.c_uint32]),
    "sdb_analyzer_inspector_set_tv_async": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_uint32]),
    "sdb_analyzer_inspector_estimator_cmd_async": (C.c_int, [C.c_void_p, C.c_int32, C.c_uint32, C.c_int, C.c_uint32]),
    "sdb_analyzer_get_samp_rate": (C.c_uint64, [C.c_void_p]),
    "sdb_analyzer_get_measured_samp_rate": (C.c_float, [C.c_void_p]),
    "sdb_sview_new": (C.c_void_p, [C.c_int]),
    "sdb_sview_destroy": (None, [C.c_void_p]),
    "sdb_sview_set_range": (C.c_int, [C.c_void_p, C.c_double, C.c_double, C.c_double, C.c_float]),
    "sdb_sview_reset": (C.c_int, [C.c_void_p]),
    "sdb_sview_size": (C.c_uint32, [C.c_void_p]),
    "sdb_sview_max_bins": (C.c_uint32, [C.c_void_p]),
    "sdb_sview_project": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int]),
    "sdb_recorder_open": (C.c_void_p, [C.c_char_p, C.c_int32, C.c_void_p]),
    "sdb_audio_recorder_open": (C.c_void_p, [C.c_char_p, C.c_int32, C.c_double, C.c_uint32]),
    "sdb_recorder_path": (C.c_char_p, [C.c_void_p]),
    "sdb_recorder_samples": (C.c_uint64, [C.c_void_p]),
    "sdb_recorder_write": (C.c_long, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "sdb_recorder_close": (C.c_int, [C.c_void_p]),
    "sdb_capture_file_name": (C.c_int, [C.c_char_p, C.c_size_t, C.c_int64, C.c_int32, C.c_double, C.c_double]),
    "sdb_audio_plan_make": (C.c_int, [C.c_double, C.c_uint32, C.c_int32, C.c_double, C.c_double, C.c_void_p]),
    "sdb_audio_plan_config": (C.c_int, [C.c_void_p, C.c_int32, C.c_float, C.c_int32, C.c_float, C.c_int32, C.c_float,
                                        C.c_void_p]),
    "sdb_inspector_forward": (C.c_long, [C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "sdb_psd_shift_db_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32]),
    "sdb_snr_estimator_new": (C.c_void_p, [C.c_uint32, C.c_uint32, C.c_int]),
    "sdb_snr_estimator_destroy": (None, [C.c_void_p]),
    "sdb_snr_estimator_set_bps": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32]),
    "sdb_snr_estimator_set_alpha": (C.c_int, [C.c_void_p, C.c_uint32, C.c_float]),
    "sdb_snr_estimator_set_sigma": (C.c_int, [C.c_void_p, C.c_uint32, C.c_float]),
    "sdb_snr_estimator_feed": (C.c_int, [C.c_void_p, C.c_void_p]),
    "sdb_snr_estimator_read": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sdb_averager_new": (C.c_void_p, [C.c_uint32, C.c_uint32, C.c_float, C.c_int]),
    "sdb_averager_destroy": (None, [C.c_void_p]),
    "sdb_averager_set_alpha": (C.c_int, [C.c_void_p, C.c_float]),
    "sdb_averager_reset": (C.c_int, [C.c_void_p]),
    "sdb_averager_feed_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t]),
    "sdb_averager_device": (C.c_void_p, [C.c_void_p]),
    "sdb_averager_read": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "sdb_decimator_new": (C.c_void_p, [C.c_int, C.c_uint32, C.c_uint32, C.c_int32, C.c_size_t]),
    "sdb_decimator_destroy": (None, [C.c_void_p]),
    "sdb_decimator_feed_device": (C.c_long, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t]),
    "sdb_decimator_feed_host": (C.c_long, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t]),
    "sdb_decimator_output_device": (C.c_void_p, [C.c_void_p]),
    "sdb_decimator_output_stride": (C.c_size_t, [C.c_void_p]),
    "sdb_decimator_stream": (C.c_void_p, [C.c_void_p]),
    "sdb_decimator_sync": (C.c_int, [C.c_void_p]),
    "sdb_decimator_read": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "sdb_decimator_reset": (C.c_int, [C.c_void_p]),
    "sdb_sview_contrib": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                    C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]),
    "sdb_sview_contrib_copy": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "sdb_sview_feed_view": (C.c_int, [C.c_void_p, C.c_void_p]),
    "sdb_sview_accumulate": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "sdb_sview_read": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "sdb_tv_params_pal": (None, [C.c_void_p, C.c_float]),
    "sdb_tv_params_ntsc": (None, [C.c_void_p, C.c_float]),
    "sdb_tv_processor_new": (C.c_void_p, [C.c_void_p, C.c_uint32, C.c_int]),
    "sdb_tv_processor_destroy": (None, [C.c_void_p]),
    "sdb_tv_processor_set_params": (C.c_int, [C.c_void_p, C.c_void_p]),
    "sdb_tv_processor_geometry": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "sdb_tv_processor_feed": (C.c_long, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p]),
    "sdb_tv_processor_feed_device": (C.c_long, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p]),
    "sdb_tv_processor_frames": (C.c_int, [C.c_void_p, C.c_void_p]),
    "sdb_tv_processor_read_frame": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p, C.c_size_t]),
    "sdb_tv_processor_estimates": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sdb_tv_feed_transform": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int, C.c_float, C.c_float, C.c_void_p]),
    "sdb_task_power": (C.c_long, [C.c_void_p, C.c_size_t, C.c_size_t, C.c_uint64, C.c_void_p, C.c_void_p,
                                  C.c_size_t]),
    "sdb_task_inspector": (C.c_long, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_size_t]),
}

EXPORTED_SYMBOLS = sorted(_PROTOS)


def load_library():
    """dlopen the native library and bind every symbol the header declares. No fallback."""
    global _lib
    if _lib is None:
        # SDB_LIB selects the instrumented twin (libsigdigger_b200_prof.so: per-role cycle counters compiled into
        # the inspector kernel); the product library is the default and the only one tests load
        path = os.environ.get("SDB_LIB") or LIB_PATH
        if not os.path.exists(path):
            raise RuntimeError("native library %s missing: run `python __graft_entry__.py` (build())" % path)
        L = C.CDLL(path)
        for name, (res, args) in _PROTOS.items():
            fn = getattr(L, name)      # AttributeError if the .so does not export it
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def last_error():
    return load_library().sdb_last_error().decode()


def device_count():
    return load_library().sdb_device_count()


def psd_shift_db(lin_ptr, db_ptr, n_frames, psd_size):
    """Device pass: linear PSD (DC first) -> PSDMessage layout (halves swapped, dB); out of place."""
    _check(load_library().sdb_psd_shift_db_device(lin_ptr, db_ptr, n_frames, psd_size))


class SdbError(RuntimeError):
    pass


def stage_cycles(reset=False):
    """Inspector-kernel role balance: busy cycles per role warp per processed chunk-sample (zeros unless the
    instrumented library is loaded, SDB_LIB=.../libsigdigger_b200_prof.so)."""
    buf = (C.c_uint64 * 8)()
    _check(load_library().sdb_debug_stage_cycles(buf, int(reset)))
    n = max(1, buf[4])
    return {"track": buf[0] / n, "pre": buf[5] / n, "post": buf[6] / n, "carrier": buf[1] / n, "filter": buf[2] / n,
            "clock": buf[3] / n, "chunk_samples": int(buf[4])}


def cta_cycles(reset=False):
    """Inspector CTAs by class since the last reset (instrumented library only): mean / longest lifetime in SM cycles
    and the time of the class's last CTA end after the kernel's first CTA start (ns)."""
    buf = (C.c_uint64 * 64)()
    _check(load_library().sdb_debug_cta_cycles(buf, int(reset)))
    names = ["psk", "fsk", "ask", "audio", "raw"]
    out = {}
    for c in range(5):
        if buf[5 + c]:
            out[names[c]] = {"ctas": int(buf[5 + c]), "mean_cycles": buf[c] / buf[5 + c], "max_cycles": int(buf[10 + c]),
                             "last_end_ns": int(buf[15 + c]) - int(buf[20])}
            r, ns = buf[24 + 8 * c:32 + 8 * c], max(1, buf[24 + 8 * c + 4])
            out[names[c]]["role_cycles_per_sample"] = {"track": round(r[0] / ns, 1), "pre": round(r[5] / ns, 1),
                                                       "post": round(r[6] / ns, 1), "carrier": round(r[1] / ns, 1),
                                                       "filter": round(r[2] / ns, 1), "clock": round(r[3] / ns, 1)}
    return out


def _check(rc):
    if rc is None or rc < 0:
        raise SdbError(last_error())
    return rc


def _is_torch(x):
    return type(x).__module__.startswith("torch")


class Engine:
    """Batch analyzer engine: main PSD + channeliser + inspectors over S streams on one GPU."""

    def __init__(self, n_streams=1, psd_size=65536, psd_window="blackmann_harris", st_window_size=0,
                 max_feed=0, samp_rate=1.0, device=0, flags=0, input_format="f32", psd_average=0, psd_peak=0):
        """psd_average: A >= 2 also emits the mean of every A PSD frames (SPEC A, read_psd_average); 0 or 1 = off.
        psd_peak: P >= 2 also emits the per-bin maximum and minimum of every P PSD frames (SPEC PK, read_psd_peak)."""
        L = load_library()
        self.input_format = FORMAT[input_format] if isinstance(input_format, str) else int(input_format)
        p = EngineParams(n_streams, psd_size, WINDOW[psd_window] if isinstance(psd_window, str) else psd_window,
                         st_window_size, max_feed, device, flags, self.input_format, psd_average, psd_peak)
        self._L = L
        self.n_streams, self.psd_size, self.samp_rate = n_streams, psd_size, samp_rate
        self.st_window_size = st_window_size or psd_size
        self.device, self.max_feed = device, max_feed
        self._h = L.sdb_engine_new(C.byref(p), samp_rate)
        if not self._h:
            raise SdbError(last_error())
        self._info = []
        self._fac_size = {}                 # FAC block size of every channel with the FAC on (set_fac)
        self._snr_bins = {}                 # histogram bins of every channel with the SNR meter on (set_snr)
        self._bps = {}                      # bits_per_symbol of every channel's inspector (set_inspector)
        self._baud = {}                     # baud of every channel's inspector (set_inspector)

    def close(self):
        if getattr(self, "_h", None):
            self._L.sdb_engine_destroy(self._h)
            self._h = None

    __del__ = close

    def open_channel(self, f0, bw, guard=1.0, precise=False):
        info = ChannelInfo()
        p = ChannelParams(f0, bw, guard, int(precise))
        h = _check(self._L.sdb_engine_open_channel(self._h, C.byref(p), C.byref(info)))
        self._info.append(info)
        return h

    def channel_info(self, h):
        return self._info[h]

    def channel_rate(self, h):
        return self.samp_rate * self._info[h].size / self.st_window_size

    def set_inspector(self, h, cls, **kw):
        cfg = InspectorConfig()
        _check(self._L.sdb_inspector_config_default(C.byref(cfg), INSP[cls], self.channel_rate(h)))
        for k, v in kw.items():
            if not hasattr(cfg, k):
                raise KeyError(k)
            setattr(cfg, k, v)
        _check(self._L.sdb_engine_set_inspector(self._h, h, C.byref(cfg)))
        self._bps[h] = cfg.bits_per_symbol
        self._baud[h] = cfg.baud

    def commit(self):
        _check(self._L.sdb_engine_commit(self._h))

    def feed(self, x, sync=True):
        """x: [S, n] complex64 numpy array (host path, copies H2D) or torch cuda tensor (device path)."""
        if _is_torch(x):
            assert x.is_cuda and x.dim() == 2 and x.shape[0] == self.n_streams
            assert x.stride(1) == 1
            _check(self._L.sdb_engine_feed_device(self._h, x.data_ptr(), x.stride(0), x.shape[1]))
        elif self.input_format == 0:
            x = np.ascontiguousarray(x, dtype=np.complex64)
            assert x.ndim == 2 and x.shape[0] == self.n_streams
            self._keep = x
            _check(self._L.sdb_engine_feed_host(self._h, x.ctypes.data, x.shape[1], x.shape[1]))
        else:
            # native SDR format: [S, n, 2] interleaved I, Q of dtype uint8 / int8 / int16
            x = np.ascontiguousarray(x, dtype=FORMAT_DTYPE[self.input_format])
            assert x.ndim == 3 and x.shape[0] == self.n_streams and x.shape[2] == 2
            self._keep = x
            _check(self._L.sdb_engine_feed_host(self._h, x.ctypes.data, x.shape[1], x.shape[1]))
        if sync:
            self.sync()

    def feed_host_ptr(self, ptr, stride, n):
        _check(self._L.sdb_engine_feed_host(self._h, ptr, stride, n))

    def feed_device_ptr(self, ptr, stride, n):
        _check(self._L.sdb_engine_feed_device(self._h, ptr, stride, n))

    def sync(self):
        _check(self._L.sdb_engine_sync(self._h))

    def join(self):
        _check(self._L.sdb_engine_join(self._h))

    def read_psd(self, out=None):
        f = self._L.sdb_engine_psd_frames(self._h)
        if out is None:
            out = np.empty((self.n_streams, f, self.psd_size), np.float32)
        _check(self._L.sdb_engine_read_psd(self._h, out.ctypes.data, out.size))
        return out

    def read_psd_average(self, out=None):
        """-> [n_streams, means, psd_size] float32: the group means the last feed completed (SPEC A)"""
        m = self._L.sdb_engine_psd_average_frames(self._h)
        if out is None:
            out = np.empty((self.n_streams, m, self.psd_size), np.float32)
        _check(self._L.sdb_engine_read_psd_average(self._h, out.ctypes.data, out.size))
        return out

    @property
    def psd_average_frames(self):
        return self._L.sdb_engine_psd_average_frames(self._h)

    @property
    def psd_average_device_ptr(self):
        return self._L.sdb_engine_psd_average_device(self._h)

    def read_psd_peak(self):
        """-> (max, min), each [n_streams, groups, psd_size] float32: the group extremes the last feed completed
        (SPEC PK)"""
        g = self._L.sdb_engine_psd_peak_groups(self._h)
        mx = np.empty((self.n_streams, g, self.psd_size), np.float32)
        mn = np.empty_like(mx)
        _check(self._L.sdb_engine_read_psd_peak(self._h, mx.ctypes.data, mn.ctypes.data, mx.size))
        return mx, mn

    def psd_peak_groups(self):
        """groups per stream the last feed completed (0 when peak detection is off)"""
        return self._L.sdb_engine_psd_peak_groups(self._h)

    def psd_peak_device_ptr(self, which):
        """device address of the maxima (which = 0) or the minima (which = 1) of the last feed"""
        return self._L.sdb_engine_psd_peak_device(self._h, which)

    # ---- channel detector (SPEC K; detector_params of Suscan/AnalyzerParams.cpp:27-66)
    def set_channel_detector(self, alpha=0.01, beta=0.01, gamma=0.5, snr=4.0, min_bins=2):
        _check(self._L.sdb_engine_set_channel_detector(self._h, alpha, beta, gamma, snr, min_bins))

    def read_channels(self, stream, center_freq=0.0, cap=256):
        """-> (structured array of DetectedChannel fields, total found before the cap)"""
        out = (DetectedChannel * cap)()
        tot = C.c_uint32()
        n = _check(self._L.sdb_engine_read_channels(self._h, stream, center_freq, out, cap, C.byref(tot)))
        return [out[i] for i in range(n)], tot.value

    # ---- channel tracking across detector updates (oracle/SPEC_KT.md): before commit, after set_channel_detector
    def set_channel_tracking(self, hold):
        """follow detected channels across updates; a channel no update detects is kept for `hold` more updates"""
        _check(self._L.sdb_engine_set_channel_tracking(self._h, hold))

    def read_tracked_channels(self, stream, center_freq=0.0, cap=256):
        """-> (list of TrackedChannel in ascending (bin_lo, id), live tracks before the cap, detections dropped at
        the 256-track cap since commit)"""
        out = (TrackedChannel * cap)()
        tot, dropped = C.c_uint32(), C.c_uint64()
        n = _check(self._L.sdb_engine_read_tracked_channels(self._h, stream, center_freq, out, cap, C.byref(tot),
                                                            C.byref(dropped)))
        return [out[i] for i in range(n)], tot.value, dropped.value

    def read_all_tracked_channels(self, centers, cap=256):
        """-> per stream (list of TrackedChannel, dropped), from one read of every stream"""
        S = len(centers)
        c = (C.c_double * S)(*centers)
        out = (TrackedChannel * (S * cap))()
        counts, dropped = (C.c_uint32 * S)(), (C.c_uint64 * S)()
        _check(self._L.sdb_engine_read_all_tracked_channels(self._h, c, out, cap, counts, dropped))
        return [([out[s * cap + i] for i in range(counts[s])], dropped[s]) for s in range(S)]

    # ---- the inspector's FAC tab (oracle/SPEC_FC.md): before commit, after set_inspector
    def set_fac(self, h, size=65536, alpha=1.0, lags=None, sigma=5.0, enabled=True):
        """Autocorrelate h's soft symbols in blocks of `size`, averaged with `alpha` (1 - slider / 100), with the peak
        of the lag window `lags` = (lo, hi) (None: [0, size / 2)) marked above `sigma`; enabled=False turns it off."""
        if not enabled:
            _check(self._L.sdb_engine_set_fac(self._h, h, None))
            self._fac_size.pop(h, None)
            return
        lo, hi = lags if lags is not None else (0, 0)
        p = FacParams(size, alpha, lo, hi, sigma)
        _check(self._L.sdb_engine_set_fac(self._h, h, C.byref(p)))
        self._fac_size[h] = size

    def read_fac(self, h):
        """-> (fac [n_streams, size / 2] float32, list of FacStatus per stream) after the latest feed"""
        if h not in self._fac_size:
            _check(self._L.sdb_engine_read_fac(self._h, h, None, None))      # the engine's refusal and its message
            raise SdbError("the FAC is not enabled on this channel")
        size = self._fac_size[h]
        out = np.zeros((self.n_streams, size // 2), np.float32)
        st = (FacStatus * self.n_streams)()
        _check(self._L.sdb_engine_read_fac(self._h, h, out.ctypes.data, st))
        return out, list(st)

    # ---- the inspector's SNR meter (oracle/SPEC_SN.md): before commit, after set_inspector
    def set_snr(self, h, bins=256, sigma=1.0, alpha=None, enabled=True):
        """Bin h's soft symbols into a `bins`-bin decision-space histogram and fit the comb model to it once per feed,
        starting from `sigma`, with step `alpha` (None: 1 / 2^bits_per_symbol, the GUI's toggle); enabled=False: off"""
        if not enabled:
            _check(self._L.sdb_engine_set_snr(self._h, h, None))
            self._snr_bins.pop(h, None)
            return
        if alpha is None:
            alpha = 1.0 / (1 << (self._bps.get(h, 1) or 1))
        p = SnrParams(bins, sigma, alpha)
        _check(self._L.sdb_engine_set_snr(self._h, h, C.byref(p)))
        self._snr_bins[h] = bins

    def reset_snr(self, h, sigma=1.0):
        """sigma of every stream from the next feed on; the histogram is kept"""
        _check(self._L.sdb_engine_reset_snr(self._h, h, sigma))

    def read_snr(self, h):
        """-> (hist [n_streams, bins] uint32, model [n_streams, bins] float32, list of SnrStatus per stream)"""
        if h not in self._snr_bins:
            _check(self._L.sdb_engine_read_snr(self._h, h, None, None, None))   # the engine's refusal and its message
            raise SdbError("the SNR meter is not on for this channel")
        L = self._snr_bins[h]
        hist = np.zeros((self.n_streams, L), np.uint32)
        model = np.zeros((self.n_streams, L), np.float32)
        st = (SnrStatus * self.n_streams)()
        _check(self._L.sdb_engine_read_snr(self._h, h, hist.ctypes.data, model.ctypes.data, st))
        return hist, model, list(st)

    # ---- the inspector's Analog TV tab (oracle/SPEC_TI.md): before commit, after set_inspector
    def set_tv(self, h, params=None, invert=False, dc=0.0, enabled=True):
        """Run a TV processor over h's soft symbols in every stream (k |x| + dc for ask, k arg(x) / pi + dc for psk and
        fsk, k = -1 with invert); params: a tv_params(...) block, None: PAL at the inspector's symbol rate (one sample
        per symbol); dc: the tab's DC value / 100; enabled=False: off"""
        if not enabled:
            _check(self._L.sdb_engine_set_tv(self._h, h, None))
            return
        _check(self._L.sdb_engine_set_tv(self._h, h, C.byref(self._tv_tab(h, params, invert, dc))))

    def set_tv_params(self, h, params=None, invert=False, dc=0.0):
        """between feeds, from the next feed on; the picture geometry must stay (else a new plan is needed)"""
        _check(self._L.sdb_engine_set_tv_params(self._h, h, C.byref(self._tv_tab(h, params, invert, dc))))

    def _tv_tab(self, h, params, invert, dc):
        if params is None:
            params = tv_params("pal", self._baud[h])
        return TvTabParams(params, int(bool(invert)), dc)

    def read_tv(self, h):
        """-> (frames [n_streams, H, W] float32: each stream's posted frame, valid where completed > 0, list of TvStatus
        per stream) after the latest feed"""
        st = (TvStatus * self.n_streams)()
        _check(self._L.sdb_engine_read_tv(self._h, h, None, st))
        frames = np.zeros((self.n_streams, st[0].height, st[0].width), np.float32)
        _check(self._L.sdb_engine_read_tv(self._h, h, frames.ctypes.data, None))
        return frames, list(st)

    # ---- inspector spectrum sources / estimators (SPEC U; Suscan/Analyzer.cpp:539-565)
    def set_spectrum_source(self, h, kind, size=1024):
        k = SPECTSRC[kind] if isinstance(kind, str) else int(kind)
        _check(self._L.sdb_engine_set_spectrum_source(self._h, h, k, size))
        self._spect_size = getattr(self, "_spect_size", {})
        self._spect_size[h] = size
        self._spect_kind = getattr(self, "_spect_kind", {})
        self._spect_kind[h] = k

    def set_estimator(self, h, estimator, enabled=True):
        e = ESTIMATOR[estimator] if isinstance(estimator, str) else int(estimator)
        _check(self._L.sdb_engine_set_estimator(self._h, h, e, int(enabled)))

    def read_spectrum(self, h):
        """-> (spectra [n_streams, size] float32, sizes [n_streams] uint32: floats emitted per stream)"""
        size = self._spect_size[h]
        out = np.zeros((self.n_streams, size), np.float32)
        sizes = np.zeros(self.n_streams, np.uint32)
        _check(self._L.sdb_engine_read_spectrum(self._h, h, out.ctypes.data, sizes.ctypes.data))
        return out, sizes

    def read_estimate(self, h, estimator):
        e = ESTIMATOR[estimator] if isinstance(estimator, str) else int(estimator)
        vals = np.zeros(self.n_streams, np.float32)
        valid = np.zeros(self.n_streams, np.int32)
        _check(self._L.sdb_engine_read_estimate(self._h, h, e, vals.ctypes.data, valid.ctypes.data))
        return vals, valid

    def set_spectrum_interval(self, h, interval):
        """Emit h's spectrum and estimates every `interval` channel samples, from a window carried across feeds
        (SPEC US); 0 = once per feed (SPEC U.1).  Before commit."""
        _check(self._L.sdb_engine_set_spectrum_interval(self._h, h, int(interval)))
        self._spect_interval = getattr(self, "_spect_interval", {})
        self._spect_interval[h] = int(interval)

    def _emits_cap(self, h):
        # ceil(channel samples per max_feed / I): what one feed can emit
        n_max = (self.max_feed // (self.st_window_size // 2)) * (self.channel_info(h).size // 2)
        return -(-n_max // self._spect_interval[h])

    def read_spectra(self, h):
        """-> (spectra [n_streams, emissions, out_size] float32, ends [emissions] uint64: t_j of each): every emission
        of the last feed on a scheduled channel (SPEC US); out_size = size, or size / 2 for "fac"."""
        cap = self._emits_cap(h)
        size = getattr(self, "_spect_size", {}).get(h, 1024)
        w = size // 2 if getattr(self, "_spect_kind", {}).get(h) == SPECTSRC["fac"] else size
        out = np.zeros((self.n_streams, cap, w), np.float32)
        ends = np.zeros(cap, np.uint64)
        n = _check(self._L.sdb_engine_read_spectra(self._h, h, out.ctypes.data, ends.ctypes.data, cap))
        return out[:, :n].copy(), ends[:n].copy()

    def read_estimates(self, h, estimator):
        """-> (values [n_streams, emissions] float32, valid [n_streams, emissions] int32) of the last feed (SPEC US)"""
        e = ESTIMATOR[estimator] if isinstance(estimator, str) else int(estimator)
        cap = self._emits_cap(h)
        vals = np.zeros((self.n_streams, cap), np.float32)
        valid = np.zeros((self.n_streams, cap), np.int32)
        n = _check(self._L.sdb_engine_read_estimates(self._h, h, e, vals.ctypes.data, valid.ctypes.data, cap))
        return vals[:, :n].copy(), valid[:, :n].copy()

    def read_channel(self, stream, h, cap=None):
        cap = cap or (1 << 24)
        out = np.empty(cap, np.complex64)
        n = _check(self._L.sdb_engine_read_channel(self._h, stream, h, out.ctypes.data, cap))
        return out[:n].copy()

    def read_symbols(self, stream, h):
        cap = self._L.sdb_engine_symbol_capacity(self._h)
        soft = np.empty(cap, np.complex64)
        hard = np.empty(cap, np.uint8)
        n = _check(self._L.sdb_engine_read_symbols(self._h, stream, h, soft.ctypes.data, hard.ctypes.data, cap))
        return soft[:n].copy(), hard[:n].copy()

    def read_psd_async(self, out):
        _check(self._L.sdb_engine_read_psd_async(self._h, out.ctypes.data, out.size))

    def read_all_symbols_async(self, counts, soft, hard, cap):
        _check(self._L.sdb_engine_read_all_symbols_async(self._h, counts.ctypes.data,
                                                         soft.ctypes.data if soft is not None else None,
                                                         hard.ctypes.data if hard is not None else None, cap))

    def read_symbols_packed_async(self, counts, offsets, soft, hard, cap_total):
        """soft / hard: pinned host arrays (or device pointers as ints); the GPU writes them directly"""
        ptr = lambda a: None if a is None else (a if isinstance(a, int) else a.ctypes.data)
        _check(self._L.sdb_engine_read_symbols_packed_async(self._h, counts.ctypes.data, offsets.ctypes.data,
                                                            ptr(soft), ptr(hard), cap_total))

    def read_symbols_packed(self, counts, offsets, soft, hard, cap_total):
        ptr = lambda a: None if a is None else (a if isinstance(a, int) else a.ctypes.data)
        _check(self._L.sdb_engine_read_symbols_packed(self._h, counts.ctypes.data, offsets.ctypes.data,
                                                      ptr(soft), ptr(hard), cap_total))

    def read_all_symbols(self, counts, soft, hard, cap):
        _check(self._L.sdb_engine_read_all_symbols(self._h, counts.ctypes.data,
                                                   soft.ctypes.data if soft is not None else None,
                                                   hard.ctypes.data if hard is not None else None, cap))

    @property
    def symbol_capacity(self):
        return self._L.sdb_engine_symbol_capacity(self._h)

    @property
    def psd_device_ptr(self):
        return self._L.sdb_engine_psd_device(self._h)

    @property
    def stream_ptr(self):
        return self._L.sdb_engine_stream(self._h)

    @property
    def launches(self):
        return self._L.sdb_engine_launch_count(self._h)

    def timing(self, enable=True):
        self._L.sdb_engine_timing(self._h, int(enable))

    def kernel_time(self, family):
        ms, n = C.c_double(), C.c_uint64()
        _check(self._L.sdb_engine_kernel_time(self._h, family.encode(), C.byref(ms), C.byref(n)))
        return ms.value, n.value


def _task(fn, x, *args):
    x = np.ascontiguousarray(x, dtype=np.complex64)
    batch = 1 if x.ndim == 1 else x.shape[0]
    n = x.shape[-1]
    out = np.empty_like(x)
    _check(fn(x.ctypes.data, out.ctypes.data, n, batch, *args))
    return out


def carrier_xlate(x, rel_freq, phase=0.0):
    """Tasks/CarrierXlator.cpp"""
    return _task(load_library().sdb_task_carrier_xlate, x, rel_freq, phase)


def quad_demod(x):
    """Tasks/QuadDemodTask.cpp"""
    return _task(load_library().sdb_task_quad_demod, x)


def costas(x, kind, tau, loop_bw):
    """Tasks/CostasRecoveryTask.cpp"""
    return _task(load_library().sdb_task_costas, x, kind, tau, loop_bw)


def pll(x, bw):
    """Tasks/PLLSyncTask.cpp"""
    return _task(load_library().sdb_task_pll, x, bw)


def agc(x, tau):
    """Tasks/AGCTask.cpp"""
    return _task(load_library().sdb_task_agc, x, tau)


def lpf(x, bw):
    """Tasks/LPFTask.cpp"""
    return _task(load_library().sdb_task_lpf, x, bw)


SPACE = {"amplitude": 0, "phase": 1, "frequency": 2}


def _batch(x):
    x = np.ascontiguousarray(x, dtype=np.complex64)
    return (x[None, :], True) if x.ndim == 1 else (x, False)


def delayed_conj(x, delay):
    """Tasks/DelayedConjTask.cpp"""
    return _task(load_library().sdb_task_delayed_conj, x, delay)


def histogram_feed(x, space):
    """Tasks/HistogramFeeder.cpp -> float32 [batch, n] (n - 1 for "frequency")"""
    x, one = _batch(x)
    sp = SPACE[space] if isinstance(space, str) else int(space)
    out = np.empty((x.shape[0], x.shape[1] - (1 if sp == 2 else 0)), np.float32)
    _check(load_library().sdb_task_histogram_feed(x.ctypes.data, out.ctypes.data, x.shape[1], x.shape[0], sp))
    return out[0] if one else out


def sample_manual(x, space, symbol_count, symbol_sync=0):
    """Tasks/WaveSampler.cpp sampleManual -> complex64 [batch, int(symbol_count)]"""
    x, one = _batch(x)
    sp = SPACE[space] if isinstance(space, str) else int(space)
    out = np.empty((x.shape[0], int(symbol_count)), np.complex64)
    _check(load_library().sdb_task_sample_manual(x.ctypes.data, x.shape[1], x.shape[0], sp, symbol_sync,
                                                 float(symbol_count), out.ctypes.data))
    return out[0] if one else out


def sample_zero_crossing(x, space, bnor, amplitude=False, threshold=0j, zc_angle=1 + 0j, cap=None):
    """Tasks/WaveSampler.cpp sampleZeroCrossing -> list of uint8 bit arrays (one per buffer)"""
    x, one = _batch(x)
    sp = SPACE[space] if isinstance(space, str) else int(space)
    cap = cap or x.shape[1]
    sym = np.empty((x.shape[0], cap), np.uint8)
    cnt = np.zeros(x.shape[0], np.uint32)
    t, z = complex(threshold), complex(zc_angle)
    _check(load_library().sdb_task_sample_zero_crossing(x.ctypes.data, x.shape[1], x.shape[0], sp, int(amplitude),
                                                        t.real, t.imag, z.real, z.imag, bnor, sym.ctypes.data,
                                                        cnt.ctypes.data, cap))
    res = [sym[b, :min(int(cnt[b]), cap)].copy() for b in range(x.shape[0])]
    return (res[0], int(cnt[0])) if one else (res, cnt)


def carrier_detect(x, avg_rel_bw=0.01, dc_notch_rel_bw=0.0):
    """Tasks/CarrierDetector.cpp -> carrier offset(s) in rad / sample"""
    x, one = _batch(x)
    peak = np.empty(x.shape[0], np.float32)
    _check(load_library().sdb_task_carrier_detect(x.ctypes.data, x.shape[1], x.shape[0], avg_rel_bw, dc_notch_rel_bw,
                                                  peak.ctypes.data))
    return float(peak[0]) if one else peak


def decide(soft, mode, bps, vmin, vmax):
    """Decider (SPEC D): mode "argument" / "modulus" -> uint8 symbols"""
    soft = np.ascontiguousarray(soft, dtype=np.complex64).ravel()
    sym = np.empty(soft.size, np.uint8)
    m = {"argument": 0, "modulus": 1}[mode] if isinstance(mode, str) else int(mode)
    _check(load_library().sdb_task_decide(soft.ctypes.data, sym.ctypes.data, soft.size, m, bps, vmin, vmax))
    return sym


def inspector_run(cls, fs, x, **kw):
    """Offline inspector over captured channel-rate buffers x [batch, n] -> list of (soft, hard)."""
    L = load_library()
    x = np.ascontiguousarray(x, dtype=np.complex64)
    if x.ndim == 1:
        x = x[None, :]
    batch, n = x.shape
    cfg = InspectorConfig()
    _check(L.sdb_inspector_config_default(C.byref(cfg), INSP[cls], fs))
    for k, v in kw.items():
        if not hasattr(cfg, k):
            raise KeyError(k)
        setattr(cfg, k, v)
    cap = n
    soft = np.empty((batch, cap), np.complex64)
    hard = np.empty((batch, cap), np.uint8)
    counts = np.zeros(batch, np.uint32)
    _check(L.sdb_task_inspector(C.byref(cfg), x.ctypes.data, n, batch, soft.ctypes.data, hard.ctypes.data,
                                counts.ctypes.data, cap))
    return [(soft[b, :counts[b]].copy(), hard[b, :counts[b]].copy()) for b in range(batch)]


def task_power(x, integrate_samples):
    """Offline power inspector (SPEC PW) over captured channel-rate buffers: x [n] or [batch, n] complex64 ->
    one complex64 array of (mean, 0) samples per buffer, each buffer integrated from an empty group."""
    L = load_library()
    x = np.ascontiguousarray(x, dtype=np.complex64)
    if x.ndim == 1:
        x = x[None, :]
    batch, n = x.shape
    cap = max(1, n // max(1, integrate_samples))
    means = np.empty((batch, cap), np.complex64)
    counts = np.zeros(batch, np.uint32)
    _check(L.sdb_task_power(x.ctypes.data, n, batch, integrate_samples, means.ctypes.data, counts.ctypes.data, cap))
    return [means[b, :counts[b]].copy() for b in range(batch)]


class SnrEstimator:
    """Batch of the inspector tab's SNR estimators (Misc/SNREstimator.cpp) on decision-space histograms."""

    def __init__(self, n_estimators, length, device=0):
        self._L = load_library()
        self.n, self.length = n_estimators, length
        self._h = self._L.sdb_snr_estimator_new(n_estimators, length, device)
        if not self._h:
            raise SdbError(last_error())

    def close(self):
        if getattr(self, "_h", None):
            self._L.sdb_snr_estimator_destroy(self._h)
            self._h = None

    __del__ = close

    def set_bps(self, index, bps):
        _check(self._L.sdb_snr_estimator_set_bps(self._h, index, bps))

    def set_alpha(self, index, alpha):
        _check(self._L.sdb_snr_estimator_set_alpha(self._h, index, alpha))

    def set_sigma(self, index, sigma):
        _check(self._L.sdb_snr_estimator_set_sigma(self._h, index, sigma))

    def feed(self, histories):
        h = np.ascontiguousarray(histories, dtype=np.uint32)
        assert h.shape == (self.n, self.length)
        _check(self._L.sdb_snr_estimator_feed(self._h, h.ctypes.data))

    def read(self, model=False):
        sigma, snr = np.empty(self.n, np.float32), np.empty(self.n, np.float32)
        m = np.empty((self.n, self.length), np.float32) if model else None
        _check(self._L.sdb_snr_estimator_read(self._h, sigma.ctypes.data, snr.ctypes.data,
                                              m.ctypes.data if model else None))
        return (sigma, snr, m) if model else (sigma, snr)


class Averager:
    """Spectrum averager (Misc/Averager.cpp) over device PSD frames, one state row per stream."""

    def __init__(self, psd_size, n_streams=1, alpha=1.0, device=0):
        self._L = load_library()
        self.psd_size, self.n_streams = psd_size, n_streams
        self._h = self._L.sdb_averager_new(psd_size, n_streams, alpha, device)
        if not self._h:
            raise SdbError(last_error())

    def close(self):
        if getattr(self, "_h", None):
            self._L.sdb_averager_destroy(self._h)
            self._h = None

    __del__ = close

    def set_alpha(self, alpha):
        _check(self._L.sdb_averager_set_alpha(self._h, alpha))

    def reset(self):
        _check(self._L.sdb_averager_reset(self._h))

    def feed_ptr(self, psd_ptr, frames, stream_stride=None):
        _check(self._L.sdb_averager_feed_device(self._h, psd_ptr, frames,
                                                frames * self.psd_size if stream_stride is None else stream_stride))

    def feed(self, psd):
        """psd: CUDA float32 tensor [n_streams, frames, psd_size]"""
        assert psd.is_cuda and psd.dim() == 3 and psd.shape[0] == self.n_streams and psd.shape[2] == self.psd_size
        psd = psd.contiguous()
        self._keep = psd
        self.feed_ptr(psd.data_ptr(), psd.shape[1])

    @property
    def device_ptr(self):
        return self._L.sdb_averager_device(self._h)

    def read(self):
        out = np.empty((self.n_streams, self.psd_size), np.float32)
        _check(self._L.sdb_averager_read(self._h, out.ctypes.data, out.size))
        return out


class Decimator:
    """Source decimator (SPEC L): FIR decimation by `decimation` of n_streams streams in a native sample format."""

    def __init__(self, decimation, n_streams=1, input_format="f32", max_feed=1 << 20, device=0):
        self._L = load_library()
        self.decimation, self.n_streams, self.max_feed = decimation, n_streams, max_feed
        self.input_format = FORMAT[input_format] if isinstance(input_format, str) else int(input_format)
        self._h = self._L.sdb_decimator_new(device, n_streams, decimation, self.input_format, max_feed)
        if not self._h:
            raise SdbError(last_error())
        self.last_out = 0

    def close(self):
        if getattr(self, "_h", None):
            self._L.sdb_decimator_destroy(self._h)
            self._h = None

    __del__ = close

    def _rows(self, x):
        """x: [n_streams, n] complex64 (f32) or [n_streams, 2 n] interleaved integers -> (array, n)"""
        x = np.ascontiguousarray(x)
        if x.ndim == 1:
            x = x.reshape(1, -1)
        assert x.shape[0] == self.n_streams
        return x, x.shape[1] if self.input_format == FORMAT["f32"] else x.shape[1] // 2

    def feed(self, x):
        """Host feed; returns the outputs per stream of this feed (read them with read())."""
        x, n = self._rows(x)
        self.last_out = _check(self._L.sdb_decimator_feed_host(self._h, x.ctypes.data, n, n))
        return self.last_out

    def feed_ptr(self, ptr, n, stream_stride=None):
        """Device feed: n samples per stream in the input format, stream_stride samples apart."""
        self.last_out = _check(self._L.sdb_decimator_feed_device(self._h, ptr, n if stream_stride is None
                                                                 else stream_stride, n))
        return self.last_out

    @property
    def output_ptr(self):
        return self._L.sdb_decimator_output_device(self._h)

    @property
    def output_stride(self):
        return self._L.sdb_decimator_output_stride(self._h)

    @property
    def stream_ptr(self):
        """cudaStream_t the feeds run on (e.g. for torch.cuda.ExternalStream)"""
        return self._L.sdb_decimator_stream(self._h)

    def sync(self):
        _check(self._L.sdb_decimator_sync(self._h))

    def read(self):
        """-> complex64 [n_streams, outputs of the last feed]"""
        out = np.empty((self.n_streams, self.last_out), np.complex64)
        _check(self._L.sdb_decimator_read(self._h, out.ctypes.data, out.shape[0] * out.shape[1]))
        return out

    def reset(self):
        _check(self._L.sdb_decimator_reset(self._h))
        self.last_out = 0


class PanoramicParams(C.Structure):
    """sdb_panoramic_params"""
    _fields_ = [("psd_size", C.c_uint32), ("psd_window", C.c_int32), ("fft_bandwidth", C.c_double),
                ("rel_bw", C.c_float), ("freq_min", C.c_double), ("freq_max", C.c_double), ("device", C.c_int32),
                ("detect", C.c_int32), ("det_alpha", C.c_float), ("det_gamma", C.c_float), ("det_snr", C.c_float),
                ("det_min_bins", C.c_uint32), ("channel_cap", C.c_uint32), ("frames_per_hop", C.c_uint32)]


class PanoramicTiming(C.Structure):
    """sdb_panoramic_timing"""
    _fields_ = [("psd_project_ms", C.c_float), ("gather_ms", C.c_float), ("accumulate_ms", C.c_float),
                ("gather_bytes", C.c_uint64), ("n_hops_local", C.c_uint64)]


def panoramic_unique_id():
    """128-byte NCCL id (rank 0); hand it to the other ranks before they build their Panoramic."""
    buf = (C.c_ubyte * 128)()
    L = load_library()
    if L.sdb_panoramic_unique_id(buf) != 0:
        raise SdbError(L.sdb_panoramic_last_error().decode())
    return bytes(buf)


class Panoramic:
    """sdb_panoramic_*: the sharded sweep + NCCL gather + stitch, all behind the C-ABI."""

    def __init__(self, psd_size, window, fft_bandwidth, view_range, rel_bw=0.5, device=0, rank=0, world=1,
                 unique_id=None, detect=None, channel_cap=64, frames_per_hop=1):
        self._L = L = load_library()
        d = detect or {}
        p = PanoramicParams(psd_size, WINDOW[window] if isinstance(window, str) else window, fft_bandwidth, rel_bw,
                            view_range[0], view_range[1], device, 1 if detect is not None else 0,
                            d.get("alpha", 1.0), d.get("gamma", 0.5), d.get("snr", 6.0), d.get("min_bins", 2), channel_cap,
                            frames_per_hop)
        idb = (C.c_ubyte * 128).from_buffer_copy(unique_id) if unique_id is not None else None
        self._h = L.sdb_panoramic_new(C.byref(p), rank, world, idb)
        if not self._h:
            raise SdbError(L.sdb_panoramic_last_error().decode())
        self.rank, self.world, self.channel_cap = rank, world, channel_cap

    def close(self):
        if getattr(self, "_h", None):
            self._L.sdb_panoramic_destroy(self._h)
            self._h = None

    __del__ = close

    @staticmethod
    def shard(n_hops, world, rank):
        lo, hi = C.c_size_t(), C.c_size_t()
        load_library().sdb_panoramic_shard(n_hops, world, rank, C.byref(lo), C.byref(hi))
        return lo.value, hi.value

    def sweep(self, hops_local, centers_all):
        """hops_local: this rank's shard [hi - lo, psd_size]: torch cuda complex64 tensor or numpy array."""
        c = np.ascontiguousarray(centers_all, dtype=np.float64)
        if _is_torch(hops_local):
            assert hops_local.is_cuda and hops_local.is_contiguous()
            rc = self._L.sdb_panoramic_sweep_device(self._h, hops_local.data_ptr() if hops_local.numel() else None,
                                                    c.ctypes.data, len(c))
        else:
            x = np.ascontiguousarray(hops_local, dtype=np.complex64)
            rc = self._L.sdb_panoramic_sweep_host(self._h, x.ctypes.data if x.size else None, c.ctypes.data, len(c))
        if rc != 0:
            raise SdbError(self._L.sdb_panoramic_last_error().decode())

    def reset(self):
        _check(self._L.sdb_panoramic_reset(self._h))

    def read(self):
        n = self._L.sdb_panoramic_size(self._h)
        out = [np.empty(n, np.float32) for _ in range(3)]
        if self._L.sdb_panoramic_read(self._h, out[0].ctypes.data, out[1].ctypes.data, out[2].ctypes.data, n) != 0:
            raise SdbError(self._L.sdb_panoramic_last_error().decode())
        return tuple(out)

    def read_channels(self, hop):
        buf = (DetectedChannel * self.channel_cap)()
        n = self._L.sdb_panoramic_read_channels(self._h, hop, buf, self.channel_cap)
        return [buf[i] for i in range(max(0, n))]

    def timing(self):
        t = PanoramicTiming()
        self._L.sdb_panoramic_last_timing(self._h, C.byref(t))
        return {"psd_project_ms": t.psd_project_ms, "gather_ms": t.gather_ms, "accumulate_ms": t.accumulate_ms,
                "gather_bytes": int(t.gather_bytes), "n_hops_local": int(t.n_hops_local)}


class SpectrumView:
    """Panoramic stitcher (Panoramic/Scanner.cpp:36-293). project() per rank, accumulate() on the owner."""

    def __init__(self, freq_min, freq_max, fft_bandwidth, rel_bw=0.5, device=0):
        self._L = load_library()
        self._h = self._L.sdb_sview_new(device)
        if not self._h:
            raise SdbError(last_error())
        _check(self._L.sdb_sview_set_range(self._h, freq_min, freq_max, fft_bandwidth, rel_bw))

    def close(self):
        if getattr(self, "_h", None):
            self._L.sdb_sview_destroy(self._h)
            self._h = None

    __del__ = close

    @property
    def size(self):
        return self._L.sdb_sview_size(self._h)

    @property
    def max_bins(self):
        return self._L.sdb_sview_max_bins(self._h)

    def reset(self):
        _check(self._L.sdb_sview_reset(self._h))

    def project(self, psd_dev_ptr, psd_size, centers, adjust_sides=True):
        centers = np.ascontiguousarray(centers, dtype=np.float64)
        self._centers = centers
        _check(self._L.sdb_sview_project(self._h, psd_dev_ptr, psd_size, centers.ctypes.data, len(centers),
                                         int(adjust_sides)))
        self._n_hops = len(centers)

    def contrib_ptrs(self):
        p = [C.c_void_p() for _ in range(4)]
        _check(self._L.sdb_sview_contrib(self._h, *[C.byref(q) for q in p]))
        return [q.value for q in p]

    def contrib_copy(self, j0_ptr, nb_ptr, va_ptr, vc_ptr, n_hops):
        _check(self._L.sdb_sview_contrib_copy(self._h, j0_ptr, nb_ptr, va_ptr, vc_ptr, n_hops))

    def accumulate(self, j0_ptr=None, nb_ptr=None, va_ptr=None, vc_ptr=None, n_hops=None):
        if j0_ptr is None:
            j0_ptr, nb_ptr, va_ptr, vc_ptr = self.contrib_ptrs()
            n_hops = self._n_hops
        _check(self._L.sdb_sview_accumulate(self._h, j0_ptr, nb_ptr, va_ptr, vc_ptr, n_hops))

    def feed_view(self, detail):
        """SpectrumView::feed(SpectrumView const &): the zoom path of the scanner"""
        _check(self._L.sdb_sview_feed_view(self._h, detail._h))

    def read(self):
        n = self.size
        psd, acc, cnt = (np.empty(n, np.float32) for _ in range(3))
        _check(self._L.sdb_sview_read(self._h, psd.ctypes.data, acc.ctypes.data, cnt.ctypes.data, n))
        return psd, acc, cnt


class TvParams(C.Structure):
    """sdb_tv_params == struct sigutils_tv_processor_params (Default/GenericInspector/TVProcessorTab.cpp:549-597)."""
    _fields_ = [("enable_sync", C.c_int32), ("reverse", C.c_int32), ("interlace", C.c_int32), ("enable_agc", C.c_int32),
                ("x_off", C.c_float), ("dominance", C.c_int32), ("frame_lines", C.c_uint32),
                ("frame_spacing", C.c_float), ("enable_comb", C.c_int32), ("comb_reverse", C.c_int32),
                ("hsync_len", C.c_float), ("vsync_len", C.c_float), ("line_len", C.c_float),
                ("vsync_odd_trigger", C.c_uint32), ("t_tol", C.c_float), ("l_tol", C.c_float), ("g_tol", C.c_float),
                ("hsync_huge_err", C.c_float), ("hsync_max_err", C.c_float), ("hsync_min_err", C.c_float),
                ("hsync_len_tau", C.c_float), ("line_len_tau", C.c_float), ("agc_tau", C.c_float),
                ("hsync_fast_track_tau", C.c_float), ("hsync_slow_track_tau", C.c_float)]


def tv_params(standard="pal", samp_rate=1e6, **kw):
    p = TvParams()
    getattr(load_library(), "sdb_tv_params_" + standard)(C.byref(p), samp_rate)
    for k, v in kw.items():
        setattr(p, k, v)
    return p


class TvProcessor:
    """A batch of analog-TV processors (one warp each): TVProcessorWorker::work over [batch][n] float samples."""

    def __init__(self, params, batch=1, device=0):
        self._L = load_library()
        self.batch = batch
        self._h = self._L.sdb_tv_processor_new(C.byref(params), batch, device)
        if not self._h:
            raise SdbError(last_error())
        w, h = C.c_uint32(), C.c_uint32()
        _check(self._L.sdb_tv_processor_geometry(self._h, C.byref(w), C.byref(h)))
        self.width, self.height = w.value, h.value

    def close(self):
        if getattr(self, "_h", None):
            self._L.sdb_tv_processor_destroy(self._h)
            self._h = None

    __del__ = close

    def set_params(self, params):
        _check(self._L.sdb_tv_processor_set_params(self._h, C.byref(params)))

    def feed(self, x):
        x = np.ascontiguousarray(x, dtype=np.float32).reshape(self.batch, -1)
        done = np.zeros(self.batch, np.uint32)
        rc = self._L.sdb_tv_processor_feed(self._h, x.ctypes.data, x.shape[1], x.shape[1], done.ctypes.data)
        if rc < 0:
            raise SdbError(last_error())
        return done

    def frames(self):
        c = np.zeros(self.batch, np.uint64)
        _check(self._L.sdb_tv_processor_frames(self._h, c.ctypes.data))
        return c

    def read_frame(self, which, frame_no):
        out = np.empty((self.height, self.width), np.float32)
        _check(self._L.sdb_tv_processor_read_frame(self._h, which, int(frame_no), out.ctypes.data, out.size))
        return out

    def estimates(self, which=0):
        a, b, g = C.c_float(), C.c_float(), C.c_float()
        _check(self._L.sdb_tv_processor_estimates(self._h, which, C.byref(a), C.byref(b), C.byref(g)))
        return a.value, b.value, g.value


class TvTabParams(C.Structure):
    """sdb_tv_tab_params: the Analog TV tab of one inspector (oracle/SPEC_TI.md)."""
    _fields_ = [("tv", TvParams), ("invert_sync", C.c_int32), ("dc", C.c_float)]


class TvStatus(C.Structure):
    """sdb_tv_status: one stream's TV processor after the latest feed."""
    _fields_ = [("frames", C.c_uint64), ("posted_no", C.c_uint64), ("completed", C.c_uint32), ("width", C.c_uint32),
                ("height", C.c_uint32), ("line_len", C.c_float), ("hsync_len", C.c_float), ("agc_gain", C.c_float)]


def tv_feed_transform(x, mode, k=1.0, dc=0.0):
    """TVProcessorTab::feed: mode "modulus" -> k |x| + dc, "argument" -> k arg(x) / pi + dc."""
    x = np.ascontiguousarray(x, dtype=np.complex64)
    out = np.empty(x.size, np.float32)
    _check(load_library().sdb_tv_feed_transform(x.ctypes.data, x.size, {"modulus": 0, "argument": 1}[mode], k, dc,
                                                out.ctypes.data))
    return out
