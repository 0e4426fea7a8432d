"""ctypes mirror of the suscan-style asynchronous analyzer (include/sigdigger_b200.h, sdb_analyzer_*).

Plays the role of `Suscan::Analyzer` + `Analyzer::AsyncThread` (Suscan/Analyzer.cpp:63-115, 601-638): construct,
queue requests, drain messages.  Message payloads are copied into Python objects and disposed at once."""
import ctypes as C

import numpy as np

from . import (INSP, WINDOW, FacParams, FacStatus, InspectorConfig, SdbError, SnrParams, SnrStatus, TvStatus,
               TvTabParams, last_error, load_library)

MSG = {"SOURCE_INFO": 0, "SOURCE_INIT": 1, "CHANNEL": 2, "EOS": 3, "READ_ERROR": 4, "INTERNAL": 5, "SAMPLES": 6,
       "INSPECTOR": 7, "PSD": 8, "PARAMS": 9, "HALT": 0xffffffff, "TIMEOUT": 0xfffffffe}
MSG_NAME = {v: k for k, v in MSG.items()}
# sdb_analyzer_params.psd_detector (SPEC PK): which spectrum a PSD message carries
PSD_DETECTOR = {"default": 0, "pos_peak": 1, "neg_peak": 2}
KIND = {0: "OPEN", 1: "SET_ID", 2: "GET_CONFIG", 3: "SET_CONFIG", 4: "ESTIMATOR", 5: "SPECTRUM", 6: "CLOSE",
        7: "INVALID_CHANNEL", 8: "WRONG_HANDLE", 9: "WRONG_OBJECT", 10: "WRONG_KIND", 11: "FAC",
        12: "SNR", 13: "TV"}


class Timeval(C.Structure):
    _fields_ = [("tv_sec", C.c_long), ("tv_usec", C.c_long)]


class SigutilsChannel(C.Structure):
    _fields_ = [("fc", C.c_double), ("ft", C.c_double), ("f_lo", C.c_double), ("f_hi", C.c_double), ("bw", C.c_float)]


class DetectorParams(C.Structure):
    _fields_ = [("window_size", C.c_uint64), ("window", C.c_int32), ("alpha", C.c_float), ("beta", C.c_float),
                ("gamma", C.c_float), ("snr", C.c_float)]


class AnalyzerParams(C.Structure):
    _fields_ = [("mode", C.c_int32), ("detector_params", DetectorParams), ("channel_update_int", C.c_float),
                ("psd_update_int", C.c_float), ("min_freq", C.c_double), ("max_freq", C.c_double),
                ("psd_average", C.c_int32), ("psd_detector", C.c_int32), ("spectrum_update_int", C.c_float),
                ("channel_hold_int", C.c_float)]


READ_FN = C.CFUNCTYPE(C.c_long, C.c_void_p, C.c_void_p, C.c_size_t)
BB_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64)
SETF_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_double)


class SourceConfig(C.Structure):
    _fields_ = [("samp_rate", C.c_double), ("freq", C.c_double), ("read_size", C.c_size_t), ("read", READ_FN),
                ("priv", C.c_void_p), ("data", C.c_void_p), ("length", C.c_size_t), ("loop", C.c_int32),
                ("device", C.c_int32), ("input_format", C.c_int32), ("set_frequency", SETF_FN),
                ("decimation", C.c_uint32)]


class SourceInfo(C.Structure):
    _fields_ = [("permissions", C.c_uint64), ("source_samp_rate", C.c_uint64), ("effective_samp_rate", C.c_uint64),
                ("measured_samp_rate", C.c_float), ("frequency", C.c_double), ("seekable", C.c_int32)]


class PsdMsg(C.Structure):
    _fields_ = [("fc", C.c_int64), ("inspector_id", C.c_uint32), ("timestamp", Timeval), ("rt_time", Timeval),
                ("looped", C.c_int32), ("history_size", C.c_uint64), ("samp_rate", C.c_float),
                ("measured_samp_rate", C.c_float), ("psd_size", C.c_uint64), ("psd_data", C.POINTER(C.c_float))]


class SampleBatchMsg(C.Structure):
    _fields_ = [("inspector_id", C.c_uint32), ("samples", C.POINTER(C.c_float)), ("sample_count", C.c_uint64),
                ("symbols", C.POINTER(C.c_uint8))]


class InspectorMsg(C.Structure):
    _fields_ = [("kind", C.c_int32), ("inspector_id", C.c_uint32), ("req_id", C.c_uint32), ("handle", C.c_int32),
                ("class_name", C.c_char_p), ("channel", SigutilsChannel), ("config", InspectorConfig),
                ("fs", C.c_float), ("equiv_fs", C.c_float), ("bandwidth", C.c_float), ("lo", C.c_float),
                ("spectsrc_count", C.c_uint32), ("estimator_count", C.c_uint32), ("spectsrc_id", C.c_uint32),
                ("spectrum_data", C.POINTER(C.c_float)), ("spectrum_size", C.c_uint64), ("samp_rate", C.c_uint64),
                ("estimator_id", C.c_uint32), ("enabled", C.c_int32), ("value", C.c_float), ("fac", FacStatus),
                ("snr", SnrStatus), ("snr_histogram", C.POINTER(C.c_uint32)), ("tv", TvStatus),
                ("tv_frame", C.POINTER(C.c_float))]


class ChannelMsg(C.Structure):
    _fields_ = [("source", C.c_void_p), ("channel_count", C.c_uint32), ("channel_list", C.c_void_p),
                ("tracked_list", C.c_void_p)]


class StatusMsg(C.Structure):
    _fields_ = [("code", C.c_int32), ("err_msg", C.c_char_p)]


class Analyzer:
    def __init__(self, samp_rate, window_size=8192, window="hann", psd_update_int=0.04, data=None, read=None,
                 read_size=0, loop=False, freq=0.0, device=0, channel_update_int=0.0, alpha=0.25, beta=0.25,
                 gamma=0.5, snr=8.0, wide=False, min_freq=0.0, max_freq=0.0, set_frequency=None, decimation=1,
                 psd_average=0, psd_detector=0, spectrum_update_int=0.0, channel_hold_int=0.0):
        """decimation: source decimation D (SPEC L); the analyzer then runs at samp_rate / D.
        psd_average: non-zero posts the mean of the frames of every psd_update_int instead of one frame (SPEC A).
        psd_detector: "pos_peak" / "neg_peak" (or PSD_DETECTOR's numbers) post the per-bin maximum / minimum of those
        frames instead (SPEC PK); 0 or "default" leaves the choice to psd_average.
        spectrum_update_int: > 0 emits inspector spectra and baud estimates every that many seconds of channel time,
        over 4096-point frames carried across blocks (SPEC US); 0 = once per block that fills a frame.
        channel_hold_int: > 0 follows detected channels across blocks (SPEC KT): CHANNEL messages then list tracks,
        kept through gaps shorter than this many seconds, with S0 smoothed by beta and id / age / present /
        misses; needs channel_update_int > 0 (the detector)."""
        self._L = load_library()
        p = AnalyzerParams()
        p.mode = 1 if wide else 0                      # SDB_ANALYZER_MODE_{CHANNEL, WIDE_SPECTRUM}
        p.min_freq, p.max_freq = min_freq, max_freq
        p.detector_params.window_size = window_size
        p.detector_params.window = WINDOW[window] if isinstance(window, str) else window
        p.detector_params.alpha, p.detector_params.beta = alpha, beta
        p.detector_params.gamma, p.detector_params.snr = gamma, snr
        p.psd_update_int = psd_update_int
        p.channel_update_int = channel_update_int
        p.psd_average = psd_average
        p.psd_detector = PSD_DETECTOR[psd_detector] if isinstance(psd_detector, str) else psd_detector
        p.spectrum_update_int = spectrum_update_int
        p.channel_hold_int = channel_hold_int
        self.params = p
        s = SourceConfig()
        s.samp_rate, s.freq, s.read_size, s.loop, s.device = samp_rate, freq, read_size, int(loop), device
        s.decimation = decimation
        if data is not None:
            data = np.asarray(data)
            if data.dtype in (np.uint8, np.int8, np.int16):       # native capture formats: interleaved I,Q
                from . import FORMAT
                self._data = np.ascontiguousarray(data).reshape(-1)
                s.input_format = {np.dtype(np.uint8): FORMAT["u8"], np.dtype(np.int8): FORMAT["s8"],
                                  np.dtype(np.int16): FORMAT["s16"]}[self._data.dtype]
                s.data, s.length = self._data.ctypes.data, len(self._data) // 2
            else:
                self._data = np.ascontiguousarray(data, dtype=np.complex64)
                s.data, s.length = self._data.ctypes.data, len(self._data)
            s.read = READ_FN(0)
        else:
            self._cb = READ_FN(read)
            s.read = self._cb
        if set_frequency is not None:
            self._setf = SETF_FN(lambda priv, f: int(set_frequency(f) or 0))
            s.set_frequency = self._setf
        self._h = self._L.sdb_analyzer_new(C.byref(p), C.byref(s))
        if not self._h:
            raise SdbError(last_error() or "sdb_analyzer_new failed (no CUDA device or invalid parameters)")

    def close(self):
        if getattr(self, "_h", None):
            self._L.sdb_analyzer_destroy(self._h)
            self._h = None

    __del__ = close

    def halt(self):
        self._L.sdb_analyzer_req_halt(self._h)

    def open(self, cls, fc, bw, precise=False, req_id=0, parent=-1):
        """parent >= 0: sub-carrier inspector on that inspector's channel (fc relative to its centre)."""
        ch = SigutilsChannel(fc, 0.0, fc - bw / 2 - fc, fc + bw / 2 - fc, bw)
        ch.f_lo, ch.f_hi = -bw / 2, bw / 2          # as InspToolWidget.cpp:688-693 fills it
        if self._L.sdb_analyzer_open_ex_async(self._h, cls.encode(), C.byref(ch), int(precise), parent, req_id):
            raise SdbError("open_ex_async rejected")

    def set_inspector_id(self, handle, inspector_id, req_id=0):
        self._L.sdb_analyzer_set_inspector_id_async(self._h, handle, inspector_id, req_id)

    def set_inspector_config(self, handle, cfg, req_id=0):
        self._L.sdb_analyzer_set_inspector_config_async(self._h, handle, C.byref(cfg), req_id)

    def set_inspector_watermark(self, handle, watermark, req_id=0):
        self._L.sdb_analyzer_set_inspector_watermark_async(self._h, handle, int(watermark), req_id)

    def set_inspector_freq(self, handle, freq):
        self._L.sdb_analyzer_set_inspector_freq_overridable(self._h, handle, float(freq))

    def set_inspector_bandwidth(self, handle, bw):
        self._L.sdb_analyzer_set_inspector_bandwidth_overridable(self._h, handle, float(bw))

    # wide-spectrum (panoramic) mode controls, Panoramic/Scanner.cpp:396-503
    def set_hop_range(self, fmin, fmax):
        return self._L.sdb_analyzer_set_hop_range(self._h, float(fmin), float(fmax)) == 0

    def set_rel_bandwidth(self, rel_bw):
        self._L.sdb_analyzer_set_rel_bandwidth(self._h, float(rel_bw))

    def set_buffering_size(self, samples):
        self._L.sdb_analyzer_set_buffering_size(self._h, int(samples))

    def set_sweep_strategy(self, progressive=True):
        self._L.sdb_analyzer_set_sweep_strategy(self._h, 1 if progressive else 0)

    def set_spectrum_partitioning(self, continuous=False):
        self._L.sdb_analyzer_set_spectrum_partitioning(self._h, 1 if continuous else 0)

    def set_history_size(self, samples):
        return self._L.sdb_analyzer_set_history_size(self._h, int(samples)) == 0

    def replay(self, enabled=True):
        self._L.sdb_analyzer_replay(self._h, int(enabled))

    def seek(self, seconds):
        tv = Timeval(int(seconds), int(round((seconds - int(seconds)) * 1e6)))
        return self._L.sdb_analyzer_seek(self._h, C.byref(tv)) == 0

    def set_iq_reverse(self, enabled=True):
        self._L.sdb_analyzer_set_iq_reverse(self._h, int(enabled))

    def set_throttle(self, samp_rate, req_id=0):
        self._L.sdb_analyzer_set_throttle_async(self._h, int(samp_rate), req_id)

    def register_baseband_filter(self, fn):
        """fn(samples: complex64 ndarray view (writable), offset) -> truthy; runs on the worker thread."""
        def tramp(priv, a, ptr, length, offset):
            buf = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_float)), shape=(2 * length,)).view(np.complex64)
            return 1 if fn(buf, offset) else 0
        cb = BB_FN(tramp)
        self._bb = getattr(self, "_bb", []) + [cb]          # keep the trampolines alive
        self._L.sdb_analyzer_register_baseband_filter(self._h, C.cast(cb, C.c_void_p), None)

    def set_spectrum_source(self, handle, spectsrc_id, req_id=0):
        self._L.sdb_analyzer_inspector_set_spectrum_async(self._h, handle, spectsrc_id, req_id)

    def set_fac(self, handle, size=65536, alpha=1.0, lags=None, sigma=5.0, enabled=True, req_id=0):
        """the FAC tab of a psk / fsk / ask inspector (oracle/SPEC_FC.md), from the next block; enabled=False: off"""
        if not enabled:
            self._L.sdb_analyzer_inspector_set_fac_async(self._h, handle, None, req_id)
            return
        lo, hi = lags if lags is not None else (0, 0)
        p = FacParams(size, alpha, lo, hi, sigma)
        self._L.sdb_analyzer_inspector_set_fac_async(self._h, handle, C.byref(p), req_id)

    def set_snr(self, handle, alpha, bins=256, sigma=1.0, enabled=True, req_id=0):
        """the SNR meter of a psk / fsk / ask inspector (oracle/SPEC_SN.md), from the next block; enabled=False: off.
        The GUI's toggle uses sigma = 1 and alpha = 1 / 2^bits_per_symbol of the inspector."""
        if not enabled:
            self._L.sdb_analyzer_inspector_set_snr_async(self._h, handle, None, req_id)
            return
        p = SnrParams(bins, sigma, alpha)
        self._L.sdb_analyzer_inspector_set_snr_async(self._h, handle, C.byref(p), req_id)

    def reset_snr(self, handle, sigma=1.0, req_id=0):
        """the meter's sigma from the next block on; the histogram is kept"""
        self._L.sdb_analyzer_inspector_reset_snr_async(self._h, handle, sigma, req_id)

    def set_tv(self, handle, params=None, invert=False, dc=0.0, enabled=True, req_id=0):
        """the Analog TV tab of a psk / fsk / ask inspector (oracle/SPEC_TI.md): params a tv_params(...) block at the
        inspector's symbol rate, invert the tab's "invert sync", dc its DC value / 100; enabled=False (or params None):
        off.  A change that keeps the picture geometry applies at the next block without a re-plan."""
        if not enabled or params is None:
            self._L.sdb_analyzer_inspector_set_tv_async(self._h, handle, None, req_id)
            return
        p = TvTabParams(params, int(bool(invert)), dc)
        self._L.sdb_analyzer_inspector_set_tv_async(self._h, handle, C.byref(p), req_id)

    def estimator_cmd(self, handle, estimator_id, enabled=True, req_id=0):
        self._L.sdb_analyzer_inspector_estimator_cmd_async(self._h, handle, estimator_id, int(enabled), req_id)

    def set_params(self, req_id=0, **changes):
        """suscan_analyzer_set_params_async: the current params with `changes` (AnalyzerParams field names; the
        detector's window_size / window as such)"""
        p = AnalyzerParams()
        C.memmove(C.byref(p), C.byref(self.params), C.sizeof(p))
        for k, v in changes.items():
            if k in ("window_size", "window"):
                setattr(p.detector_params, k, WINDOW[v] if k == "window" and isinstance(v, str) else v)
            elif k == "psd_detector":
                p.psd_detector = PSD_DETECTOR[v] if isinstance(v, str) else v
            elif hasattr(p, k):
                setattr(p, k, v)
            else:
                raise KeyError(k)
        if self._L.sdb_analyzer_set_params_async(self._h, C.byref(p), req_id):
            raise SdbError("set_params_async rejected")
        self.params = p

    def close_inspector(self, handle, req_id=0):
        self._L.sdb_analyzer_close_async(self._h, handle, req_id)

    def read(self, timeout_ms=None):
        """-> (type name, payload dict); payload memory is disposed before returning."""
        t = C.c_uint32()
        if timeout_ms is None:
            ptr = self._L.sdb_analyzer_read(self._h, C.byref(t))
        else:
            ptr = self._L.sdb_analyzer_read_timeout(self._h, C.byref(t), timeout_ms)
        name = MSG_NAME.get(t.value, str(t.value))
        out = {}
        if ptr:
            if name == "PSD":
                m = C.cast(ptr, C.POINTER(PsdMsg)).contents
                out = dict(psd=np.ctypeslib.as_array(m.psd_data, shape=(m.psd_size,)).copy(), samp_rate=m.samp_rate,
                           measured_samp_rate=m.measured_samp_rate, fc=m.fc, looped=m.looped,
                           history_size=m.history_size,
                           timestamp=m.timestamp.tv_sec + 1e-6 * m.timestamp.tv_usec)
            elif name == "SAMPLES":
                m = C.cast(ptr, C.POINTER(SampleBatchMsg)).contents
                n = m.sample_count
                out = dict(inspector_id=m.inspector_id,
                           samples=np.ctypeslib.as_array(m.samples, shape=(2 * n,)).copy().view(np.complex64),
                           symbols=np.ctypeslib.as_array(m.symbols, shape=(n,)).copy())
            elif name == "INSPECTOR":
                m = C.cast(ptr, C.POINTER(InspectorMsg)).contents
                cfg = InspectorConfig()
                C.memmove(C.byref(cfg), C.byref(m.config), C.sizeof(cfg))
                out = dict(kind=KIND.get(m.kind, m.kind), req_id=m.req_id, handle=m.handle,
                           inspector_id=m.inspector_id, class_name=(m.class_name or b"").decode(), config=cfg,
                           fs=m.fs, equiv_fs=m.equiv_fs, bandwidth=m.bandwidth, lo=m.lo,
                           spectsrc_count=m.spectsrc_count, estimator_count=m.estimator_count,
                           spectsrc_id=m.spectsrc_id, estimator_id=m.estimator_id, enabled=m.enabled, value=m.value,
                           samp_rate=m.samp_rate, spectrum=None)
                if m.spectrum_data and m.spectrum_size:
                    out["spectrum"] = np.ctypeslib.as_array(m.spectrum_data, shape=(m.spectrum_size,)).copy()
                if out["kind"] == "FAC":
                    f = m.fac
                    out["fac"] = dict(blocks=f.blocks, peak_lag=f.peak_lag, max=f.max, min=f.min, sigmas=f.sigmas,
                                      marker=f.marker)
                if out["kind"] == "SNR":
                    q = m.snr
                    out["snr"] = dict(counted=q.counted, steps=q.steps, stepped=q.stepped, sigma=q.sigma, snr=q.snr,
                                      delta=q.delta)
                    out["histogram"] = None
                    if m.snr_histogram and m.spectrum_size:
                        out["histogram"] = np.ctypeslib.as_array(m.snr_histogram, shape=(m.spectrum_size,)).copy()
                if out["kind"] == "TV":
                    q = m.tv
                    out["tv"] = dict(frames=q.frames, posted_no=q.posted_no, completed=q.completed, width=q.width,
                                     height=q.height, line_len=q.line_len, hsync_len=q.hsync_len, agc_gain=q.agc_gain)
                    out["frame"] = None
                    if m.tv_frame and q.width and q.height:
                        out["frame"] = np.ctypeslib.as_array(m.tv_frame, shape=(q.height, q.width)).copy()
            elif name == "CHANNEL":
                from . import DetectedChannel
                m = C.cast(ptr, C.POINTER(ChannelMsg)).contents
                arr = C.cast(m.channel_list, C.POINTER(DetectedChannel))
                out = dict(channels=[dict(fc=arr[i].fc, f_lo=arr[i].f_lo, f_hi=arr[i].f_hi, bw=arr[i].bw,
                                          snr=arr[i].snr, S0=arr[i].S0, N0=arr[i].N0) for i in range(m.channel_count)])
                if m.tracked_list:
                    from . import TrackedChannel
                    tr = C.cast(m.tracked_list, C.POINTER(TrackedChannel))
                    for i, c in enumerate(out["channels"]):
                        c.update(id=tr[i].id, age=tr[i].age, present=tr[i].present, misses=tr[i].misses)
            elif name == "SOURCE_INFO":
                m = C.cast(ptr, C.POINTER(SourceInfo)).contents
                out = dict(source_samp_rate=m.source_samp_rate, effective_samp_rate=m.effective_samp_rate,
                           frequency=m.frequency, seekable=m.seekable)
            elif name == "PARAMS":
                m = C.cast(ptr, C.POINTER(AnalyzerParams)).contents
                out = dict(mode=m.mode, window_size=m.detector_params.window_size, window=m.detector_params.window,
                           psd_update_int=m.psd_update_int, channel_update_int=m.channel_update_int,
                           psd_average=m.psd_average, psd_detector=m.psd_detector,
                           spectrum_update_int=m.spectrum_update_int)
            elif name in ("EOS", "READ_ERROR", "HALT", "SOURCE_INIT"):
                m = C.cast(ptr, C.POINTER(StatusMsg)).contents
                out = dict(code=m.code, err_msg=(m.err_msg or b"").decode())
            self._L.sdb_analyzer_dispose_message(t.value, ptr)
        return name, out


__all__ = ["Analyzer", "MSG", "INSP"]
