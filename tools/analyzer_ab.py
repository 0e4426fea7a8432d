"""Message-stream A/B of the analyzer: the analyzer's counterpart of tools/gpu_ab.sh.

Usage: python tools/analyzer_ab.py <parent library .so>

Runs one scripted session in two subprocesses, one with SDB_LIB=<parent library> and one with this tree's library,
records every message (its type, every payload field and every array it points to; only rt_time and
measured_samp_rate, which come from the wall clock, are left out) and compares the two records for exact equality.

The session is stepped one block at a time: after the first read, the worker parks in a baseband filter in every
block (replayed blocks included), and each block's requests are queued while it is parked there, so both runs see
the same block boundaries.  It covers a PSK and an FSK baseband inspector, a two-level sub-carrier chain, a spectrum
source with both estimators, the channel detector, a watermark, a mid-stream SET_CONFIG and SET_FREQ, closing a
parent (its children close too), history and replay, and a baseband filter registered mid-stream.  A second session
decimates by 2 and parks in every read: the engine reads the decimated block in device memory until a baseband filter
is registered, then from the host.  Then a u8 in-memory capture with decimation 4 and a separate wide-spectrum sweep,
each without requests."""
import ctypes as C
import os
import pickle
import subprocess
import sys
import tempfile
import threading

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SKIP = {"rt_time", "measured_samp_rate"}


def leaves(s, prefix=""):
    """(name, raw bytes) of every scalar field of structure s, recursively; pointers are left to the caller."""
    out = []
    for f in s._fields_:
        name, typ = f[0], f[1]
        if name in SKIP or issubclass(typ, (C._Pointer, C.c_char_p, C.c_void_p, C._CFuncPtr)):
            continue
        if issubclass(typ, C.Structure):
            out += leaves(getattr(s, name), prefix + name + ".")
        else:
            d = getattr(type(s), name)
            out.append((prefix + name, C.string_at(C.addressof(s) + d.offset, d.size)))
    return out


def record(L, ptr, t):
    """One message as (type, scalar fields, arrays)."""
    from sigdigger_b200 import DetectedChannel
    from sigdigger_b200.analyzer import (MSG_NAME, AnalyzerParams, ChannelMsg, InspectorMsg, PsdMsg, SampleBatchMsg,
                                         SourceInfo, StatusMsg)
    name = MSG_NAME.get(t, str(t))
    typ = {"PSD": PsdMsg, "SAMPLES": SampleBatchMsg, "INSPECTOR": InspectorMsg, "CHANNEL": ChannelMsg,
           "SOURCE_INFO": SourceInfo, "PARAMS": AnalyzerParams, "EOS": StatusMsg, "READ_ERROR": StatusMsg,
           "SOURCE_INIT": StatusMsg, "HALT": StatusMsg}[name]
    m = C.cast(ptr, C.POINTER(typ)).contents
    arrays = []
    if name == "PSD":
        arrays = [C.string_at(m.psd_data, 4 * m.psd_size)]
    elif name == "SAMPLES":
        arrays = [C.string_at(m.samples, 8 * m.sample_count), C.string_at(m.symbols, m.sample_count)]
    elif name == "INSPECTOR":
        arrays = [m.class_name, C.string_at(m.spectrum_data, 4 * m.spectrum_size) if m.spectrum_data else None]
    elif name == "CHANNEL":
        lst = C.cast(m.channel_list, C.POINTER(DetectedChannel))
        arrays = [leaves(lst[k]) for k in range(m.channel_count)]
    elif typ is StatusMsg:
        arrays = [m.err_msg]
    return name, leaves(m), arrays


def drain(a):
    L, out, t = a._L, [], C.c_uint32()
    while True:
        ptr = L.sdb_analyzer_read_timeout(a._h, C.byref(t), 60000)
        if t.value == 0xfffffffe:
            raise RuntimeError("no message for 60 s")
        out.append(record(L, ptr, t.value))
        L.sdb_analyzer_dispose_message(t.value, ptr)
        if out[-1][0] in ("EOS", "READ_ERROR", "HALT"):
            return out


class SteppedSource:
    """Float32 callback source over x.  in_read: the worker parks in every read.  Otherwise the first read waits for
    first.set() and from then on the worker parks in park(), a baseband filter, once per block."""

    def __init__(self, x, in_read=False):
        self.x, self.pos, self.in_read = x, 0, in_read
        self.first, self.parked, self.go, self.ended = threading.Event(), threading.Semaphore(0), \
            threading.Semaphore(0), threading.Event()

    def read(self, priv, dst, maxn):
        if self.in_read:
            self.park(None, 0)
        elif self.pos == 0:
            self.first.wait(60)
        take = min(maxn, len(self.x) - self.pos)
        C.memmove(dst, self.x.ctypes.data + 8 * self.pos, 8 * max(take, 0))
        self.pos += max(take, 0)
        if take < maxn:
            self.ended.set()
        return max(take, 0)

    def park(self, buf, offset):
        self.parked.release()
        self.go.acquire()
        return True

    def step(self):
        """Wait until the worker parks in its next block; False once the source has run out."""
        while not self.parked.acquire(timeout=0.05):
            if self.ended.is_set():
                return False
        return True


def channel_session():
    import numpy as np
    import sigdigger_b200 as sdb
    from sigdigger_b200 import synth
    from sigdigger_b200.analyzer import Analyzer
    N, fs = 4096, 1.0e6
    blk, blocks = N * 8, 30
    baud = fs / 512.0
    x, _ = synth.multi_carrier(blocks * blk, fs, [("qpsk", 0.125 * fs + fs / 64.0, baud, -10.0, {}),
                                                  ("qpsk", -0.2 * fs, fs / 100.0, -12.0, {}),
                                                  ("fsk", 0.3 * fs, fs / 200.0, -14.0, {})], noise_db=-50.0, seed=5)
    src = SteppedSource(x)
    a = Analyzer(fs, window_size=N, window="blackmann_harris", psd_update_int=3 * N / fs, read=src.read,
                 read_size=blk, channel_update_int=0.05)

    def cfg(cls, fs_ch, **kw):
        c = sdb.InspectorConfig()
        sdb._check(sdb.load_library().sdb_inspector_config_default(C.byref(c), sdb.INSP[cls], fs_ch))
        c.clock_running = 1
        for k, v in kw.items():
            setattr(c, k, v)
        return c

    fs_psk, fs_fsk, fs_par = fs * 128 / N, fs * 64 / N, fs * 512 / N       # 128-, 64- and 512-point channels
    fs_ch = fs_par * 128 / 512 * 32 / 128                                   # 512 -> 128 -> 32 points

    def block0():
        a.open("psk", -0.2 * fs, 3 * fs / 100.0, req_id=1)                       # 0: PSK on the baseband
        a.set_inspector_id(0, 100, req_id=2)
        a.set_inspector_config(0, cfg("psk", fs_psk, baud=fs / 100.0, mf_type=1, clock_gain=0.1), req_id=3)
        a.set_spectrum_source(0, 1, req_id=4)
        a.estimator_cmd(0, 0, True, req_id=5)
        a.estimator_cmd(0, 1, True, req_id=6)
        a.open("fsk", 0.3 * fs, 3 * fs / 200.0, req_id=7)                        # 1: FSK on the baseband
        a.set_inspector_id(1, 101, req_id=8)
        a.set_inspector_config(1, cfg("fsk", fs_fsk, baud=fs / 200.0), req_id=9)
        a.set_inspector_watermark(1, 5000, req_id=10)
        a.open("raw", 0.125 * fs, fs / 8.0, req_id=11)                          # 2: parent
        a.set_inspector_id(2, 102, req_id=12)
        a.open("raw", fs / 64.0, fs_par / 4, req_id=13, parent=2)                # 3: child on the parent's channel
        a.open("psk", 0.0, 3 * baud, req_id=14, parent=3)                        # 4: grandchild on the child's
        a.set_inspector_id(4, 104, req_id=15)
        a.set_inspector_config(4, cfg("psk", fs_ch, baud=baud, mf_type=1, clock_gain=0.1), req_id=16)
        a.open("psk", 0.0, 1e9, req_id=17, parent=4)                             # wider than its parent: rejected
        a.set_history_size(4 * blk)

    def scale(buf, offset):
        buf *= np.float32(0.9)
        return True

    script = {
        0: block0,
        5: lambda: (a.set_inspector_config(0, cfg("psk", fs_psk, baud=fs / 100.0, mf_type=1, clock_gain=0.2,
                                                  loop_bw=fs_psk * 3e-3), req_id=20),
                    a.set_inspector_freq(4, 20.0)),
        8: lambda: a.register_baseband_filter(scale),
        12: lambda: a.close_inspector(2, req_id=21),                            # 3 and 4 close with it
        15: lambda: a.replay(True),
        22: lambda: a.replay(False),
    }
    a.register_baseband_filter(src.park)
    src.first.set()
    k = 0
    while src.step():
        script.get(k, lambda: None)()
        k += 1
        src.go.release()
    msgs = drain(a)
    a.close()
    return msgs


def decimated_session():
    """Decimation 2, parked in every read: the engine reads the decimated block in device memory until a baseband
    filter is registered, then the block comes to the host; history from then on too."""
    import numpy as np
    import sigdigger_b200 as sdb
    from sigdigger_b200 import synth
    from sigdigger_b200.analyzer import Analyzer
    N, fs, D, blk, blocks = 4096, 2.0e6, 2, 4096 * 4, 16
    x, _ = synth.multi_carrier(blocks * blk * D, fs, [("qpsk", 0.1 * fs / D, fs / D / 100.0, -10.0, {})],
                               noise_db=-50.0, seed=9)
    src = SteppedSource(x, in_read=True)
    a = Analyzer(fs, window_size=N, window="hann", psd_update_int=0.0, read=src.read, read_size=blk, decimation=D)
    cfg = sdb.InspectorConfig()
    fs_ch = fs / D * 128 / N
    sdb._check(sdb.load_library().sdb_inspector_config_default(C.byref(cfg), sdb.INSP["psk"], fs_ch))
    cfg.clock_running, cfg.baud = 1, fs / D / 100.0

    def scale(buf, offset):
        buf *= np.float32(0.5)
        return True

    script = {
        0: lambda: (a.open("psk", 0.1 * fs / D, 3 * fs / D / 100.0, req_id=1), a.set_inspector_id(0, 200, req_id=2),
                    a.set_inspector_config(0, cfg, req_id=3)),
        4: lambda: a.register_baseband_filter(scale),
        8: lambda: a.set_history_size(2 * blk),
    }
    k = 0
    while src.step():
        script.get(k, lambda: None)()
        k += 1
        src.go.release()
    msgs = drain(a)
    a.close()
    return msgs


def u8_session():
    import numpy as np
    from sigdigger_b200.analyzer import Analyzer
    N, fs, D = 2048, 4.0e6, 4
    n = 10 * N * 4 * D
    t = np.arange(n)
    z = 0.3 * np.exp(2j * np.pi * 0.03 * t) + 0.2 * np.exp(-2j * np.pi * 0.2 * t)
    iq = np.empty(2 * n)
    iq[0::2], iq[1::2] = z.real, z.imag
    raw = np.clip(np.round(iq * 127 + 128), 0, 255).astype(np.uint8)
    a = Analyzer(fs, window_size=N, window="hann", psd_update_int=0.0, data=raw, read_size=N * 4, decimation=D)
    msgs = drain(a)
    a.close()
    return msgs


def wide_session():
    import numpy as np
    from sigdigger_b200.analyzer import Analyzer
    N, fs = 1024, 2.0e6
    n = 40 * 16 * N
    x = (0.2 * np.exp(2j * np.pi * 0.1 * np.arange(n)) +
         0.01 * np.random.default_rng(3).standard_normal(n)).astype(np.complex64)
    pos = [0]

    def read(priv, dst, maxn):
        take = min(maxn, n - pos[0])
        C.memmove(dst, x.ctypes.data + 8 * pos[0], 8 * take)
        pos[0] += take
        return take

    a = Analyzer(fs, window_size=N, window="hann", read=read, wide=True, min_freq=100e6, max_freq=110e6,
                 set_frequency=lambda f: 0)
    msgs = drain(a)
    a.close()
    return msgs


def main():
    if len(sys.argv) == 3 and sys.argv[1] == "--record":
        out = channel_session() + decimated_session() + u8_session() + wide_session()
        with open(sys.argv[2], "wb") as f:
            pickle.dump(out, f)
        return 0
    if len(sys.argv) != 2:
        sys.stderr.write(__doc__)
        return 2
    arms = {"parent": os.path.abspath(sys.argv[1]),
            "new": os.path.join(ROOT, "sigdigger_b200", "libsigdigger_b200.so")}
    recs = {}
    with tempfile.TemporaryDirectory() as tmp:
        for arm, lib in arms.items():
            path = os.path.join(tmp, arm + ".pkl")
            subprocess.run([sys.executable, os.path.abspath(__file__), "--record", path], check=True,
                           env=dict(os.environ, SDB_LIB=lib))
            with open(path, "rb") as f:
                recs[arm] = pickle.load(f)
    p, n = recs["parent"], recs["new"]
    def key(m):            # INSPECTOR messages by kind, SAMPLES by inspector id
        f = dict(m[1])
        if m[0] == "INSPECTOR":
            return "INSPECTOR/%d" % int.from_bytes(f["kind"], "little")
        return "SAMPLES/%d" % int.from_bytes(f["inspector_id"], "little") if m[0] == "SAMPLES" else m[0]

    count = lambda r: {k: sum(1 for m in r if key(m) == k) for k in sorted({key(m) for m in r})}
    print("parent: %d messages %s" % (len(p), count(p)))
    print("new:    %d messages %s" % (len(n), count(n)))
    if p == n:
        print("identical message streams")
        return 0
    k = next((i for i, (u, v) in enumerate(zip(p, n)) if u != v), min(len(p), len(n)))
    print("streams DIFFER at message %d: parent %s / new %s" % (k, p[k][0] if k < len(p) else None,
                                                               n[k][0] if k < len(n) else None))
    return 1


if __name__ == "__main__":
    sys.exit(main())
