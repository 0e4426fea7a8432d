"""-m gpu: how the analyzer plans its engines -- the OPEN replies at the channel-geometry limits, what a commit that
rejects an inspector's configuration does to a sub-carrier level and to the baseband, and that SET_PARAMS does not
switch the worker's mode."""
import ctypes as C
import math

import numpy as np
import pytest

from sigdigger_b200 import synth
from test_gpu_analyzer import Gate

pytestmark = pytest.mark.gpu


def gated_analyzer(x, N, per_block, fs):
    """Analyzer over x behind a Gate: requests sent once gate.parked is set take effect after the first block."""
    from sigdigger_b200.analyzer import Analyzer
    gate, pos = Gate(), [0]

    def read(priv, dst, maxn):
        gate.wait(30)
        take = min(maxn, len(x) - pos[0])
        if take > 0:
            C.memmove(dst, x.ctypes.data + 8 * pos[0], 8 * take)
            pos[0] += take
        return take

    a = Analyzer(fs, window_size=N, window="hann", psd_update_int=1.0, read=read, read_size=per_block)
    assert a.read(5000)[0] == "SOURCE_INFO"
    assert gate.parked.wait(10)
    return a, gate


def drain(a):
    msgs = []
    while True:
        name, m = a.read(30000)
        assert name != "TIMEOUT"
        msgs.append((name, m))
        if name in ("EOS", "READ_ERROR", "HALT"):
            return msgs


def psk_config(sdb, fs_ch, **kw):
    cfg = sdb.InspectorConfig()
    sdb._check(sdb.load_library().sdb_inspector_config_default(C.byref(cfg), sdb.INSP["psk"], fs_ch))
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


def test_open_replies_at_geometry_limits(sdb):
    """A baseband channel above 16384 bins is INVALID_CHANNEL; a sub-carrier open on a parent whose channel has fewer
    than 16 bins is WRONG_HANDLE, on a 32-bin parent INVALID_CHANNEL (a channeliser window needs 64 points), and on a
    128-bin parent OPEN at the rate sdb_channel_geometry gives."""
    N, fs = 65536, 1.0e6
    x = np.zeros(4 * N * 2, np.complex64)
    a, gate = gated_analyzer(x, N, 2 * N, fs)
    bins = lambda k: k * fs / N
    a.open("raw", 0.0, fs / 2, req_id=1)                     # 32768-point channel
    a.open("raw", 0.1 * fs, bins(7.5), req_id=2)             # handle 0: 8-point channel
    a.open("raw", 0.0, bins(1), req_id=3, parent=0)
    a.open("raw", 0.2 * fs, bins(30), req_id=4)              # handle 1: 32-point channel
    a.open("raw", 0.0, bins(1), req_id=5, parent=1)
    a.open("raw", -0.2 * fs, bins(100), req_id=6)            # handle 2: 128-point channel
    fs_par = fs * 128 / N
    a.open("psk", fs_par / 8, fs_par / 4, req_id=7, parent=2)
    a.close_inspector(0, req_id=8)
    a.close_inspector(1, req_id=9)
    gate.set()
    msgs = drain(a)
    a.close()
    assert msgs[-1][0] == "EOS"
    replies = [(m["kind"], m["req_id"], m["handle"]) for name, m in msgs if name == "INSPECTOR"]
    assert replies == [("INVALID_CHANNEL", 1, -1), ("OPEN", 2, 0), ("WRONG_HANDLE", 3, 0), ("OPEN", 4, 1),
                       ("INVALID_CHANNEL", 5, -1), ("OPEN", 6, 2), ("OPEN", 7, 3), ("CLOSE", 8, 0), ("CLOSE", 9, 1)]
    par = next(m for name, m in msgs if name == "INSPECTOR" and m["req_id"] == 6)
    assert par["equiv_fs"] == np.float32(fs_par)
    cp = sdb.ChannelParams(np.float32(2 * math.pi * ((fs_par / 8 / fs_par + 1.0) % 1.0)),
                           np.float32(2 * math.pi * (fs_par / 4) / fs_par), 1.0, 0)
    info = sdb.ChannelInfo()
    sdb._check(sdb.load_library().sdb_channel_geometry(128, C.byref(cp), C.byref(info)))
    assert info.size == 32
    child = next(m for name, m in msgs if name == "INSPECTOR" and m["req_id"] == 7)
    assert child["equiv_fs"] == np.float32(fs_par / info.decimation)


def subcarrier_run(sdb, with_child):
    """A PSK inspector on the baseband; with_child: a PSK sub-carrier inspector on its channel whose costas_order (4)
    the commit of the sub-carrier engine rejects."""
    N, fs = 8192, 1.0e6
    baud = fs / 512.0
    per_block = N * 8
    x, _ = synth.multi_carrier(6 * per_block, fs, [("qpsk", 0.125 * fs + fs / 64.0, baud, -10.0, {})],
                               noise_db=-55.0, seed=17)
    a, gate = gated_analyzer(x, N, per_block, fs)
    fs_par = fs / 8.0
    a.open("psk", 0.125 * fs, fs / 8.0, req_id=1)
    a.set_inspector_id(0, 0x10, req_id=2)
    a.set_inspector_config(0, psk_config(sdb, fs_par, clock_running=1), req_id=3)
    if with_child:
        fs_ch = fs_par * 64 / 1024
        a.open("psk", fs / 64.0, 3 * baud, req_id=4, parent=0)
        a.set_inspector_id(1, 0x11, req_id=5)
        a.set_inspector_config(1, psk_config(sdb, fs_ch, baud=baud, costas_order=4, clock_running=1), req_id=6)
    gate.set()
    msgs = drain(a)
    a.close()
    return msgs


def test_rejected_subcarrier_config_unmaps_only_that_level(sdb):
    """The sub-carrier engine's commit fails: its inspectors deliver nothing, the worker goes on, and the parent's
    samples are bit-identical to a run in which the child was never opened."""
    with_child, alone = subcarrier_run(sdb, True), subcarrier_run(sdb, False)
    assert with_child[-1][0] == "EOS" and alone[-1][0] == "EOS"
    assert not any(name == "READ_ERROR" for name, _ in with_child)
    kinds = [m["kind"] for name, m in with_child if name == "INSPECTOR"]
    assert kinds == ["OPEN", "SET_ID", "SET_CONFIG", "OPEN", "SET_ID", "SET_CONFIG"]
    assert not any(name == "SAMPLES" and m["inspector_id"] == 0x11 for name, m in with_child)
    samples = lambda msgs: [m for name, m in msgs if name == "SAMPLES"]
    got, ref = samples(with_child), samples(alone)
    assert ref and all(m["inspector_id"] == 0x10 for m in got)
    assert np.array_equal(np.concatenate([m["samples"] for m in got]).view(np.uint32),
                          np.concatenate([m["samples"] for m in ref]).view(np.uint32))
    assert np.array_equal(np.concatenate([m["symbols"] for m in got]), np.concatenate([m["symbols"] for m in ref]))


def test_rejected_baseband_config_ends_the_worker(sdb):
    """The baseband engine's commit fails: SOURCE_INIT / INIT_FAILURE with the engine's message, then READ_ERROR."""
    N, fs = 8192, 1.0e6
    x = np.zeros(6 * N * 8, np.complex64)
    a, gate = gated_analyzer(x, N, N * 8, fs)
    a.open("psk", 0.125 * fs, fs / 8.0, req_id=1)
    a.set_inspector_config(0, psk_config(sdb, fs / 8.0, costas_order=4), req_id=2)
    gate.set()
    msgs = drain(a)
    a.close()
    assert [(m["kind"], m["req_id"]) for name, m in msgs if name == "INSPECTOR"] == [("OPEN", 1), ("SET_CONFIG", 2)]
    (n1, init), (n2, end) = msgs[-2:]
    assert (n1, init["code"]) == ("SOURCE_INIT", -1) and n2 == "READ_ERROR"
    assert "invalid inspector configuration" in init["err_msg"]
    assert "invalid inspector configuration" in end["err_msg"]


def test_set_params_keeps_the_mode(sdb):
    """A channel-mode analyzer stays in channel mode when SET_PARAMS asks for wide-spectrum sweeps: every frame of
    every block gives a PSD at the source frequency, none at a hop centre."""
    from sigdigger_b200.analyzer import AnalyzerParams
    N, fs, blocks = 4096, 1.0e6, 6
    x = (0.1 * np.exp(2j * np.pi * 0.1 * np.arange(blocks * N * 8))).astype(np.complex64)
    a, gate = gated_analyzer(x, N, N * 8, fs)
    p = AnalyzerParams()
    C.memmove(C.byref(p), C.byref(a.params), C.sizeof(p))
    p.mode, p.min_freq, p.max_freq, p.psd_update_int = 1, 100e6, 110e6, 0.0
    assert a._L.sdb_analyzer_set_params_async(a._h, C.byref(p), 7) == 0
    gate.set()
    msgs = drain(a)
    a.close()
    assert msgs[-1][0] == "EOS"
    assert [name for name, _ in msgs].count("PARAMS") == 1
    psd = [m for name, m in msgs if name == "PSD"]
    assert len(psd) >= (blocks - 1) * 8 and all(m["fc"] == 0 and m["samp_rate"] == fs for m in psd)
