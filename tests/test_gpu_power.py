"""-m gpu: the "power" inspector (SPEC PW, oracle/SPEC_PW.md), the RMS tool's integrated channel power.  The engine's
means are bit-identical to the oracle applied to the same engine's channel samples; a power channel leaves every
other inspector of the plan unchanged; a re-plan keeps the partial group unless M changes; through the analyzer the
means equal the RMS tab's raw-mode integration of a "raw" inspector on the same channel; and the suscan names carry
power.integrate-samples."""
import ctypes as C
import math
import os
import subprocess
import threading

import numpy as np
import pytest

import power_oracle as P
import shim_build as SB
from sigdigger_b200 import synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

W = 65536
# (f0 rad / sample, bw as a fraction of fs, precise, M): channel sizes 64, 1024 (k_chan_ifft16) and 16384; M = 0 is
# read as 1, 1000 divides no feed, 10^9 is longer than the whole run
POWER_PLAN = [(0.3, 0.0008, False, 1), (1.7, 0.01, True, 7), (3.5, 0.2, False, 512), (5.0, 0.012, False, 1000),
              (2.5, 0.0005, False, 10**9), (4.2, 0.0008, True, 0)]


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _signal(S, n, seed):
    rng = np.random.default_rng(seed)
    tone = np.exp(1j * 2 * np.pi * 0.27 * np.arange(n))
    return np.stack([(0.05 * (rng.standard_normal(n) + 1j * rng.standard_normal(n)) + 0.3 * tone)
                     .astype(np.complex64) for _ in range(S)])


def _power_engine(sdb, S, max_feed, plan=POWER_PLAN, input_format="f32"):
    e = sdb.Engine(n_streams=S, psd_size=W, psd_window="hann", max_feed=max_feed, samp_rate=1.0,
                   input_format=input_format)
    hs = []
    for f0, frac, precise, M in plan:
        h = e.open_channel(f0, 2 * np.pi * frac, 1.0, precise)
        e.set_inspector(h, "power", power_integrate_samples=M)
        hs.append(h)
    e.commit()
    return e, hs


def _check_feed(e, hs, S, oracles):
    """the means of the last feed against the oracle fed the same engine's channel samples of that feed"""
    for s in range(S):
        for h in hs:
            soft, hard = e.read_symbols(s, h)
            ref = oracles[(s, h)].feed(e.read_channel(s, h))
            assert np.array_equal(_bits(soft.real), _bits(ref)), (s, h, len(soft), len(ref))
            assert not soft.imag.any() and not hard.any()


@pytest.mark.parametrize("mode", ["host", "ragged", "device", "u8"])
def test_engine_means_match_oracle(sdb, mode):
    S = 3
    sizes = {"ragged": [1, 3, 2, 4, 1, 2]}.get(mode, [2] * 5)
    n = sum(sizes) * W
    e, hs = _power_engine(sdb, S, max(sizes) * W, input_format="u8" if mode == "u8" else "f32")
    assert sorted({e.channel_info(h).size for h in hs}) == [64, 1024, 16384]
    x = _signal(S, n, 3)
    if mode == "u8":
        x = np.clip(np.round(np.stack([x.real, x.imag], -1) * 128 + 128), 0, 255).astype(np.uint8)
    oracles = {(s, h): P.Power(M) for s in range(S) for h, (_, _, _, M) in zip(hs, POWER_PLAN)}
    e.timing(True)
    pos, means = 0, 0
    for m in sizes:
        blk = x[:, pos * W:(pos + m) * W]
        if mode == "device":
            import torch
            e.feed(torch.from_numpy(np.ascontiguousarray(blk)).cuda())
        else:
            e.feed(blk)
        _check_feed(e, hs, S, oracles)
        means += len(e.read_symbols(0, hs[0])[0])
        pos += m
    assert means > 0
    assert len(e.read_symbols(0, hs[4])[0]) == 0               # M = 10^9: the group never closes
    ms, launches = e.kernel_time("power")
    assert launches == len(sizes) and ms > 0


def test_kernel_keeps_the_kahan_compensation(sdb):
    """The kernel itself on an input where the compensation decides the binary32 mean (tests/test_power_oracle.py,
    kahan_case): 37 buffers (two warps) of 200 samples (not a whole number of 32-sample chunks), scaled by powers of two
    so that every buffer keeps its tie, bit-identical to the oracle and not to an uncompensated sum; and noise buffers
    for M = 1, 3 and 64."""
    from test_power_oracle import kahan_case, noise, plain_sum
    base = kahan_case(50)
    x = np.stack([base * np.float32(2.0 ** (b % 5 - 2)) for b in range(37)])
    got = sdb.task_power(x, 4)
    for b in range(37):
        ref = P.Power(4).feed(x[b])
        assert len(ref) == 50 and not got[b].imag.any()
        assert np.array_equal(_bits(got[b].real), _bits(ref)), b
        assert not np.array_equal(_bits(got[b].real), _bits(plain_sum(x[b], 4))), b
    y = np.stack([noise(5000, s) for s in range(40)])
    for M in (1, 3, 64):
        got = sdb.task_power(y, M)
        for b in range(40):
            assert np.array_equal(_bits(got[b].real), _bits(P.Power(M).feed(y[b]))), (M, b)


def _mixed_plan(sdb, with_power):
    """psk, fsk, ask, audio and raw inspectors, with or without power channels between them -> (engine, handles of
    the non-power inspectors)"""
    fs = 1.0
    baud = fs / 200.0
    e = sdb.Engine(n_streams=3, psd_size=W, psd_window="hann", max_feed=2 * W, samp_rate=fs)
    insp = [(0.4, "psk", dict(baud=baud, costas_order=2, bits_per_symbol=2, mf_type=1, clock_gain=0.1)),
            (1.1, "fsk", dict(baud=baud)), (2.0, "ask", dict(baud=baud)), (2.9, "audio", {}), (3.6, "raw", {})]
    hs = []
    for k, (f0, cls, kw) in enumerate(insp):
        if with_power:
            hp = e.open_channel(f0 + 0.2, 2 * np.pi * 0.01, 1.0, k % 2 == 1)
            e.set_inspector(hp, "power", power_integrate_samples=100 + k)
        h = e.open_channel(f0, 2 * np.pi * 0.01, 1.0, False)
        kw = dict(kw)
        if "loop_bw" not in kw and cls == "psk":
            kw["loop_bw"] = e.channel_rate(h) * 2e-3
        e.set_inspector(h, cls, **kw)
        hs.append(h)
    e.commit()
    return e, hs


def test_mixed_plan_leaves_other_inspectors_unchanged(sdb):
    S = 3
    x = _signal(S, 8 * W, 5)
    x += np.stack([synth.multi_carrier(8 * W, 1.0, [("qpsk", 0.4 / (2 * np.pi), 1 / 200.0, -10.0, {})],
                                       noise_db=-60.0, seed=s)[0].astype(np.complex64) for s in range(S)])
    runs = []
    for with_power in (False, True):
        e, hs = _mixed_plan(sdb, with_power)
        out = []
        for f in range(4):
            e.feed(x[:, f * 2 * W:(f + 1) * 2 * W])
            out.append([e.read_symbols(s, h) for s in range(S) for h in hs])
        runs.append(out)
        e.close()
    total = 0
    for fa, fb in zip(*runs):
        for (sa, ha), (sb, hb) in zip(fa, fb):
            assert np.array_equal(_bits(sa.view(np.float32)), _bits(sb.view(np.float32))) and np.array_equal(ha, hb)
            total += len(sa)
    assert total > 0


def test_migration_keeps_group_and_m_change_restarts(sdb):
    """Re-planned mid-group (a raw channel added, channels in another order) the means are those of an engine that
    never re-planned; a re-plan that changes M restarts the group at that feed."""
    S = 3
    plan = [(1.7, 0.01, True, 1000), (0.3, 0.0008, False, 7)]
    x = _signal(S, 10 * W, 9)
    ref_e, ref_h = _power_engine(sdb, S, 2 * W, plan)
    first, _ = _power_engine(sdb, S, 2 * W, plan)
    L = first._L
    ref_means = {(s, h): [] for s in range(S) for h in ref_h}
    for f in range(5):
        ref_e.feed(x[:, f * 2 * W:(f + 1) * 2 * W])
        for s in range(S):
            for h in ref_h:
                ref_means[(s, h)].append(ref_e.read_symbols(s, h)[0].real)
    for f in range(2):
        first.feed(x[:, f * 2 * W:(f + 1) * 2 * W])
    for M1 in (7, 8):                       # same M: the group goes on; another M: it restarts
        second = sdb.Engine(n_streams=S, psd_size=W, psd_window="hann", max_feed=2 * W, samp_rate=1.0)
        hr = second.open_channel(2.2, 2 * np.pi * 0.01, 1.0, False)
        second.set_inspector(hr, "raw")
        h1 = second.open_channel(0.3, 2 * np.pi * 0.0008, 1.0, False)
        second.set_inspector(h1, "power", power_integrate_samples=M1)
        h0 = second.open_channel(1.7, 2 * np.pi * 0.01, 1.0, True)
        second.set_inspector(h0, "power", power_integrate_samples=1000)
        second.commit()
        sdb._check(L.sdb_engine_migrate_map(second._h, first._h, (C.c_int32 * 3)(-1, 1, 0), 3))
        restart = {(s, 1): P.Power(M1) for s in range(S)}
        for f in range(2, 5):
            second.feed(x[:, f * 2 * W:(f + 1) * 2 * W])
            for s in range(S):
                m0 = second.read_symbols(s, h0)[0].real
                m1 = second.read_symbols(s, h1)[0].real
                assert np.array_equal(_bits(m0), _bits(ref_means[(s, 0)][f])), (M1, f, s)
                want = ref_means[(s, 1)][f] if M1 == 7 else restart[(s, 1)].feed(second.read_channel(s, h1))
                assert np.array_equal(_bits(m1), _bits(want)), (M1, f, s)
        second.close()


# ---------------------------------------------------------------------------------------------- analyzer
class Stepper:
    """In-memory source read block by block: read call k parks until the test allows it, so that requests sent
    while the worker is parked in call k take effect from block k + 1."""

    def __init__(self, x):
        self.x, self.pos, self.calls, self.allowed = x, 0, 0, 0
        self.cv = threading.Condition()

    def read(self, priv, dst, maxn):
        with self.cv:
            self.calls += 1
            self.cv.notify_all()
            self.cv.wait_for(lambda: self.calls <= self.allowed, timeout=60)
        take = min(maxn, len(self.x) - self.pos)
        if take > 0:
            C.memmove(dst, self.x.ctypes.data + 8 * self.pos, 8 * take)
            self.pos += take
        return take

    def park(self, k):
        """wait until the worker is in read call k (it has handled the requests sent before)"""
        with self.cv:
            assert self.cv.wait_for(lambda: self.calls >= k, timeout=60)

    def release(self, k):
        with self.cv:
            self.allowed = k
            self.cv.notify_all()


def _drain(a):
    msgs = []
    while True:
        name, m = a.read(60000)
        assert name != "TIMEOUT"
        msgs.append((name, m))
        if name in ("EOS", "READ_ERROR", "HALT"):
            return msgs


def test_analyzer_power_is_the_raw_mode_integration(sdb):
    """"power" and "raw" on one channel, from block 2: the power SAMPLES are the RMS tab's raw-mode integration of the
    raw SAMPLES, bit for bit, across an inspector opened mid-stream (live from block 5), and restart with the new M
    from the block after a SET_CONFIG (block 7).  The OPEN reply carries the default M, SET_CONFIG / GET_CONFIG the new one."""
    from sigdigger_b200.analyzer import Analyzer
    N, fs, blocks = 8192, 1.0e6, 9
    per_block = 4 * N
    x, _ = synth.multi_carrier(blocks * per_block, fs, [("qpsk", 0.1 * fs, fs / 100, -10.0, {})], noise_db=-40.0,
                               seed=21)
    x = np.ascontiguousarray(x, np.complex64)
    src = Stepper(x)
    a = Analyzer(fs, window_size=N, window="hann", psd_update_int=1.0, read=src.read, read_size=per_block)
    assert a.read(5000)[0] == "SOURCE_INFO"
    M1, M2 = 500, 333
    src.park(1)
    a.open("raw", 0.1 * fs, fs / 32, req_id=1)                       # handle 0
    a.open("power", 0.1 * fs, fs / 32, req_id=2)                     # handle 1
    a.set_inspector_id(0, 10, req_id=3)
    a.set_inspector_id(1, 11, req_id=4)
    cfg1 = sdb.InspectorConfig()
    sdb._check(a._L.sdb_inspector_config_default(C.byref(cfg1), sdb.INSP["power"], 1.0))
    cfg1.power_integrate_samples = M1
    a.set_inspector_config(1, cfg1, req_id=7)
    src.release(3)
    src.park(4)
    a.open("psk", -0.2 * fs, fs / 64, req_id=5)                      # handle 2, live from block 5
    src.release(5)
    src.park(6)
    cfg = sdb.InspectorConfig()
    assert a._L.sdb_analyzer_get_inspector_config(a._h, 1, C.byref(cfg)) == 0
    cfg.power_integrate_samples = M2
    a.set_inspector_config(1, cfg, req_id=6)                          # live from block 7
    src.release(6)
    src.park(7)
    got = sdb.InspectorConfig()
    assert a._L.sdb_analyzer_get_inspector_config(a._h, 1, C.byref(got)) == 0
    assert got.power_integrate_samples == M2 and got.insp_class == sdb.INSP["power"]
    src.release(10**6)
    msgs = _drain(a)
    a.close()
    assert msgs[-1][0] == "EOS"
    replies = {m["req_id"]: m for name, m in msgs if name == "INSPECTOR"}
    assert replies[2]["kind"] == "OPEN" and replies[2]["class_name"] == "power"
    equiv = float(replies[2]["equiv_fs"])
    assert replies[2]["config"].power_integrate_samples == max(1, int(math.floor(0.1 * equiv + 0.5)))
    assert replies[7]["kind"] == "SET_CONFIG" and replies[7]["config"].power_integrate_samples == M1
    assert replies[6]["kind"] == "SET_CONFIG" and replies[6]["config"].power_integrate_samples == M2
    raw = [m["samples"] for name, m in msgs if name == "SAMPLES" and m["inspector_id"] == 10]
    power = [m for name, m in msgs if name == "SAMPLES" and m["inspector_id"] == 11]
    assert len(raw) == blocks - 1                                     # blocks 2 .. 9, one batch each
    got_means = np.concatenate([m["samples"] for m in power])
    assert not got_means.imag.any() and not np.concatenate([m["symbols"] for m in power]).any()
    # blocks 2-6 with M1 (the psk open at block 5 keeps the group), blocks 7-9 with M2 from an empty group
    before, after = P.gui_raw_mode(np.concatenate(raw[:5]), M1), P.gui_raw_mode(np.concatenate(raw[5:]), M2)
    assert len(before) >= 5 and len(after) >= 5
    want = np.concatenate([before, after])
    assert np.array_equal(_bits(got_means.real), _bits(want))


def test_shim_power_session(sdb):
    """Through libsuscan.so: open_async("power"), a "power" bag with power.integrate-samples set by
    suscan_config_set_integer, set_inspector_config_async; the SAMPLES' real parts equal the oracle over the channel
    samples from the block the configuration went live."""
    so = os.path.join(SB.build_dir(), "libpowertu.so")
    libdir = os.path.join(ROOT, "sigdigger_b200")
    subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "shim", "power_tu.cpp"), "-o", so, "-L", libdir, "-lsuscan",
                    "-lsigutils", "-Wl,-rpath," + libdir, "-lpthread"], check=True)
    tu = C.CDLL(so)
    tu.tu_power_session.restype = C.c_long
    tu.tu_power_session.argtypes = [C.c_void_p, C.c_size_t, C.c_uint, C.c_uint, C.c_size_t, C.c_double, C.c_double,
                                    C.c_uint64, C.c_void_p, C.c_size_t]
    N, fs, blocks = 8192, 1000000, 6
    per_block = 4 * N
    n = blocks * per_block
    fc, bw, M = 0.125 * fs, fs / 50.0, 777
    x, _ = synth.multi_carrier(n, float(fs), [("qpsk", fc, fs / 200.0, -10.0, {})], noise_db=-40.0, seed=23)
    x = np.ascontiguousarray(x, np.complex64)
    out = np.zeros(n, np.float32)
    got = tu.tu_power_session(x.ctypes.data, n, fs, N, per_block, fc, bw, M, out.ctypes.data, n)
    assert got > 0, got
    # the analyzer's channel from block 2 on: a fresh channeliser over the source from there (the block-1 engine had
    # no channel, so no history)
    e = sdb.Engine(n_streams=1, psd_size=N, psd_window="blackmann_harris", max_feed=per_block, samp_rate=float(fs))
    h = e.open_channel(np.float32(2 * np.pi * math.fmod(fc / fs + 1.0, 1.0)), np.float32(2 * np.pi * bw / fs), 1.0)
    e.commit()
    pw, ref = P.Power(M), []
    for b in range(1, blocks):
        e.feed(x[None, b * per_block:(b + 1) * per_block])
        ref.append(pw.feed(e.read_channel(0, h)))
    ref = np.concatenate(ref)
    assert got == len(ref)
    assert np.array_equal(_bits(out[:got]), _bits(ref))
