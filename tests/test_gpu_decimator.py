"""-m gpu: source decimation (SPEC L, oracle/SPEC_L.md).  The batched decimator (k_decimate) bit-identical to oracle/decimate.c at every
D, format, stream and feed split, and the analyzer / suscan shim running behind it at fs / D."""
import ctypes as C
import threading

import numpy as np
import pytest

import decim_oracle

from sigdigger_b200 import synth
from test_decimator_f64 import FORMATS, make_input, feed_rows, STOP_DB

pytestmark = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a, np.complex64).view(np.uint32)


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("D", [1, 2, 3, 7, 8, 16, 64, 256])
def test_decimator_bit_identical_to_oracle(sdb, D, fmt):
    S = 3
    m = 700 * D + 13
    xs = [make_input(fmt, m, seed=1000 * D + 17 * s + FORMATS.index(fmt)) for s in range(S)]
    rng = np.random.default_rng(D)
    # ragged feeds: shorter than D, D - 1, D + 1, a long one and random cuts
    cuts = sorted({1, max(1, D - 1) + 1, 2 * D + 2, 600 * D} | set(int(v) for v in rng.integers(1, m, 5)))
    cuts = [c for c in cuts if c < m] + [m]
    dec = sdb.Decimator(D, n_streams=S, input_format=fmt, max_feed=m)
    refs = [decim_oracle.Decimator(D, fmt) for _ in range(S)]
    for rnd in range(2):                                   # the second round runs after reset()
        a = 0
        for b in cuts:
            rows = np.stack([feed_rows(x, fmt, a, b) for x in xs])
            k = dec.feed(rows)
            got = dec.read()
            for s in range(S):
                ref = refs[s].feed(feed_rows(xs[s], fmt, a, b))
                assert k == len(ref)
                assert np.array_equal(bits(got[s]), bits(ref)), (rnd, s, a, b)
            a = b
        dec.reset()
        for r in refs:
            r.reset()
    dec.close()


def test_decimator_device_feed_and_strides(sdb):
    import torch
    D, S, n = 8, 2, 8 * 4096
    x = (0.2 * torch.randn(S, n + 100, dtype=torch.complex64, device="cuda"))
    torch.cuda.synchronize()
    dec = sdb.Decimator(D, n_streams=S, max_feed=n)
    assert dec.feed_ptr(x.data_ptr(), n, stream_stride=n + 100) == n // D
    got = dec.read()
    xh = x.cpu().numpy()
    for s in range(S):
        assert np.array_equal(bits(got[s]), bits(decim_oracle.Decimator(D).feed(xh[s, :n])))
    assert dec.output_stride >= n // D
    dec.close()


def test_decimator_rejects_bad_arguments(sdb):
    with pytest.raises(sdb.SdbError, match="decimation must be in"):
        sdb.Decimator(300)
    with pytest.raises(sdb.SdbError, match="decimation must be in"):
        sdb.Decimator(0)
    dec = sdb.Decimator(4, max_feed=1024)
    with pytest.raises(sdb.SdbError, match="feed size"):
        dec.feed(np.zeros(2048, np.complex64))


# ---- analyzer --------------------------------------------------------------------------------------------------------
def drain(a, timeout=20000):
    msgs = []
    while True:
        name, m = a.read(timeout)
        assert name != "TIMEOUT"
        msgs.append((name, m))
        if name in ("EOS", "READ_ERROR", "HALT"):
            return msgs


def test_analyzer_u8_capture_decimated(sdb, oracle):
    """D = 8 over an in-memory u8 capture: every PSD frame equals the PSD of the oracle-decimated stream; rates; a
    tone in the decimated band lands in its bin and a strong tone outside it stays below the alias bound."""
    from sigdigger_b200.analyzer import Analyzer
    N, fs, D = 4096, 8.0e6, 8
    blk = N * 4
    n = 6 * blk * D
    t = np.arange(n)
    f_in, f_out = 0.2 * fs / D, 0.7 * fs / D                # in band; aliases to -0.3 fs/D after decimation
    z = 0.3 * np.exp(2j * np.pi * f_in / fs * t) + 0.6 * np.exp(2j * np.pi * f_out / fs * t)
    iq = np.empty(2 * n, np.float64)
    iq[0::2], iq[1::2] = z.real, z.imag
    raw = np.clip(np.round(iq * 127 + 128), 0, 255).astype(np.uint8)
    a = Analyzer(fs, window_size=N, window="blackmann_harris", psd_update_int=0.0, data=raw, read_size=blk,
                 decimation=D)
    msgs = drain(a)
    a.close()
    assert msgs[0][0] == "SOURCE_INFO"
    assert msgs[0][1]["source_samp_rate"] == int(fs) and msgs[0][1]["effective_samp_rate"] == int(fs / D)
    assert msgs[-1][0] == "EOS"
    psd = [m for name, m in msgs if name == "PSD"]
    assert len(psd) == n // D // N
    assert all(m["samp_rate"] == fs / D for m in psd)
    y = decim_oracle.Decimator(D, "u8").feed(raw)
    ref = oracle.psd_frames(y, N, "blackmann_harris")
    assert np.array_equal(np.stack([m["psd"] for m in psd]).view(np.uint32), ref.view(np.uint32))
    # the tone at +0.2 fs/D sits in bin 0.2 N of the decimated spectrum (DC at index 0)
    p = np.stack([m["psd"] for m in psd])[1:]
    assert all(int(np.argmax(f)) == round(0.2 * N) for f in p)
    # the 0.6-amplitude tone at 0.7 fs/D aliases to bin -0.3 N, attenuated by at least the stopband bound
    k_alias = round(-0.3 * N) % N
    rel_db = 10 * np.log10(p[:, k_alias - 3:k_alias + 4].max(axis=1) / p[:, round(0.2 * N)] * (0.3 / 0.6) ** 2)
    assert np.all(rel_db <= -STOP_DB), rel_db


def test_analyzer_decimation_limits(sdb):
    from sigdigger_b200.analyzer import Analyzer
    x = np.zeros(1 << 16, np.complex64)
    with pytest.raises(sdb.SdbError, match="at most 256"):
        Analyzer(1e6, window_size=4096, data=x, decimation=300)
    with pytest.raises(sdb.SdbError, match="wide-spectrum"):
        Analyzer(1e6, window_size=4096, read=lambda priv, dst, n: 0, wide=True, min_freq=1e8, max_freq=1e8 + 4e6,
                 decimation=2)


class GatedSource:
    """Callback source over x (complex64) that parks before read number `park_at` until release() (requests queued
    while it is parked take effect from the next block on)."""

    def __init__(self, x, park_at):
        self.x, self.pos, self.calls, self.park_at = x, 0, 0, park_at
        self.parked, self.go = threading.Event(), threading.Event()

    def __call__(self, priv, dst, maxn):
        if self.calls == self.park_at:
            self.parked.set()
            self.go.wait(30)
        self.calls += 1
        take = min(maxn, len(self.x) - self.pos)
        if take > 0:
            C.memmove(dst, self.x.ctypes.data + 8 * self.pos, 8 * take)
            self.pos += take
        return take


def run_gated(fs, x, N, blk, D, park_at, on_park, **kw):
    from sigdigger_b200.analyzer import Analyzer
    src = GatedSource(x, park_at)
    a = Analyzer(fs, window_size=N, window="blackmann_harris", psd_update_int=0.0, read=src, read_size=blk,
                 decimation=D, **kw)
    assert src.parked.wait(20)
    on_park(a)
    src.go.set()
    msgs = drain(a)
    a.close()
    return msgs


def test_inspector_open_mid_stream_on_decimated_analyzer(sdb):
    """Opening an inspector mid-stream leaves the PSD stream of a decimated analyzer untouched, and its symbols equal
    those of an undecimated analyzer fed the oracle-decimated samples."""
    N, fs, D = 8192, 8.0e6, 8
    rate = fs / D
    baud = rate / 100.0
    blk = N * 8
    n = 6 * blk * D
    x, _ = synth.multi_carrier(n, fs, [("qpsk", 0.125 * rate + 3.0, baud, -10.0, {})], noise_db=-50.0, seed=41)
    x = np.ascontiguousarray(x, np.complex64)
    fs_ch = rate * 256 / N
    kw = dict(baud=baud, costas_order=2, bits_per_symbol=2, loop_bw=fs_ch * 2e-3, mf_type=1, mf_rolloff=0.35,
              clock_type=1, clock_gain=0.1, clock_running=1)

    def open_insp(a):
        a.open("psk", 0.125 * rate, 3 * baud, req_id=1)
        a.set_inspector_id(0, 0x51, req_id=2)
        cfg = sdb.InspectorConfig()
        sdb._check(sdb.load_library().sdb_inspector_config_default(C.byref(cfg), sdb.INSP["psk"], fs_ch))
        for k, v in kw.items():
            setattr(cfg, k, v)
        a.set_inspector_config(0, cfg, req_id=3)

    with_open = run_gated(fs, x, N, blk, D, 2, open_insp)
    without = run_gated(fs, x, N, blk, D, 2, lambda a: None)
    psd_a = np.stack([m["psd"] for name, m in with_open if name == "PSD"])
    psd_b = np.stack([m["psd"] for name, m in without if name == "PSD"])
    assert psd_a.shape[0] == n // D // N
    assert np.array_equal(psd_a.view(np.uint32), psd_b.view(np.uint32))
    soft_a = np.concatenate([m["samples"] for name, m in with_open if name == "SAMPLES"])
    hard_a = np.concatenate([m["symbols"] for name, m in with_open if name == "SAMPLES"])
    assert len(hard_a) > 100
    y = decim_oracle.Decimator(D).feed(x)
    undec = run_gated(rate, y, N, blk, 1, 2, open_insp)
    soft_b = np.concatenate([m["samples"] for name, m in undec if name == "SAMPLES"])
    hard_b = np.concatenate([m["symbols"] for name, m in undec if name == "SAMPLES"])
    assert np.array_equal(bits(soft_a), bits(soft_b)) and np.array_equal(hard_a, hard_b)


def test_baseband_filter_and_history_see_decimated_samples(sdb):
    N, fs, D = 4096, 4.0e6, 4
    blk = N * 2
    nblk = 7
    # block k carries a tone in bin 100 + 50 k of the decimated spectrum
    x = np.concatenate([(0.3 * np.exp(2j * np.pi * (100 + 50 * k) / N / D * np.arange(blk * D)))
                        for k in range(nblk)]).astype(np.complex64)
    seen = []

    def on_park(a):
        a.register_baseband_filter(lambda s, off: seen.append((off, s.copy())) or True)
        assert a.set_history_size(3 * blk)

    msgs = run_gated(fs, x, N, blk, D, 0, on_park)
    y = decim_oracle.Decimator(D).feed(x)
    assert [off for off, _ in seen] == [k * blk for k in range(nblk)]
    assert np.array_equal(bits(np.concatenate([s for _, s in seen])), bits(y))
    psd = [m for name, m in msgs if name == "PSD"]
    assert all(m["samp_rate"] == fs / D for m in psd)
    assert psd[-1]["history_size"] == 3 * blk


def test_replay_holds_decimated_samples(sdb):
    from sigdigger_b200.analyzer import Analyzer
    N, fs, D = 4096, 4.0e6, 4
    blk = N * 2
    step = threading.Semaphore(0)
    parked, go = threading.Event(), threading.Event()
    calls = [0]

    def read(priv, dst, n):
        if calls[0] == 0:
            parked.set()
            go.wait(30)
        if not step.acquire(timeout=30):
            return 0
        k = calls[0]
        calls[0] += 1
        x = (0.3 * np.exp(2j * np.pi * (100 + 50 * k) / N / D * np.arange(n))).astype(np.complex64)
        C.memmove(dst, x.ctypes.data, 8 * n)
        return n

    a = Analyzer(fs, window_size=N, window="hann", psd_update_int=0.0, read=read, read_size=blk, decimation=D)
    assert a.read(5000)[0] == "SOURCE_INFO"
    assert parked.wait(10)
    assert a.set_history_size(3 * blk)
    go.set()

    def frames(k, release=True):
        out = []
        if release:
            for _ in range(k):
                step.release()
        while len(out) < 2 * k:
            name, m = a.read(20000)
            assert name not in ("TIMEOUT", "EOS", "READ_ERROR", "HALT")
            if name == "PSD":
                out.append(m)
        return out

    live = frames(7)                                      # blocks 0..6; the ring is armed from block 1 on
    assert [int(np.argmax(m["psd"])) for m in live[2:]] == [100 + 50 * (i // 2) for i in range(2, 14)]
    a.replay(True)
    live += frames(1)                                     # the block in flight when the request lands
    n_calls = calls[0]
    rep = frames(3, release=False)                        # the source is paused: the ring holds blocks 5, 6, 7
    assert calls[0] == n_calls
    assert [int(np.argmax(m["psd"])) for m in rep] == [100 + 50 * b for b in (5, 5, 6, 6, 7, 7)]
    # the ring holds the decimated samples: every replayed frame is bit-identical to the live one
    for m, ref in zip(rep, live[10:16]):
        assert np.array_equal(m["psd"].view(np.uint32), ref["psd"].view(np.uint32))
        assert m["samp_rate"] == fs / D
    a.halt()
    for _ in range(4):
        step.release()
    a.close()


# ---- suscan shim -----------------------------------------------------------------------------------------------------
SHIM_TU = r"""
#include <analyzer/analyzer.h>
#include <analyzer/source.h>
#include <analyzer/mq.h>
#include <analyzer/msg.h>
#include <string.h>
// an in-memory float32 source with suscan_source_config_set_average(cfg, average); every PSD message until EOS
extern "C" long tu_average_psd(const SUCOMPLEX *x, SUSCOUNT n, unsigned samp_rate, unsigned fft_size, unsigned average,
                               float *rates, float *psd, size_t cap)
{
  struct suscan_analyzer_params params = suscan_analyzer_params_INITIALIZER;
  params.mode = SUSCAN_ANALYZER_MODE_CHANNEL;
  params.detector_params.window_size = fft_size;
  params.detector_params.window = SU_CHANNEL_DETECTOR_WINDOW_BLACKMANN_HARRIS;
  params.psd_update_int = 0;
  params.channel_update_int = 0;
  suscan_source_config_t *cfg = suscan_source_config_new("file", SUSCAN_SOURCE_FORMAT_RAW_FLOAT32);
  suscan_source_config_set_samp_rate(cfg, samp_rate);
  suscan_source_config_set_memory(cfg, x, n);
  suscan_source_config_set_read_size(cfg, 4 * fft_size);
  suscan_source_config_set_average(cfg, average);
  struct suscan_mq mq;
  if (!suscan_mq_init(&mq)) return -1;
  suscan_analyzer_t *a = suscan_analyzer_new(&params, cfg, &mq);
  if (!a) return -2;
  long got = 0;
  for (;;) {
    uint32_t type = 0;
    void *m = suscan_mq_read(&mq, &type);
    if (type == SUSCAN_ANALYZER_MESSAGE_TYPE_PSD) {
      const struct suscan_analyzer_psd_msg *p = (const struct suscan_analyzer_psd_msg *) m;
      if ((size_t) got < cap && p->psd_size == fft_size) {
        rates[got] = p->samp_rate;
        memcpy(psd + (size_t) got * fft_size, p->psd_data, fft_size * sizeof(float));
        ++got;
      }
    }
    suscan_analyzer_dispose_message(type, m);
    if (type == SUSCAN_ANALYZER_MESSAGE_TYPE_EOS || type == SUSCAN_ANALYZER_MESSAGE_TYPE_READ_ERROR) break;
  }
  suscan_analyzer_destroy(a);
  suscan_mq_finalize(&mq);
  suscan_source_config_destroy(cfg);
  return got;
}
"""


def test_shim_average_decimates(sdb, tmp_path):
    """suscan_source_config_set_average(cfg, 4): PSD messages at fs / 4 with the tone in its bin (without the
    decimator the tone landed at 4x its offset)."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libdir = os.path.join(root, "sigdigger_b200")
    src, so = tmp_path / "average_tu.cpp", tmp_path / "libaverage_tu.so"
    src.write_text(SHIM_TU)
    subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-I", os.path.join(root, "include"), str(src),
                    "-o", str(so), "-L", libdir, "-lsuscan", "-lsigutils", "-Wl,-rpath," + libdir, "-lpthread"],
                   check=True)
    L = C.CDLL(str(so))
    L.tu_average_psd.restype = C.c_long
    L.tu_average_psd.argtypes = [C.c_void_p, C.c_uint64, C.c_uint, C.c_uint, C.c_uint, C.c_void_p, C.c_void_p,
                                 C.c_size_t]
    N, fs, D = 4096, 4_000_000, 4
    f = 0.1 * fs / D
    n = 16 * N * D
    x = (0.3 * np.exp(2j * np.pi * f / fs * np.arange(n))).astype(np.complex64)
    cap = 64
    rates, psd = np.zeros(cap, np.float32), np.zeros((cap, N), np.float32)
    got = L.tu_average_psd(x.ctypes.data, n, fs, N, D, rates.ctypes.data, psd.ctypes.data, cap)
    assert got == n // D // N, got
    assert np.all(rates[:got] == fs / D)
    # +f at fs / D is bin 0.1 N (linear PSD, DC at index 0); the undecimated path put it at 0.4 N
    assert all(int(np.argmax(p)) == round(0.1 * N) for p in psd[1:got])
