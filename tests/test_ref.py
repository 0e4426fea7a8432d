"""CPU: the oracle pinned to the REFERENCE ITSELF where the reference contains the arithmetic.  oracle/_ref/libsdref.so
is built by `make -C oracle ref` from the reference's own sources where they lie (Panoramic/Scanner.cpp:1-293,
Tasks/QuadDemodTask.cpp, Tasks/DelayedConjTask.cpp, Tasks/WaveSampler.cpp, Misc/Averager.cpp,
Default/GenericInspector/TVProcessorWorker.cpp) behind no-behaviour Qt
stubs (oracle/ref_shim/, oracle/ref_glue.cpp); nothing of the reference is copied.  The restatements of oracle/*.c are
compared with it here; the Python transcriptions of tests/golden/make_golden.py stay as a second opinion.
What the compiled reference computed on these inputs is stored in tests/golden/ref_compiled.npz (as SHA-256 of the
bytes where the comparison is bit for bit; `python tests/golden/make_golden.py --compiled-reference` rewrites it)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_golden as G     # noqa: E402


@pytest.fixture(scope="module")
def ref():
    with np.load(os.path.join(ROOT, "tests", "golden", "ref_compiled.npz")) as z:
        return {k: z[k] for k in z.files}


def _bits(*arrays):
    return [G.sha(a) for a in arrays]


def _sview_oracle(oracle, fmin, fmax, feeds, rel_bw=0.5):
    L = oracle.lib()
    v = oracle.SpectrumView()
    assert L.sdo_sview_init(C.byref(v)) == 0
    L.sdo_sview_set_range(C.byref(v), fmin, fmax)
    v.fft_bandwidth = feeds[0][2]
    v.fft_rel_bw = rel_bw
    for psd, fc, bw in feeds:
        p = np.ascontiguousarray(psd, np.float32)
        L.sdo_sview_feed(C.byref(v), oracle.ptr(p), None, len(p), float(fc), 1)
    n = v.spectrum_size
    return [np.ctypeslib.as_array(q, shape=(65536,))[:n].copy() for q in (v.psd, v.psd_accum, v.psd_count)], v


def test_spectrumview_restatement_equals_the_compiled_reference(ref, oracle):
    """linear mode with revisits (forgetting rule, gap filling), histogram mode, and view-to-view feed"""
    (fmin, fmax, fftbw, feeds), (fmin2, fmax2, _, feeds2), (fmin3, fmax3, _, _) = G.sview_cases()
    got, ov = _sview_oracle(oracle, fmin, fmax, feeds)
    assert len(got[0]) == ref["sview0_size"] and _bits(*got) == list(ref["sview0_sha"])
    # histogram mode: hops narrower than two destination bins
    got, ov2 = _sview_oracle(oracle, fmin2, fmax2, feeds2)
    assert len(got[0]) == ref["sview1_size"] and _bits(*got) == list(ref["sview1_sha"])
    # SpectrumView::feed(SpectrumView const &): zoom path of Scanner::setViewRange
    L = oracle.lib()
    wide_o = oracle.SpectrumView(); assert L.sdo_sview_init(C.byref(wide_o)) == 0
    L.sdo_sview_set_range(C.byref(wide_o), fmin3, fmax3)
    wide_o.fft_bandwidth = fftbw; wide_o.fft_rel_bw = 0.5
    L.sdo_sview_feed_view(C.byref(wide_o), C.byref(ov))
    L.sdo_sview_interpolate(C.byref(wide_o))
    n = wide_o.spectrum_size
    assert n == ref["sview2_size"]
    assert _bits(*(np.ctypeslib.as_array(q, shape=(65536,))[:n] for q in (wide_o.psd, wide_o.psd_accum,
                                                                         wide_o.psd_count))) == list(ref["sview2_sha"])


def test_timewindow_tasks_equal_the_compiled_reference(ref, oracle):
    c = G.timewindow_case()
    # QuadDemodTask: the reference calls std::arg (libm), the oracle its SPEC M atan2: equal to rounding
    x = c["tone"][:5000]
    y = ref["quad_demod"]
    o = np.empty_like(x)
    prev = oracle.Cpx(0, 0); primed = C.c_int(0)
    oracle.lib().sdo_quad_demod(oracle.ptr(x), oracle.ptr(o), len(x), C.byref(prev), C.byref(primed))
    assert y[0] == 0 and np.all(y.real == 0) and np.max(np.abs(y.imag - o.imag)) < 2e-7
    # DelayedConjTask: to one ulp of cabsf (libm's hypot vs sqrtf of the sum of squares)
    for delay in (7, 500):
        x = c["tone"][:3000]
        y = ref["delayed_conj_%d" % delay]
        o = oracle.delayed_conj(x, delay)
        assert np.max(np.abs(y - o)) <= 4e-7 * np.max(np.abs(y))
    # WaveSampler MANUAL in the three decision spaces: soft symbols bit for bit
    for space, sig in (("amplitude", "ask"), ("phase", "psk"), ("frequency", "psk")):
        x = np.ascontiguousarray(c[sig][:6000])
        out = ref["manual_" + space]
        n = len(out)
        o = oracle.sample_manual(x, space, 487.3, 5)
        assert n == len(o) == 487
        assert np.array_equal(out[:n].view(np.uint32), o.view(np.uint32)), space
    # WaveSampler ZERO_CROSSING: recovered bit streams bit for bit
    for i, (sig, space, amp, thr, zc, bnor) in enumerate(G.ZC_CASES):
        x = np.ascontiguousarray(c[sig])
        sym = ref["zero_crossing_%d" % i]
        n = len(sym)
        o, k = oracle.sample_zero_crossing(x, space, bnor, amp, thr, zc)
        assert n == k and np.array_equal(sym[:n], o), (sig, space, amp)


def test_gardner_sampler_of_the_reference_over_the_clock_detector_shim(ref, oracle):
    """Tasks/WaveSampler.cpp sampleGardner() compiled from the reference, running on THIS repo's su_clock_detector
    (libsigutils.so): equal to the oracle's Gardner detector fed the same way."""
    import shim_build as SB
    x = np.ascontiguousarray(G.timewindow_case()["psk"])
    want = SB.oracle_gardner_frequency(oracle, x, 0.2, 1.0 / 12)
    assert G.sha(want) == ref["gardner_sha"]


def test_averager_restatement_equals_the_compiled_reference(ref, oracle):
    frames = G.averager_frames()
    for alpha in (0.25, 1.0):
        last = frames[0].copy()
        L = oracle.lib()
        for f in range(1, 7):
            if alpha < 1.0:
                L.sdo_averager_feed(oracle.ptr(last), oracle.ptr(np.ascontiguousarray(frames[f])), 4096, C.c_float(alpha))
            else:
                last = frames[f].copy()
        assert G.sha(last) == ref["averager_%g_sha" % alpha], alpha


@pytest.mark.parametrize("interlace,lines", [(False, 40), (True, 61)])
def test_tv_worker_of_the_reference_over_the_tvproc_shim(ref, oracle, interlace, lines):
    """Default/GenericInspector/TVProcessorWorker.cpp COMPILED FROM THE REFERENCE (setParams / start / pushData /
    process / work with its acknowledgement window / returnFrame) drives this repo's <sigutils/tvproc.h> unmodified:
    the frames it emits are, bit for bit, the oracle's (SPEC TV) and those of the reference-shaped TU."""
    import shim_build as SB
    import test_oracle_tv as T
    x, _, _ = T.toy_signal(lines, interlace, frames=10)
    sp = T.toy_params(lines, interlace, 4, cls=T.ShimTvParams)
    W, H, cap, block = int(np.floor(T.LINE)), lines, 16, 7000
    out = np.zeros((cap, H, W), np.float32)
    w, h = C.c_int(), C.c_int()
    got, rw, rh = (int(v) for v in ref["tv_%d_%d" % (interlace, lines)])
    assert got >= 5 and (rw, rh) == (W, H)
    assert SB.reference_tu().tu_tv_worker(C.byref(sp), x.ctypes.data, x.size, block, out.ctypes.data, cap,
                                          C.byref(w), C.byref(h)) == got
    assert G.sha(out) == ref["tv_%d_%d_sha" % (interlace, lines)]
    t = T.OracleTv(T.toy_params(lines, interlace, 4))
    k = 0
    for p0 in range(0, x.size, block):
        blk, sent = x[p0:p0 + block], False
        for pos in range(0, blk.size, 64):
            f0 = t.frames
            t.feed(blk[pos:pos + 64])
            if t.frames > f0 and not sent:
                assert np.array_equal(out[k].view(np.uint32), t.frame(f0).view(np.uint32))
                k, sent = k + 1, True
    assert k == got
    t.close()


def test_psd_message_of_the_reference_over_the_shim_headers(ref, oracle):
    """Suscan/Messages/PSDMessage.cpp + Suscan/Message.cpp COMPILED FROM THE REFERENCE against include/analyzer/msg.h:
    the constructor's fft-shift + SU_POWER_DB pass (:26-39) is the reference's own; the oracle's sdo_psd_shift_db
    (= the PSD kernels' SDB_FLAG_PSD_SHIFT_DB epilogue, bit for bit) is held to it -- the layout exactly, the values to
    the difference between libm's log10f and the SPEC M polynomial."""
    rng = np.random.default_rng(21)
    n = 8192
    lin = (rng.standard_normal(n) ** 2 * 10.0 ** rng.uniform(-9, 1, n)).astype(np.float32)
    lin[:4] = [0.0, 1e-12, 1.0, 123.5]
    out = ref["psd_message"]
    assert len(out) == n and list(ref["psd_message_meta"]) == [433920000.0, 2000000]
    mine = lin.copy()
    oracle.lib().sdo_psd_shift_db(oracle.ptr(mine), n)
    assert np.all(np.isfinite(out)) and out.min() >= -80.0 - 1e-3          # the 1e-8 floor of SU_POWER_DB
    assert np.max(np.abs(out - mine)) < 2e-5                                # dB; same bins in the same places
    want = 10.0 * np.log10(np.concatenate([lin[n // 2:], lin[:n // 2]]).astype(np.float64) + 1e-8)
    assert np.max(np.abs(out - want)) < 2e-5


def test_mq_and_message_wrappers_of_the_reference_over_libsuscan(ref):
    """Suscan/MQ.cpp (caller-owned suscan_mq: init / read / finalize), SamplesMessage and StatusMessage over the shim
    library: payloads posted with suscan_mq_write come back through the reference's wrapper classes and are released by
    their shared_ptr deleter (suscan_analyzer_dispose_message): the same calls from the reference-shaped TU."""
    import shim_build as SB
    tu = SB.reference_tu()
    x = G.mq_input()
    out = np.zeros_like(x)
    iid = C.c_uint()
    assert tu.tu_mq_samples(x.ctypes.data, x.size, 0xBEEF, out.ctypes.data, C.byref(iid)) == x.size
    assert iid.value == 0xBEEF and np.array_equal(out, x)
    assert list(ref["mq_samples"]) == [x.size, 0xBEEF] and G.sha(out) == ref["mq_samples_sha"]
    status = []
    for code, text in G.MQ_STATUS_CASES:
        buf = C.create_string_buffer(64)
        status += [str(tu.tu_status_message(code, text, buf, 64)), buf.value.decode()]
    assert status == list(ref["status_messages"])


def _qpsk(n, seed=5):
    from sigdigger_b200 import synth
    x, _ = synth.multi_carrier(n, 1.0, [("qpsk", 0.01, 0.1, -6.0, {})], noise_db=-40.0, seed=seed)
    return np.ascontiguousarray(x, np.complex64)


def test_tasks_of_the_reference_over_the_sigutils_shim(ref, oracle):
    """Tasks/CostasRecoveryTask.cpp, PLLSyncTask.cpp, AGCTask.cpp, CarrierXlator.cpp COMPILED FROM THE REFERENCE
    (constructor + work() loops, `destination[p] = su_costas_feed(&costas, origin[p])`) over this repo's
    <sigutils/{pll,agc,ncqo}.h> and libsigutils.so: the north-star's "Tasks/ are drop-in".  Outputs equal the oracle's
    bit for bit (the shim's per-sample entry points run the kernels' step functions on the host)."""
    import shim_build as SB
    n = 2 * 4096 + 777
    x = _qpsk(n)
    for kind in (1, 2, 3):
        assert G.sha(SB.oracle_costas(oracle, x, kind, 0.1, 2e-3)) == ref["task_costas_%d_sha" % kind]
    assert G.sha(SB.oracle_pll(oracle, x, 5e-3)) == ref["task_pll_sha"]
    assert G.sha(SB.oracle_agc(oracle, x, 20.0)) == ref["task_agc_sha"]
    assert G.sha(SB.oracle_xlate(oracle, x, 0.0123, 0.5)) == ref["task_xlate_sha"]


def test_histogram_feeder_of_the_reference(ref, oracle):
    """Tasks/HistogramFeeder.cpp compiled from the reference against the oracle's restatement (SPEC Y.2): amplitude
    exactly; phase / frequency to one ulp of libm's cargf against the SPEC M atan2."""
    L = oracle.lib()
    L.sdo_histogram_feed.restype = C.c_size_t
    L.sdo_histogram_feed.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
    n = 3 * 4096 + 55
    x = _qpsk(n, seed=8)
    for space, tol in ((0, 0.0), (1, 4e-7), (2, 4e-7)):
        got = ref["histogram_%d" % space]
        mine = np.zeros(n, np.float32)
        k = len(got)
        m = L.sdo_histogram_feed(x.ctypes.data, mine.ctypes.data, n, space)
        assert k == m == (n - 1 if space == 2 else n)
        if tol == 0.0:
            assert np.max(np.abs(got[:k] - mine[:k]) / np.maximum(np.abs(mine[:k]), 1e-30)) < 2e-7   # cabsf vs SPEC M
        else:
            d = np.abs(got[:k] - mine[:k])
            d = np.minimum(d, np.abs(d - 2 * np.pi))                  # +-pi branch
            assert d.max() < tol


def test_snr_estimator_restatement_tracks_the_compiled_reference(ref, oracle):
    """Misc/SNREstimator.cpp compiled from the reference against the oracle's restatement (SPEC Y.7): same trajectory
    of sigma over successive feeds and the same model histogram, to the difference between libm's exp and SPEC M's."""
    rng = np.random.default_rng(4)
    for bps, length in ((1, 256), (2, 256), (3, 400)):
        k = 1 << bps
        centres = (rng.integers(0, k, 200000) + 0.5) / k
        v = (centres + 0.03 * rng.standard_normal(200000)) % 1.0
        h = np.bincount((v * length).astype(int) % length, minlength=length).astype(np.uint32)
        feeds = 6
        r = ref["snr_%d_%d" % (bps, length)]
        sig, snr, model = r[:feeds], r[feeds:2 * feeds], r[2 * feeds:]
        assert len(model) == length
        e = oracle.SnrEstimator(bps, length, alpha=0.5)
        for f in range(feeds):
            e.feed(h)
            assert abs(e.sigma - sig[f]) <= 5e-5 * abs(sig[f]), (bps, f, e.sigma, sig[f])
            assert abs(e.snr - snr[f]) <= 1e-4 * abs(snr[f])
        assert np.abs(e.model() - model).max() < 5e-5
        e.close()


def test_carrier_detector_restatement_tracks_the_compiled_reference(ref, oracle):
    """Tasks/CarrierDetector.cpp compiled from the reference (Blackman-Harris taps from this repo's <sigutils/taps.h>,
    its FFT through a binary64 stand-in for FFTW) against sdo_carrier_detect (SPEC Y.5, binary32 SPEC transform): the
    same peak to the transforms' rounding."""
    rng = np.random.default_rng(12)
    for (n, f0, notch), got in zip(((5000, 0.0371, 0.0), (16384, -0.212, 0.0), (3000, 0.11, 0.05), (9000, -0.4, 0.02)),
                                   ref["carrier_detect"]):
        t = np.arange(n)
        x = (np.exp(2j * np.pi * f0 * t) * (1 + 0.3 * np.cos(2 * np.pi * 0.001 * t))
             + 0.05 * (rng.standard_normal(n) + 1j * rng.standard_normal(n)) + 0.5).astype(np.complex64)
        got = float(got)
        mine = float(oracle.carrier_detect(x, 0.01, notch))
        assert abs(got - mine) < 2e-5, (n, f0, got, mine)
        assert abs(got - 2 * np.pi * f0) < 2e-3 or notch > 0
