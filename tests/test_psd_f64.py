"""The CPU oracle's main PSD (oracle/fft.c, oracle/fft_spec.c, oracle/tasks.c) against the float64 statement of SPEC
W, P, Q, R and M.6 (tests/psd_f64.py).

The CUDA PSD is held bit for bit to the oracle; these tests hold the oracle to the SPEC, so that a mistake shared by
both sides -- a wrong window formula or denominator, a wrong bin order, a DC estimate summed or updated in the wrong
order -- cannot pass unnoticed.  Known-answer tests keep the float64 statement itself honest."""
import ctypes as C

import numpy as np
import pytest

import parity
import psd_f64 as pf

SIZES = [1 << k for k in range(4, 21)]
WINDOWED = [k for k in pf.KINDS if k != "none"]


def tone_noise(n, seed, f=0.1234, amp=0.5, noise=0.3):
    """complex64 noise plus one tone, the PSD tests' usual input."""
    rng = np.random.default_rng(seed)
    x = noise * (rng.standard_normal(n) + 1j * rng.standard_normal(n)) + amp * np.exp(2j * np.pi * f * np.arange(n))
    return x.astype(np.complex64)


def impulse_positions(N):
    return sorted({0, 1, N // 3, N // 2 - 1, N // 2, N - 2, N - 1})


def impulse_frames(N, amps):
    """One frame per position of impulse_positions(N): amps[i] at position p_i, zeros elsewhere."""
    ps = impulse_positions(N)
    x = np.zeros(len(ps) * N, np.complex64)
    for i, p in enumerate(ps):
        x[i * N + p] = amps[i % len(amps)]
    return x, ps


def impulse_expect(N, kind, ps, amps):
    """[frames] float64: |a|^2 w[p]^2 / N, the value of every bin of the impulse frame at p."""
    w = pf.window(N, kind)
    a = np.asarray([amps[i % len(amps)] for i in range(len(ps))], np.complex128)
    return np.abs(a) ** 2 * w[ps] ** 2 / N


def assert_impulse(got, N, kind, ps, amps, rtol=2e-6):
    """Every bin of each impulse frame within rtol of |a|^2 w64[p]^2 / N; exactly zero where the float32 tap is zero;
    returns the worst relative error."""
    want = impulse_expect(N, kind, ps, amps)
    w32 = pf.window(N, kind).astype(np.float32)
    worst = 0.0
    for f, p in enumerate(ps):
        g = np.asarray(got[f], np.float64)
        if w32[p] == 0:
            assert np.all(g == 0), (N, kind, p, float(np.max(np.abs(g))))
            continue
        r = float(np.max(np.abs(g - want[f])) / want[f])
        assert r <= rtol, "N %d %s impulse at %d: relative error %.3g" % (N, kind, p, r)
        worst = max(worst, r)
    return worst


IMPULSE_AMPS = [np.complex64(0.8 - 0.45j), np.complex64(-0.3 + 0.9j), np.complex64(1.0), np.complex64(-0.6j)]


# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", SIZES)
def test_oracle_psd_matches_f64_statement(oracle, N):
    """SPEC transform (oracle.psd_frames, bit-identical to the CUDA path) within T of |FFT(w x)|^2 / N in complex128,
    with windows evaluated from the SPEC W formulas, at every accepted size and window."""
    x = tone_noise(2 * N, seed=N % 113)
    for kind in pf.KINDS:
        got = oracle.psd_frames(x, N, kind)
        r = parity.psd_err_ratio(got, pf.psd(x, N, kind))
        assert r <= 1.0, "N %d %s: worst bin at %.2f x tolerance" % (N, kind, r)


@pytest.mark.parametrize("kind", WINDOWED)
def test_oracle_window_is_f64_formula_rounded_once(oracle, kind):
    """oracle.window is the SPEC W formula (denominator N - 1) rounded to binary32 once: within half an ulp, at every
    size (<= 3.0e-8 absolute below 1, <= 2.4e-7 for the flat-top's peak above 4)."""
    for N in SIZES:
        w64 = pf.window(N, kind)
        got = oracle.window(N, kind).astype(np.float64)
        half_ulp = np.spacing(np.abs(w64).astype(np.float32)).astype(np.float64) / 2
        bad = np.flatnonzero(np.abs(got - w64) > half_ulp)
        assert len(bad) == 0, (N, kind, int(bad[0]), got[bad[0]], w64[bad[0]])
        assert np.max(np.abs(got - w64)) <= (2.4e-7 if kind == "flat_top" else 3.0e-8)


def test_f64_window_known_values():
    """Symmetric form: Hann is 0 at both ends and 1 in the middle of an odd length; every window is symmetric;
    Hamming's ends are 0.08; the flat-top peaks at 4.636."""
    for N in (16, 17, 1024):
        for kind in pf.KINDS:
            w = pf.window(N, kind)
            np.testing.assert_allclose(w, w[::-1], rtol=0, atol=1e-14)
    assert pf.window(16, "hann")[0] == 0.0 and abs(pf.window(16, "hann")[15]) < 1e-16
    assert abs(pf.window(17, "hann")[8] - 1.0) < 1e-15
    assert abs(pf.window(64, "hamming")[0] - 0.08) < 1e-15
    assert abs(pf.window(17, "flat_top")[8] - 4.636) < 1e-12
    assert np.all(pf.window(64, "none") == 1.0)


@pytest.mark.parametrize("N", SIZES)
def test_impulse_probe(oracle, N):
    """A frame holding a delta[n - p] has |a|^2 w[p]^2 / N in every bin: the oracle's PSD within 2e-6 of that value
    with w from the float64 formula, and exactly zero where the tap is zero (the Hann end points)."""
    x, ps = impulse_frames(N, IMPULSE_AMPS)
    for kind in WINDOWED:
        assert_impulse(oracle.psd_frames(x, N, kind), N, kind, ps, IMPULSE_AMPS)


def test_f64_psd_known_answers():
    """The float64 statement itself: a tone on bin k puts N |a|^2 in bin k alone (no window); Parseval; shift_db
    moves bin k to (k + N/2) mod N and adds the 1e-8 floor."""
    N, k, a = 64, 5, 0.5 - 0.25j
    x = a * np.exp(2j * np.pi * k * np.arange(N) / N)
    p = pf.psd(x, N, "none")[0]
    assert abs(p[k] - N * abs(a) ** 2) < 1e-12 and np.max(np.delete(p, k)) < 1e-20
    y = np.random.default_rng(1).standard_normal(N) + 0j
    assert abs(pf.psd(y, N, "none")[0].sum() - np.sum(np.abs(y) ** 2)) < 1e-10
    d = pf.shift_db(p)
    assert d[(k + N // 2) % N] == 10 * np.log10(p[k] + 1e-8)
    assert abs(d[N // 2] - (-80.0)) < 1e-6                 # DC bin holds nothing: the floor


def test_oracle_shift_db_matches_f64(oracle):
    """sdo_psd_shift_db: halves swapped exactly, dB within the float32 rounding of SPEC M.3 / M.6."""
    for N in (16, 2048, 65536):
        p = oracle.psd_frames(tone_noise(N, seed=N), N, "hann")[0]
        q = p.copy()
        oracle.lib().sdo_psd_shift_db(oracle.ptr(q), N)
        want = pf.shift_db(p.astype(np.float64))
        bound = 1.5e-6 * np.abs(want) + np.spacing(np.abs(want).astype(np.float32))
        assert np.all(np.abs(q - want) <= bound), (N, float(np.max(np.abs(q - want) - bound)))


def _dc_oracle(oracle, blocks, fs):
    L = oracle.lib()
    c = (C.c_float * 2)(0.0, 0.0)
    out = []
    for b in blocks:
        b = np.ascontiguousarray(b, np.complex64)
        y = np.empty_like(b)
        alpha = np.float32(1.0 - np.exp(-len(b) / (fs * 0.1)))
        L.sdo_dc_remove(c, oracle.ptr(b), oracle.ptr(y), C.c_size_t(len(b)), C.c_float(float(alpha)))
        out.append(y)
    return out


def test_dc_remove_statement_is_oracle_bit_for_bit(oracle):
    """SPEC R as written equals sdo_dc_remove bit for bit over blocks shorter than one run (48), with a partial run
    (80, 300) and over many runs with a partial last one (65536 + 17), with a large DC offset and a small signal so
    that the order of the binary64 sums shows in the rounded mean."""
    fs = 1000.0
    rng = np.random.default_rng(7)
    sizes = [48, 80, 300, 65536 + 17, 48]
    blocks = []
    for i, n in enumerate(sizes):
        b = 1e-3 * (rng.standard_normal(n) + 1j * rng.standard_normal(n)) + (0.7 - 0.31j) * (1 + 0.1 * i)
        blocks.append(b.astype(np.complex64))
    got = pf.dc_remove(blocks, fs)
    ref = _dc_oracle(oracle, blocks, fs)
    for g, r in zip(got, ref):
        assert np.array_equal(g.view(np.uint32), r.view(np.uint32))
    # the estimate moves: the last block's residual DC is far below the first's
    assert abs(got[-1].mean()) < 0.5 * abs(got[0].mean())


def test_dc_remove_sums_in_runs_of_256():
    """The statement's binary64 mean is the two-level sum of SPEC R: 1 + 2^-53 rounds back to 1, so a run that
    starts with 1 loses its small terms while a run that starts with them keeps their sum."""
    e = 2.0 ** -53
    v = np.array([1.0] + [e] * 255 + [e] * 255 + [1.0], np.float64)
    assert pf._block_sum(v) == 1.0 + (255 * e + 1.0)
    assert pf._block_sum(v) != pf._seq_sum(v)
    assert pf._seq_sum(np.array([1.0, e, e])) == 1.0
    assert pf._seq_sum(np.array([e, e, 1.0])) == 1.0 + 2 * e


@pytest.mark.parametrize("fmt", ["f32", "u8", "s8", "s16"])
def test_convert_is_exact(fmt):
    """SPEC Q: every code of the 8-bit formats and the 16-bit extremes convert exactly; iq_reverse swaps the pair."""
    if fmt == "f32":
        x = np.array([0.25 - 0.5j, 1e-30 + 3j], np.complex64)
        assert np.array_equal(pf.convert(x, fmt), x)
        assert np.array_equal(pf.convert(x, fmt, True), (x.imag + 1j * x.real).astype(np.complex64))
        return
    dt = {"u8": np.uint8, "s8": np.int8, "s16": np.int16}[fmt]
    info = np.iinfo(dt)
    codes = np.arange(info.min, info.max + 1) if fmt != "s16" else np.array([info.min, -1, 0, 1, 12345, info.max])
    raw = np.stack([codes, codes[::-1]], axis=-1).astype(dt)
    scale, off = {"u8": (128.0, 128.0), "s8": (128.0, 0.0), "s16": (32768.0, 0.0)}[fmt]
    want = ((codes - off) / scale) + 1j * ((codes[::-1] - off) / scale)
    assert np.array_equal(pf.convert(raw, fmt).astype(np.complex128), want)
    assert np.array_equal(pf.convert(raw, fmt, True).astype(np.complex128), want.imag + 1j * want.real)
