"""The CPU oracle's inspector chains (oracle/inspector.c, oracle/dsp.c, oracle/math.c) against the exact binary32
statement of SPEC M, I, N, A, C, G, E, D and X (tests/chain_stmt.py).

The CUDA inspectors are held bit for bit to the oracle; these tests hold the oracle to the SPEC: the elementary
functions over dense grids and their edges, every design, every stage, and every chain over a matrix of classes,
flags, symbol periods and inputs, bit for bit.  A statement with one deliberate mistake is rejected by a named case."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import chain_cases as cc
import chain_stmt as cs
import oracle_lib
import shim_build

_GRID_SRC = r"""
#include <stddef.h>
void sdo_sincosf(float x, float *s, float *c);
float sdo_atan2f(float y, float x);
float sdo_log10f(float x);
float sdo_exp10f(float x);
void g_sincos(const float *x, float *s, float *c, size_t n) { for (size_t i = 0; i < n; ++i) sdo_sincosf(x[i], s + i, c + i); }
void g_atan2(const float *y, const float *x, float *o, size_t n) { for (size_t i = 0; i < n; ++i) o[i] = sdo_atan2f(y[i], x[i]); }
void g_log10(const float *x, float *o, size_t n) { for (size_t i = 0; i < n; ++i) o[i] = sdo_log10f(x[i]); }
void g_exp10(const float *x, float *o, size_t n) { for (size_t i = 0; i < n; ++i) o[i] = sdo_exp10f(x[i]); }
"""
_grid = None


def grid_lib(oracle):
    """the oracle's M functions looped in C over arrays (a Python loop over ctypes calls is too slow for dense grids)"""
    global _grid
    if _grid is None:
        d = shim_build.build_dir()
        src, so = os.path.join(d, "mgrid.c"), os.path.join(d, "libmgrid.so")
        with open(src, "w") as f:
            f.write(_GRID_SRC)
        libdir = os.path.dirname(oracle.LIB_PATH)
        subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", src, "-o", so, "-L", libdir,
                        "-lsdoracle", "-Wl,-rpath," + libdir, "-lm"], check=True)
        _grid = C.CDLL(so)
    return _grid


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def assert_same(got, ref, what):
    bad = np.flatnonzero(bits(np.asarray(got, np.float32)) != bits(np.asarray(ref, np.float32)))
    assert bad.size == 0, (what, bad.size, bad[:5])


def around(v, ulps):
    """float32 values within `ulps` ulps of each v"""
    v = np.asarray(v, np.float32)
    k = np.arange(-ulps, ulps + 1, dtype=np.int64)
    b = v.view(np.int32).astype(np.int64)[:, None] + k[None, :]
    return b.astype(np.int32).view(np.float32).ravel()


# ---- binary32 fma ---------------------------------------------------------------------------------------------------
def test_fma32_equals_libm_fmaf():
    """The statement's fma32 against glibc's fmaf on 200 000 triples, a quarter of them cancelling exactly or nearly."""
    libm = C.CDLL("libm.so.6")
    libm.fmaf.restype = C.c_float
    libm.fmaf.argtypes = [C.c_float] * 3
    rng = np.random.default_rng(1)
    n = 200000
    a = (rng.standard_normal(n) * 2.0 ** rng.integers(-30, 30, n)).astype(np.float32)
    b = (rng.standard_normal(n) * 2.0 ** rng.integers(-30, 30, n)).astype(np.float32)
    c = (rng.standard_normal(n) * 2.0 ** rng.integers(-60, 60, n)).astype(np.float32)
    cancel = rng.random(n) < 0.25
    c[cancel] = -(a[cancel] * b[cancel]) * (1 + rng.integers(-2, 3, cancel.sum()) * 2.0 ** -23)
    c = c.astype(np.float32)
    ref = np.array([libm.fmaf(x, y, z) for x, y, z in zip(a.tolist(), b.tolist(), c.tolist())], np.float32)
    assert_same(cs.fma32(a, b, c), ref, "fma")
    assert cs.fma32(np.float32(1 + 2 ** -23), np.float32(1 - 2 ** -23), np.float32(-1)) == np.float32(-2.0 ** -46)


# ---- M: elementary functions over dense grids -----------------------------------------------------------------------
def test_sincos_grid(oracle):
    """M.1 on 4M points over [-64, 64] plus the quadrant boundaries of rint(x 2/pi), where q flips."""
    rng = np.random.default_rng(2)
    x = np.concatenate([rng.uniform(-64, 64, 1 << 22), np.linspace(-7, 7, 1 << 20),
                        around((np.arange(-40, 41) + 0.5) * (np.pi / 2), 200),
                        around(np.arange(-40, 41) * (np.pi / 2), 50), [0.0, -0.0]]).astype(np.float32)
    s, c = np.empty_like(x), np.empty_like(x)
    grid_lib(oracle).g_sincos(oracle.ptr(x), oracle.ptr(s), oracle.ptr(c), C.c_size_t(x.size))
    gs, gc = cs.sincos(x)
    assert_same(gs, s, "sin")
    assert_same(gc, c, "cos")


def test_atan2_grid(oracle):
    """M.2 on 4M pairs of every sign and magnitude, |y|/|x| within a few ulps of 0.41421356 and 2.41421356, zeros of
    either argument, and x = 0."""
    rng = np.random.default_rng(3)
    n = 1 << 22
    sgn = lambda k: np.where(rng.random(k) < 0.5, -1.0, 1.0)
    x = sgn(n) * 10.0 ** rng.uniform(-6, 6, n)
    y = sgn(n) * 10.0 ** rng.uniform(-6, 6, n)
    xb = (sgn(4000) * 10.0 ** rng.uniform(-3, 3, 4000)).astype(np.float32)
    ys = []
    for r in (0.4142135623730950, 2.414213562373095, 1.0):
        yb = np.float32(r) * np.abs(xb)
        ys.append(np.stack([xb.repeat(41), around(yb, 20) * np.tile(sgn(41), 4000)]))
    edge = np.stack([np.repeat(xb, 1)[:1000], np.zeros(1000)])
    yy = np.concatenate([y] + [v[1] for v in ys] + [edge[1], xb[:1000], np.zeros(3), -np.zeros(1)])
    xx = np.concatenate([x] + [v[0] for v in ys] + [edge[0], np.zeros(1000), [0.0, -0.0, 1.0], [-1.0]])
    yy, xx = yy.astype(np.float32), xx.astype(np.float32)
    o = np.empty_like(xx)
    grid_lib(oracle).g_atan2(oracle.ptr(yy), oracle.ptr(xx), oracle.ptr(o), C.c_size_t(xx.size))
    assert_same(cs.atan2(yy, xx), o, "atan2")


def test_log10_grid(oracle):
    """M.3 on every binary exponent including the subnormals, with mantissas on both sides of sqrt(1/2) (the split
    constant 1.41421356f) and random ones."""
    rng = np.random.default_rng(4)
    exps = np.arange(0, 255, dtype=np.uint32)
    mant = np.concatenate([rng.integers(1, 1 << 23, 8000), np.arange(0x3504F3 - 200, 0x3504F3 + 200), [0, 1],
                           [(1 << 23) - 1]]).astype(np.uint32)
    x = ((exps[:, None] << np.uint32(23)) | mant[None, :]).ravel().view(np.float32)
    x = x[x > 0]
    o = np.empty_like(x)
    grid_lib(oracle).g_log10(oracle.ptr(x), oracle.ptr(o), C.c_size_t(x.size))
    assert_same(cs.log10(x), o, "log10")


def test_exp10_grid(oracle):
    """M.4 on 2M points over [-45, 45], around the clamp edges -37 and 38, and around the rounding boundaries of
    p = floor(3.3219 x + 0.5)."""
    rng = np.random.default_rng(5)
    k = np.arange(-130, 131)
    x = np.concatenate([rng.uniform(-45, 45, 1 << 21), around([-37.0, 38.0], 500),
                        around((k - 0.5) / 3.32192809488736234787, 100)]).astype(np.float32)
    o = np.empty_like(x)
    grid_lib(oracle).g_exp10(oracle.ptr(x), oracle.ptr(o), C.c_size_t(x.size))
    assert_same(cs.exp10(x), o, "exp10")


# ---- designs --------------------------------------------------------------------------------------------------------
T_DESIGN = np.concatenate([np.linspace(1.0, 40.0, 157), np.linspace(40.0, 1100.0, 60), np.linspace(170.5, 171.0, 21),
                           [34.8, 34.9, 13.8, 13.9, 4.09, 4.10, 1048.6, 1048.7]]).astype(np.float32)


def test_mf_design(oracle):
    """I.2: sdo_mf_span and sdo_taps_rrc at T across 1 ... 1100, densely around the 1024-tap cap (T 170.5 ... 171)."""
    L = oracle.lib()
    for T in T_DESIGN:
        n = cs.mf_span(T)
        assert n == L.sdo_mf_span(C.c_float(T)), T
        for beta in (0.35, 0.5):
            h = np.empty(n, np.float32)
            L.sdo_taps_rrc(h.ctypes.data_as(oracle.c_float_p), n, C.c_float(T), C.c_float(beta))
            assert_same(cs.taps_rrc(n, T, beta), h, ("rrc", float(T), beta))
    assert cs.mf_span(np.float32(170.5)) == 1023 and cs.mf_span(np.float32(171.0)) == 1024


def test_butter_design(oracle):
    """I.4 at orders 2 (the Costas arm filter) and 4 (the audio low-pass) over the clamp ranges they use."""
    L = oracle.lib()
    for order in (2, 4):
        for fc in np.concatenate([np.geomspace(1e-4, 0.95, 120), [1e-3, 0.5, 0.95]]).astype(np.float32):
            b, a = np.empty(order + 1, np.float32), np.empty(order + 1, np.float32)
            assert L.sdo_butter_lp(order, C.c_float(fc), b.ctypes.data_as(oracle.c_float_p),
                                   a.ctypes.data_as(oracle.c_float_p)) == 0
            gb, ga = cs.butter_lp(order, fc)
            assert_same(gb, b, ("b", order, float(fc)))
            assert_same(ga, a, ("a", order, float(fc)))


def agc_boundary_taus():
    """T where tau (rise 10) or tau (rise 5) lies within an ulp or two of an integer: the floors that set the line
    sizes, hence the kernel's AGC path, flip there."""
    rise = np.float32(3.9062e-1)
    out = []
    for mul in (np.float32(10.0) * rise, rise * np.float32(5.0)):
        k = np.concatenate([np.arange(1, 80), [150, 159, 160, 161, 4095, 4096, 4097, 8191]])
        out.append(around((k / np.float64(mul)).astype(np.float32), 3))
    return np.concatenate(out + [np.float32([1.0, 2.0, 13.8, 13.9, 1048.5, 1048.6, 1048.7, 5000.0])])


def test_agc_design(oracle):
    """A: sdo_agc_params_from_tau and the constants of sdo_agc_init at T on both sides of every size boundary."""
    L = oracle.lib()
    flips = 0
    for T in agc_boundary_taus():
        if not T >= 1.0:
            continue
        p = oracle.AgcParams()
        L.sdo_agc_params_from_tau(C.byref(p), C.c_float(T), C.c_float(1.0))
        d = cs.AgcDesign(T, 1.0)
        assert (p.hang_max, p.delay_line_size, p.mag_history_size) == (d.hang_max, d.dl_size, d.mh_size), T
        assert_same([p.fast_rise_t, p.fast_fall_t, p.slow_rise_t, p.slow_fall_t],
                    [d.fast_rise_t, d.fast_fall_t, d.slow_rise_t, d.slow_fall_t], ("times", float(T)))
        a = oracle.Agc()
        assert L.sdo_agc_init(C.byref(a), C.byref(p)) == 0
        assert_same([a.fast_alpha_rise, a.fast_alpha_fall, a.slow_alpha_rise, a.slow_alpha_fall, a.fixed_gain,
                     a.gain_slope], [d.far, d.faf, d.sar, d.saf, d.fixed_gain, d.gain_slope], ("alphas", float(T)))
        L.sdo_agc_free(C.byref(a))
        exact = float(T) * float(np.float32(10.0) * np.float32(3.9062e-1))
        flips += d.dl_size != int(exact) and d.dl_size < 4096
    assert flips > 0       # somewhere the binary32 product floors differently from the exact one
    assert cs.AgcDesign(np.float32(1100.0)).dl_size == 4096


def test_loop_designs(oracle):
    """C: the PLL and Costas coefficients."""
    L = oracle.lib()
    for bw in np.geomspace(1e-5, 0.5, 40).astype(np.float32):
        p = oracle.Pll()
        L.sdo_pll_init(C.byref(p), 0.0, C.c_float(bw))
        assert_same([p.alpha, p.beta], cs.pll_design(bw), ("pll", float(bw)))
        c = oracle.Costas()
        assert L.sdo_costas_init(C.byref(c), 2, 0.0, C.c_float(0.5), 3, C.c_float(bw)) == 0
        assert_same([c.a, c.b], cs.costas_design(bw), ("costas", float(bw)))
        L.sdo_costas_free(C.byref(c))


# ---- stages ---------------------------------------------------------------------------------------------------------
def _cpx_in(n, seed):
    x = cc.inputs("psk", 4.0, n, seed)
    return x[[1, 3]]


def _feed(fn, obj, x):
    out = np.empty(len(x), np.complex64)
    for i, v in enumerate(x):
        r = fn(C.byref(obj), oracle_cpx(v))
        out[i] = complex(r.re, r.im)
    return out


def oracle_cpx(v):
    return oracle_lib.Cpx(float(v.real), float(v.imag))


def assert_cpx(got, ref, what):
    assert len(got) == len(ref), (what, len(got), len(ref))
    assert_same(np.asarray(got, np.complex64).view(np.float32), np.asarray(ref, np.complex64).view(np.float32), what)


@pytest.mark.parametrize("T", [2.5, 4.0, 13.9])
def test_stage_agc(oracle, T):
    L = oracle.lib()
    x = _cpx_in(2500, 7)
    d = cs.AgcDesign(np.float32(T))
    gr, gi = cs.agc(x.real.copy(), x.imag.copy(), d)
    for b in range(len(x)):
        p = oracle.AgcParams()
        L.sdo_agc_params_from_tau(C.byref(p), C.c_float(T), C.c_float(1.0))
        a = oracle.Agc()
        L.sdo_agc_init(C.byref(a), C.byref(p))
        ref = _feed(L.sdo_agc_feed, a, x[b])
        L.sdo_agc_free(C.byref(a))
        assert_cpx(gr[b] + 1j * gi[b], ref, ("agc", T, b))


@pytest.mark.parametrize("kind", [1, 2, 3])
def test_stage_costas(oracle, kind):
    L = oracle.lib()
    x = _cpx_in(2500, 8)
    arm, loop = np.float32(0.5), np.float32(4e-3)
    b, a = cs.butter_lp(2, arm)
    gr, gi = cs.costas(x.real.copy(), x.imag.copy(), kind, *cs.costas_design(loop), b, a)
    for k in range(len(x)):
        c = oracle.Costas()
        assert L.sdo_costas_init(C.byref(c), kind, 0.0, C.c_float(arm), 3, C.c_float(loop)) == 0
        ref = _feed(L.sdo_costas_feed, c, x[k])
        L.sdo_costas_free(C.byref(c))
        assert_cpx(gr[k] + 1j * gi[k], ref, ("costas", kind, k))


def test_stage_pll(oracle):
    L = oracle.lib()
    x = cc.inputs("ask", 6.25, 2500, 9)[[1, 3]]
    bw = np.float32(1e-2)
    gr, gi = cs.pll(x.real.copy(), x.imag.copy(), *cs.pll_design(bw))
    for k in range(len(x)):
        p = oracle.Pll()
        L.sdo_pll_init(C.byref(p), 0.0, C.c_float(bw))
        assert_cpx(gr[k] + 1j * gi[k], _feed(L.sdo_pll_track, p, x[k]), ("pll", k))


def _clock_ref(oracle, feed, x):
    out = []
    o = oracle.Cpx()
    for v in x:
        if feed(oracle_cpx(v), o):
            out.append(complex(o.re, o.im))
    return np.array(out, np.complex64)


@pytest.mark.parametrize("T", [1.0, 2.5, 4.0, 13.9])
def test_stage_clocks(oracle, T):
    """G: Gardner and the manual sampler (phase 0 and 0.3)."""
    L = oracle.lib()
    x = _cpx_in(2000, 10)
    bnor = np.float32(1.0) / np.float32(T)
    sr, si, em = cs.gardner(x.real.copy(), x.imag.copy(), bnor, 0.2)
    for k in range(len(x)):
        cd = oracle.Clock()
        L.sdo_clock_init(C.byref(cd), C.c_float(0.2), C.c_float(bnor))
        ref = _clock_ref(oracle, lambda v, o: L.sdo_clock_feed(C.byref(cd), v, C.byref(o)), x[k])
        assert_cpx(sr[k][em[k]] + 1j * si[k][em[k]], ref, ("gardner", T, k))
    for ph in (0.0, 0.3):
        sr, si, em = cs.sampler(x.real.copy(), x.imag.copy(), bnor, ph)
        for k in range(len(x)):
            s = oracle.Sampler()
            L.sdo_sampler_init(C.byref(s), C.c_float(bnor))
            L.sdo_sampler_set_phase(C.byref(s), C.c_float(ph))
            ref = _clock_ref(oracle, lambda v, o: L.sdo_sampler_feed(C.byref(s), v, C.byref(o)), x[k])
            assert_cpx(sr[k][em[k]] + 1j * si[k][em[k]], ref, ("sampler", T, ph, k))


class Equalizer(C.Structure):
    _fields_ = [("mu", C.c_float), ("locked", C.c_int), ("w", oracle_lib.Cpx * cs.EQ_LEN),
                ("x", oracle_lib.Cpx * cs.EQ_LEN)]


@pytest.mark.parametrize("locked", [0, 1])
def test_stage_cma(oracle, locked):
    """E: lanes of different lengths in lockstep."""
    L = oracle.lib()
    L.sdo_equalizer_feed.restype = oracle.Cpx
    L.sdo_equalizer_feed.argtypes = [C.c_void_p, oracle.Cpx]
    L.sdo_equalizer_init.argtypes = [C.c_void_p, C.c_float, C.c_int]
    x = cc.inputs("psk", 4.0, 800, 11)
    syms = [x[1][:700] * 3, x[3][:500], x[0][:1]]
    got = cs.cma(syms, 2e-2, locked)
    for k, s in enumerate(syms):
        e = Equalizer()
        L.sdo_equalizer_init(C.byref(e), C.c_float(2e-2), locked)
        assert_cpx(got[k], _feed(L.sdo_equalizer_feed, e, s), ("cma", locked, k))


def test_stage_ncqo(oracle):
    """N: the LO of the manual offset and of USB / LSB, at positive and negative frequencies."""
    L = oracle.lib()
    n = 3000
    for fnor in np.float32([1e-3, -2.5e-2, 0.3, -0.97]):
        o = oracle.Ncqo()
        L.sdo_ncqo_init(C.byref(o), C.c_float(fnor))
        ref = np.array([(lambda r: complex(r.re, r.im))(L.sdo_ncqo_read(C.byref(o))) for _ in range(n)], np.complex64)
        s, c = cs.sincos(cs.ncqo_phases(1, n, cs.PI_F * fnor)[0])
        assert_cpx(c + 1j * s, ref, ("ncqo", float(fnor)))


def _filt_ref(oracle, na, a, b, x):
    L = oracle.lib()
    f = oracle.Filt()
    a = np.asarray(a, np.float32)
    b = np.asarray(b, np.float32)
    assert L.sdo_filt_init(C.byref(f), na, a.ctypes.data_as(oracle.c_float_p) if na else None, len(b),
                           b.ctypes.data_as(oracle.c_float_p)) == 0
    out = _feed(L.sdo_filt_feed, f, x)
    L.sdo_filt_free(C.byref(f))
    return out


@pytest.mark.parametrize("T", [3.1, 34.9, 171.0])
def test_stage_matched_filter(oracle, T):
    """I.1 / I.2: the RRC matched filter, taps in ascending order, one fma each, from a zero line."""
    x = _cpx_in(1500, 13)
    T = np.float32(T)
    h = cs.taps_rrc(cs.mf_span(T), T, 0.35)
    gr, gi = cs.fir(x.real.copy(), x.imag.copy(), h)
    for k in range(len(x)):
        assert_cpx(gr[k] + 1j * gi[k], _filt_ref(oracle, 0, [], h, x[k]), ("mf", float(T), k))


@pytest.mark.parametrize("order,fc", [(2, 0.5), (2, 0.05), (4, 0.05), (4, 1e-3)])
def test_stage_butterworth(oracle, order, fc):
    """I.1 / I.4: the Costas arm filter (order 2) and the audio low-pass (order 4), every term one fma."""
    x = _cpx_in(1500, 14)
    b, a = cs.butter_lp(order, np.float32(fc))
    f = cs.Iir(b, a, len(x))
    got = np.stack([f.feed(np.stack([x[:, t].real, x[:, t].imag]).astype(np.float32)) for t in range(x.shape[1])],
                   axis=-1)
    for k in range(len(x)):
        assert_cpx(got[0, k] + 1j * got[1, k], _filt_ref(oracle, order + 1, a, b, x[k]), ("iir", order, fc, k))


def test_stage_discriminator(oracle):
    """X: the fsk / FM discriminator atan2(y conj(prev)) / pi, prev starting at 0, against sdo_quad_demod (which
    writes the same value into the imaginary part, and 0 for its first sample)."""
    x = cc.inputs("fsk", 5.0, 3000, 15)
    dr, di = cs.discriminator(x.real.copy(), x.imag.copy())
    v = cs.atan2(di, dr) * np.float32(1.0 / np.pi)
    L = oracle.lib()
    for k in range(len(x)):
        y = np.empty_like(x[k])
        prev, primed = oracle.Cpx(), C.c_int(0)
        L.sdo_quad_demod(oracle.ptr(x[k]), oracle.ptr(y), len(y), C.byref(prev), C.byref(primed))
        assert_same(v[k], y.imag, ("discriminator", k))
        assert np.all(y.real == 0) and v[k][0] == 0


@pytest.mark.parametrize("mode,bps", [(0, 1), (0, 2), (0, 3), (1, 1), (1, 2)])
def test_stage_decider(oracle, mode, bps):
    """D on random symbols, the axes, exact multiples of the interval width and |x| past 1."""
    rng = np.random.default_rng(12)
    v = (rng.standard_normal(20000) + 1j * rng.standard_normal(20000)).astype(np.complex64)
    ang = np.arange(-16, 17) * (np.pi / 8)
    edge = np.concatenate([np.exp(1j * ang), [-1 + 0j, 1, 1j, -1j, 0, -1 - 0j], np.linspace(0, 2, 64)])
    v = np.concatenate([v, edge]).astype(np.complex64)
    ref = oracle.decide(v, ("argument", "modulus")[mode], bps, *((-np.pi, np.pi), (0.0, 1.0))[mode])
    assert np.array_equal(cs.decide(v, mode, bps), ref)


# ---- chains ---------------------------------------------------------------------------------------------------------
def cfg_dict(oracle, c):
    return {k: getattr(c, k) for k, _ in oracle.InspConfig._fields_}


def run_case(oracle, name, cls, fs, kw, n, mistake=None, lanes=None):
    """Runs one case on the oracle and on the statement; returns the lanes where they differ."""
    x = cc.case_inputs(cls, fs, kw, n)
    if lanes is not None:
        x = x[lanes]
    cfg = oracle.insp_config(cc.insp_class(cls), fs, **kw)
    st = cs.run(cfg_dict(oracle, cfg), x, mistake=mistake)
    bad = []
    for b in range(len(x)):
        rs, rh = oracle.inspector_run(cfg, x[b])
        ss, sh = st[b]
        if len(rs) != len(ss) or not np.array_equal(rs.view(np.uint64), ss.view(np.uint64)) or \
                not np.array_equal(rh, sh):
            bad.append(b)
    return bad


CASES = {c[0]: c[1:] for c in cc.cases() + cc.audio_cases()}


@pytest.mark.parametrize("name", list(CASES))
def test_chain_equals_statement(oracle, name):
    """soft symbols (bits), hard symbols and counts, on noise, a capture, zeros and a 30 dB step"""
    assert run_case(oracle, name, *CASES[name]) == []


def test_case_edges_hold(oracle):
    """The T ladder reaches the design boundaries it is named for, and the cases produce symbols."""
    L = oracle.lib()
    sizes = {T: (cs.AgcDesign(np.float32(1.0) / (np.float32(1.0) / np.float32(T))).dl_size,
                 cs.mf_span(np.float32(1.0) / (np.float32(1.0) / np.float32(T)))) for T in cc.T_LADDER}
    assert sizes[4.09][0] < 16 <= sizes[4.10][0]                  # the delay line moves out of the track warp
    assert 2 * sizes[13.8][0] + sizes[13.8][0] <= 160 < 3 * sizes[13.9][0]   # the AGC lines move to the pool
    assert sizes[34.8][1] <= 209 < sizes[34.9][1]                 # the matched filter leaves the ring
    assert sizes[171.0][1] == 1024 and sizes[1100.0][0] == 4096   # both caps
    assert L.sdo_mf_span(C.c_float(1100.0)) == 1024
    cfg = oracle.insp_config("psk", 1.0, **CASES["psk_baud_above_fs"][2])
    assert cfg.baud > cfg.fs and cs.bnor_of(cfg_dict(oracle, cfg)) == 1.0   # the clamp acts
    # every case but the one that never emits carries signal through to the output: on noise, the capture and the
    # step, each lane emits at least 5 non-zero symbols (at T = 1100 the input outlasts the 4096-sample line)
    for name, (cls, fs, kw, n) in CASES.items():
        x = cc.case_inputs(cls, fs, kw, n)
        cfg = oracle.insp_config(cc.insp_class(cls), fs, **kw)
        for b in (0, 1, 3):
            soft, _ = oracle.inspector_run(cfg, x[b])
            assert (np.count_nonzero(soft) >= 5) == (name != "psk_not_running_T4"), (name, b)


# deliberate mistake -> (case, lanes) that must catch it
MISTAKE_CASES = {
    "gardner_gt": ("psk_qpsk_T4", [1]),
    "hang_gt": ("psk_qpsk_T4", [3]),
    "8psk_larger": ("psk_8psk_T5", [1]),
    "pll_phase_pre": ("ask_pll1_ch1_T6.25", [1]),
    "mf_rounded": ("psk_qpsk_T4", [1]),
    "cma_unshifted": ("psk_cma_T4", [1]),
    "no_clamp": ("ask_agcoff_gain12_T6.25", [1]),
    "rs_no_clamp": ("audio_fm_rate_above_fs", [1]),
}


@pytest.mark.parametrize("mistake", cs.MISTAKES)
def test_statement_mistakes_are_caught(oracle, mistake):
    """Each planted mistake makes its named case disagree with the oracle, which the correct statement matches."""
    name, lanes = MISTAKE_CASES[mistake]
    assert run_case(oracle, name, *CASES[name], lanes=lanes) == []
    assert run_case(oracle, name, *CASES[name], mistake=mistake, lanes=lanes) != [], (mistake, name)
