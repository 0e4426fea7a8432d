"""SPEC L (source decimation, oracle/SPEC_L.md) held to a float64 statement written from the SPEC text alone: the oracle's
sdo_decimate against numpy in binary64 for every D in 1..16, 64 and 256 and all four sample formats; known answers
(delay, DC gain, passband gain, stopband attenuation); ragged feeds bit-identical to one feed; and statements with a
deliberate mistake that the comparison must reject."""
import numpy as np
import pytest

import decim_oracle

DS = list(range(1, 17)) + [64, 256]
FORMATS = ["f32", "u8", "s8", "s16"]

# least attenuation of the float64 response over 0.65 fs/D <= |f| <= fs/2 (Hamming sidelobes): 56.47 dB at D = 2,
# 59.2-59.9 dB for every other D in DS (D = 1 has no stopband)
STOP_DB = 56.0


# ---- the float64 statement (SPEC L, with SPEC I.3 taps and SPEC Q formats) -----------------------------------------
def spec_taps(D):
    n = 16 * D + 1
    fc = float(np.float32(1.0 / D))
    i = np.arange(n, dtype=np.float64)
    t = i - (n >> 1)
    xx = np.pi * fc * t
    with np.errstate(invalid="ignore", divide="ignore"):
        v = np.where(np.abs(xx) < 1e-12, fc, fc * np.sin(xx) / xx)
    v = v * (0.54 - 0.46 * np.cos(2.0 * np.pi * i / (n - 1)))
    return v.astype(np.float32)


def spec_convert(x, fmt):
    if fmt == "f32":
        return np.asarray(x, np.complex64).astype(np.complex128)
    v = np.asarray(x).astype(np.float64)
    v = {"u8": (v - 128.0) / 128.0, "s8": v / 128.0, "s16": v / 32768.0}[fmt]
    return v[0::2] + 1j * v[1::2]


def spec_decimate(x, D, h=None, offset=0):
    """y[k] = sum_i h_i x[kD - i], x[j < 0] = 0, for every k with 0 <= kD - offset < len(x) (offset: samples of the
    stream before x, so that output indices are global)"""
    h = spec_taps(D) if h is None else h
    full = np.convolve(x, h.astype(np.float64))[:len(x)]
    first = (-offset) % D
    return full[first::D]


def tolerance(x, D, h=None):
    """SPEC T style: a relative term plus the float32 accumulation noise of 16 D + 1 fused terms (sqrt(n) growth, x4)"""
    h = spec_taps(D) if h is None else h
    mag = np.convolve(np.abs(x), np.abs(h.astype(np.float64)))[:len(x)]
    return 4.0 * 2.0 ** -24 * np.sqrt(len(h)) * mag


def agrees(y, x, D, ref=None):
    ref = spec_decimate(x, D) if ref is None else ref
    if len(y) != len(ref):
        return False
    tol = tolerance(x, D)[::D][:len(ref)] + 1e-5 * np.sqrt(np.mean(np.abs(ref) ** 2))
    return bool(np.all(np.abs(y - ref) <= tol))


def make_input(fmt, m, seed):
    rng = np.random.default_rng(seed)
    if fmt == "f32":
        return (0.3 * (rng.standard_normal(m) + 1j * rng.standard_normal(m))).astype(np.complex64)
    if fmt == "u8":
        return rng.integers(0, 256, 2 * m, dtype=np.uint8)
    if fmt == "s8":
        return rng.integers(-128, 128, 2 * m, dtype=np.int8)
    return rng.integers(-32768, 32768, 2 * m, dtype=np.int16)


def feed_rows(x, fmt, a, b):
    return x[a:b] if fmt == "f32" else x[2 * a:2 * b]


# ---- oracle vs the statement -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("D", DS)
def test_oracle_matches_f64_statement(D, fmt):
    m = 40 * D + 7
    x = make_input(fmt, m, seed=D * 7 + FORMATS.index(fmt))
    dec = decim_oracle.Decimator(D, fmt)
    taps = dec.taps
    assert len(taps) == 16 * D + 1
    assert np.allclose(taps, spec_taps(D), rtol=2 ** -23, atol=1e-30)
    # two feeds, so the carry is part of what is compared
    cut = 13 * D + 3
    y = np.concatenate([dec.feed(feed_rows(x, fmt, 0, cut)), dec.feed(feed_rows(x, fmt, cut, m))])
    assert len(y) == (m + D - 1) // D
    assert agrees(y, spec_convert(x, fmt), D)


@pytest.mark.parametrize("D", [1, 2, 3, 8, 64])
def test_deliberate_mistakes_are_rejected(D):
    """The comparison must fail for a statement that takes output k at kD - 1, or one that forgets the carry."""
    m = 40 * D + 7
    x = make_input("f32", m, seed=100 + D)
    xc = spec_convert(x, "f32")
    dec = decim_oracle.Decimator(D)
    cut = 13 * D + 3
    y = np.concatenate([dec.feed(x[:cut]), dec.feed(x[cut:])])
    assert agrees(y, xc, D)
    shifted = np.convolve(xc, spec_taps(D).astype(np.float64))[:m]
    shifted = np.concatenate([[0.0], shifted])[:m][::D]                # output at kD - 1
    assert not agrees(y, xc, D, ref=shifted)
    no_carry = np.concatenate([spec_decimate(xc[:cut], D), spec_decimate(xc[cut:], D, offset=cut)])
    assert not agrees(y, xc, D, ref=no_carry)


# ---- known answers ---------------------------------------------------------------------------------------------------
def test_d1_is_the_input_delayed_by_8():
    h = spec_taps(1)
    assert h[8] == np.float32(1.0)
    off = np.delete(np.abs(h), 8)
    assert off.max() < 1e-15                       # binary64 sinc residues at the integer offsets
    x = make_input("f32", 1000, seed=5)
    y = decim_oracle.Decimator(1).feed(x)
    ref = np.concatenate([np.zeros(8, np.complex64), x[:-8]])
    assert np.max(np.abs(y - ref)) <= off.sum() * np.abs(x).max() * 2


@pytest.mark.parametrize("D", DS)
def test_dc_gain_is_the_tap_sum(D):
    h = spec_taps(D)
    x = np.ones(40 * D, np.complex64)
    y = decim_oracle.Decimator(D).feed(x)
    g = float(np.sum(h.astype(np.float64)))
    steady = y[17:]
    assert np.all(np.abs(steady.real - g) <= 4.0 * 2.0 ** -24 * np.sqrt(len(h)) * np.abs(h).sum())
    assert np.all(steady.imag == 0)
    assert abs(g - 1.0) < 2e-3


def response(h, f):
    """float64 frequency response at f cycles per input sample"""
    i = np.arange(len(h))
    return np.exp(-2j * np.pi * np.outer(f, i)) @ h.astype(np.float64)


@pytest.mark.parametrize("D", [2, 3, 7, 8, 16, 64])
def test_passband_tone_has_the_response_gain(D):
    h = spec_taps(D)
    m = 200 * D
    n = np.arange(m)
    for f in (0.4 / D, -0.31 / D, 0.05 / D):
        x = np.exp(2j * np.pi * f * n).astype(np.complex64)
        y = decim_oracle.Decimator(D).feed(x)[20:]
        k = np.arange(20, 20 + len(y))
        ref = response(h, [f])[0] * np.exp(2j * np.pi * f * k * D)
        assert np.max(np.abs(y - ref)) < 2e-5
        assert abs(abs(response(h, [f])[0]) - 1.0) < 0.005        # 0.44 % at 0.4 fs/D


def stopband_db(D):
    h = spec_taps(D)
    f = np.linspace(0.65 / D, 0.5, 4000)
    H = np.abs(np.concatenate([response(h, f), response(h, -f)]))
    return -20 * np.log10(H.max())


@pytest.mark.parametrize("D", [d for d in DS if d > 1])
def test_stopband_attenuation(D):
    assert stopband_db(D) >= STOP_DB
    m = 200 * D
    n = np.arange(m)
    for f in (0.65 / D, -0.7 / D, 0.5, -0.37):
        if abs(f) < 0.65 / D:
            continue
        x = np.exp(2j * np.pi * f * n).astype(np.complex64)
        y = decim_oracle.Decimator(D).feed(x)[20:]
        assert 20 * np.log10(np.abs(y).max()) <= -STOP_DB


# ---- feed split ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("D", [1, 2, 3, 7, 8, 16, 64, 256])
def test_ragged_feeds_bit_identical(D, fmt):
    m = 30 * D + 11
    x = make_input(fmt, m, seed=300 + D)
    one = decim_oracle.Decimator(D, fmt).feed(x)
    rng = np.random.default_rng(D)
    splits = sorted({1, max(1, D - 1), D + 1} | set(int(v) for v in rng.integers(1, m, 6)))
    dec = decim_oracle.Decimator(D, fmt)
    parts, a = [], 0
    for b in splits + [m]:
        if b > a:
            parts.append(dec.feed(feed_rows(x, fmt, a, b)))
            a = b
    many = np.concatenate(parts)
    assert np.array_equal(one.view(np.uint32), many.view(np.uint32))
    dec.reset()
    assert np.array_equal(dec.feed(x).view(np.uint32), one.view(np.uint32))


def test_decimation_out_of_range_rejected():
    with pytest.raises(ValueError):
        decim_oracle.Decimator(0)
    with pytest.raises(ValueError):
        decim_oracle.Decimator(257)
