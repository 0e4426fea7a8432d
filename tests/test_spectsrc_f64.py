"""The CPU oracle's inspector spectrum sources and baud estimators (oracle/spectsrc.c) against the float64 statement
of SPEC U and W (tests/spectsrc_f64.py).

The CUDA kernel is held bit for bit to the oracle; these tests hold the oracle to the SPEC at every Ns = 64 ... 4096
and every kind: spectra within a stated bound of the statement (the worst ratio is reported), estimators equal to
the statement wherever its margin clears the bound, the U.1 boundary, all-zero input, a pure tone, and statements
with one deliberate mistake that a named case must reject."""

import numpy as np
import pytest

import spectsrc_f64 as sf

FS = 1000.0
SPS = (4, 5, 8, 16)

# deliberate mistake -> named case that must catch it: (what, kind or estimator, signal, Ns)
MISTAKE_CASES = {
    "window_n": ("spectrum", "psd", "qpsk_sps8_off", 64),
    "cyclo_conj": ("spectrum", "cyclo", "qpsk_sps8_off", 256),
    "fm_no_pi": ("spectrum", "fmspect", "fsk_sps8", 256),
    "fac_mean": ("estimator", "baud-fac", "qpsk_sps4", 256),
    "kmin0": ("estimator", "baud-nonlinear", "qpsk_sps8", 256),
}


def qpsk(n, sps, f_off=0.0, seed=0):
    """rectangular-pulse QPSK with whole samples per symbol, optionally offset by f_off cycles per sample"""
    rng = np.random.default_rng(seed)
    sym = np.exp(1j * (np.pi / 4 + np.pi / 2 * rng.integers(0, 4, n // sps + 1)))
    x = 0.7 * np.repeat(sym, sps)[:n] * np.exp(2j * np.pi * f_off * np.arange(n))
    return x.astype(np.complex64)


def fsk(n, sps, seed=0):
    """phase-continuous 2-FSK with tones at 0.02 and 0.12 cycles per sample (|x[n] - x[n-1]| differs per tone)"""
    rng = np.random.default_rng(seed)
    f = np.repeat(np.where(rng.integers(0, 2, n // sps + 1) > 0, 0.12, 0.02), sps)[:n]
    return (0.6 * np.exp(2j * np.pi * np.cumsum(f))).astype(np.complex64)


def signal(name, ns):
    n = 2 * ns + 37
    if name == "zeros":
        return np.zeros(n, np.complex64)
    if name == "tone":                           # exp(i pi n / 2) / 2: exact in binary32, |delta| constant
        return (0.5 * 1j ** np.arange(n)).astype(np.complex64)
    kind, sps = name.split("_sps")
    off = sps.endswith("_off")
    sps = int(sps.replace("_off", ""))
    if kind == "qpsk":
        return qpsk(n, sps, 0.013 if off else 0.0, seed=ns + sps)
    return fsk(n, sps, seed=ns + sps)


SIGNALS = ["qpsk_sps%d" % s for s in SPS] + ["qpsk_sps8_off"] + ["fsk_sps%d" % s for s in SPS]


def spectrum_ratio(oracle, kind, ns, chan):
    got = oracle.spectsrc_frame(kind, ns, chan).astype(np.float64)
    ref = sf.spectrum(kind, ns, chan)
    return float(np.max(np.abs(got - ref) / sf.spectrum_bound(kind, ns, chan)))


def estimator_agrees(oracle, est, ns, chan, mistake=None):
    """-> (agrees, margin / bound): the oracle's value and validity equal the statement's, or the margin is too small
    to require it"""
    fn = sf.baud_fac if est == "baud-fac" else sf.baud_nonlinear
    val, margin = fn(ns, FS, chan, mistake)
    if est == "baud-fac":
        bound = sf.acf_bound(ns, chan)
    else:
        b = sf.spectrum_bound("abstimediff", ns, chan)
        bound = float(np.max(b[sf.KMIN:ns // 2]))
    got = oracle.estimate_baud(est, ns, np.float32(FS), chan)
    if margin <= 2 * bound:
        return True, margin / bound
    same = (got is None) == (val is None) and (val is None or np.float32(got) == np.float32(val))
    return same, margin / bound


# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ns", sf.SIZES)
@pytest.mark.parametrize("kind", sf.KINDS)
def test_oracle_spectrum_within_bound(oracle, kind, ns):
    """Every kind at every Ns on QPSK (with and without a carrier offset) and 2-FSK: every bin within the bound."""
    for name in SIGNALS:
        chan = signal(name, ns)
        r = spectrum_ratio(oracle, kind, ns, chan)
        assert r <= 1.0, "%s Ns %d %s: worst bin at %.3g x the bound" % (kind, ns, name, r)


@pytest.mark.parametrize("ns", sf.SIZES)
def test_oracle_estimators_equal_statement(oracle, ns):
    """Both estimators equal the statement (value and validity) wherever the margin clears twice the bound, and
    baud-fac gives the exact symbol rate at whole samples per symbol."""
    for name in SIGNALS:
        chan = signal(name, ns)
        for est in ("baud-fac", "baud-nonlinear"):
            ok, m = estimator_agrees(oracle, est, ns, chan)
            assert ok, (est, ns, name, m)
        sps = int(name.split("_sps")[1].replace("_off", ""))
        val, margin = sf.baud_fac(ns, FS, chan)
        if name.startswith("qpsk") and ns >= 16 * sps and margin > 2 * sf.acf_bound(ns, chan):
            assert val == FS / sps, (name, ns, val)


def test_estimators_resolve_the_symbol_rate(oracle):
    """Known answers where the margins are wide, on QPSK: baud-fac exact; baud-nonlinear on a line of the symbol rate
    (the |x[n] - x[n-1]| of rectangular pulses is a pulse train: every harmonic is a line, the strongest wins)."""
    for ns in (256, 1024, 4096):
        for sps in (4, 8, 16):
            chan = signal("qpsk_sps%d" % sps, ns)
            val, margin = sf.baud_fac(ns, FS, chan)
            assert val == FS / sps and margin > 2 * sf.acf_bound(ns, chan), (ns, sps)
            assert oracle.estimate_baud("baud-fac", ns, FS, chan) == np.float32(FS / sps)
            val, _ = sf.baud_nonlinear(ns, FS, chan)
            m = round(val * sps / FS)
            assert m >= 1 and abs(val - m * FS / sps) <= FS / ns, (ns, sps, val)


@pytest.mark.parametrize("ns", sf.SIZES)
def test_all_zero_input(oracle, ns):
    """All zeros: every spectrum is exactly 0 (fmspect: atan2(0, 0) = 0) and both estimators are invalid."""
    chan = signal("zeros", ns)
    for kind in sf.KINDS:
        got = oracle.spectsrc_frame(kind, ns, chan)
        assert got is not None and not np.any(got) and not np.any(sf.spectrum(kind, ns, chan)), kind
    for est, fn in (("baud-fac", sf.baud_fac), ("baud-nonlinear", sf.baud_nonlinear)):
        assert oracle.estimate_baud(est, ns, FS, chan) is None and fn(ns, FS, chan)[0] is None, est


@pytest.mark.parametrize("ns", sf.SIZES)
def test_pure_tone_has_no_baud(oracle, ns):
    """A tone has a constant |x[n] - x[n-1]|: the mean-removed autocorrelation is ~0 in the statement (within the
    bound) and exactly 0 in binary32, so baud-fac is invalid."""
    chan = signal("tone", ns)
    assert np.max(np.abs(sf.baud_fac_acf(ns, chan))) <= sf.acf_bound(ns, chan)
    assert oracle.estimate_baud("baud-fac", ns, FS, chan) is None


@pytest.mark.parametrize("ns", [64, 1024, 4096])
def test_u1_boundary(oracle, ns):
    """Ns + 1 channel samples emit (x[-1] is the first of them), Ns samples emit nothing."""
    chan = signal("qpsk_sps5", ns)
    for kind in sf.KINDS:
        assert oracle.spectsrc_frame(kind, ns, chan[:ns]) is None and sf.spectrum(kind, ns, chan[:ns]) is None
        assert spectrum_ratio(oracle, kind, ns, chan[:ns + 1]) <= 1.0, kind
    for est in ("baud-fac", "baud-nonlinear"):
        assert oracle.estimate_baud(est, ns, FS, chan[:ns]) is None
        assert estimator_agrees(oracle, est, ns, chan[:ns + 1])[0]
    # x[-1] matters: the timediff spectrum changes with the sample before the frame
    other = chan[:ns + 1].copy()
    other[0] = -other[0]
    assert not np.array_equal(oracle.spectsrc_frame("timediff", ns, other),
                              oracle.spectsrc_frame("timediff", ns, chan[:ns + 1]))
    assert spectrum_ratio(oracle, "timediff", ns, other) <= 1.0


@pytest.mark.parametrize("mistake", sf.MISTAKES)
def test_statement_mistakes_are_caught(oracle, mistake):
    """Each planted mistake makes its named case disagree with the oracle beyond the bound."""
    what, kind, name, ns = MISTAKE_CASES[mistake]
    chan = signal(name, ns)
    if what == "spectrum":
        assert spectrum_ratio(oracle, kind, ns, chan) <= 1.0
        got = oracle.spectsrc_frame(kind, ns, chan).astype(np.float64)
        bad = sf.spectrum(kind, ns, chan, mistake)
        assert np.max(np.abs(got - bad) / sf.spectrum_bound(kind, ns, chan)) > 1.0, mistake
    else:
        fn = sf.baud_fac if kind == "baud-fac" else sf.baud_nonlinear
        assert estimator_agrees(oracle, kind, ns, chan)[0]
        good, bad = fn(ns, FS, chan)[0], fn(ns, FS, chan, mistake)[0]
        got = oracle.estimate_baud(kind, ns, FS, chan)
        assert good is not None and got == np.float32(good) and got != (None if bad is None else np.float32(bad))


def test_worst_ratio_report(oracle, capsys):
    """The worst spectrum-to-bound ratio over every kind, Ns and signal (printed; must be <= 1)."""
    worst = (0.0, None)
    for ns in sf.SIZES:
        for name in SIGNALS:
            chan = signal(name, ns)
            for kind in sf.KINDS:
                r = spectrum_ratio(oracle, kind, ns, chan)
                worst = max(worst, (r, (kind, ns, name)), key=lambda t: t[0])
    with capsys.disabled():
        print("\nSPEC U spectra: worst oracle-to-statement error %.3g x the bound at %s" % worst)
    assert worst[0] <= 1.0
