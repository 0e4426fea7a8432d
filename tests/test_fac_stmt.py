"""The CPU oracle of the FAC tab (oracle/fac.c) against the statement of oracle/SPEC_FC.md: FC.1 in binary64 with a
bound at every block size, FC.2 - FC.4 bit for bit in binary32 (tests/fac_stmt.py), the planted mistakes each caught by
a named case, and the oracle's v / L against the tab's own arithmetic (tests/golden/ref_fac.npz)."""
import os

import numpy as np
import pytest

import fac_f64
import fac_oracle
from fac_stmt import FacStmt, key

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SIZES = [1 << m for m in range(9, 20)]


def _symbols(n, seed, period=None):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)) * 0.1
    if period:
        base = rng.choice([-1.0, 1.0], period) + 0j
        x = x + np.resize(base, n)
    return x.astype(np.complex64)


def _blocks_v(o, x):
    L = o.L
    return [o.magnitude(x[i:i + L]) for i in range(0, len(x) - L + 1, L)]


@pytest.mark.parametrize("L", SIZES)
def test_fc1_within_float64_bound(L):
    o = fac_oracle.Fac(L)
    x = _symbols(L, L, period=37)
    v = o.magnitude(x).astype(np.float64)
    ref = fac_f64.v64(x)
    b = fac_f64.bound(x)
    assert np.abs(v - ref).max() <= b
    # decisions: the arg-max past lag 0 and the record set, wherever their margins exceed the bound
    lo, hi = 1, L // 2
    pos, margin = fac_f64.decisions(ref, lo, hi, b)
    if margin > 2 * b:
        assert fac_f64.decisions(v, lo, hi, b)[0] == pos
    rec64, m = fac_f64.records(ref, lo, hi)
    rec32, _ = fac_f64.records(v, lo, hi)
    sure = m > 2 * b
    assert np.array_equal(rec64[sure], rec32[sure])


@pytest.mark.parametrize("L", [512, 1024, 2048, 4096])
def test_fc1_inverse_equals_forward_twice(L):
    o = fac_oracle.Fac(L)
    x = _symbols(L, 7 + L, period=19)
    a, b = o.magnitude(x), o.magnitude(x, twice=True)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_oracle_against_the_tab():
    f = np.load(os.path.join(GOLD, "ref_fac.npz"))
    o = fac_oracle.Fac(1024)
    v = o.magnitude(f["x"][-1024:]).astype(np.float64) / 1024
    assert np.abs(v - f["fac"]).max() <= 2e-6 * f["fac"].max()


def _run_both(L, feeds, alpha=1.0, lags=None, sigma=5.0):
    """feed the oracle symbol by symbol and the statement with the oracle's own v of each completed block"""
    o = fac_oracle.Fac(L, alpha, lags, sigma)
    s = FacStmt(L, alpha, lags, sigma)
    v_of = fac_oracle.Fac(L)              # a second oracle, only for FC.1 of the blocks
    buf = np.zeros(0, np.complex64)
    out = []
    for x in feeds:
        st = o.feed(x)
        buf = np.concatenate([buf, x])
        nb = len(buf) // L
        vs = [v_of.magnitude(buf[i * L:(i + 1) * L]) for i in range(nb)]
        buf = buf[nb * L:]
        ss = s.feed_v(vs)
        assert st.key() == key(ss), (st.key(), key(ss))
        assert np.array_equal(o.fac.view(np.uint32), s.fac.view(np.uint32))
        assert o.p == len(buf)
        out.append(st)
    return out


@pytest.mark.parametrize("alpha", [1.0, 0.5, 0.0])
@pytest.mark.parametrize("lags", [None, (0, 200), (3, 256)])
def test_straddling_and_multi_block_feeds(alpha, lags):
    L = 512
    x = _symbols(6000, 5, period=23)
    cuts = [0, 100, 100, 700, 700, 2900, 3000, 6000]     # zero-symbol feeds, a block across feeds, 4 blocks in one
    feeds = [x[a:b] for a, b in zip(cuts[:-1], cuts[1:])]
    sts = _run_both(L, feeds, alpha, lags, sigma=2.0)
    assert [s.blocks for s in sts] == [0, 0, 1, 0, 4, 0, 6]
    if lags and lags[0] > 0:
        assert any(s.marker for s in sts)


def test_multi_tile_window():
    _run_both(8192, [_symbols(3 * 8192 + 5, 9, period=101)], alpha=0.5, lags=(1, 3000), sigma=3.0)


def test_lag_zero_window_peaks_at_zero():
    st = _run_both(1024, [_symbols(2048, 3, period=31)])[0]
    assert st.peak_lag == 0


def test_all_zero_input_is_nan():
    o = fac_oracle.Fac(512)
    st = o.feed(np.zeros(512, np.complex64))
    assert st.max == 0 and np.all(np.isnan(o.fac))
    s = FacStmt(512)
    ss = s.feed_v([np.zeros(256, np.float32)])
    assert st.key() == key(ss)


# ---- planted mistakes: each one is caught by a named case of the statement against the oracle

def _feed_with(mistake, L=512, lags=(2, 256)):
    x = _symbols(3 * L, 11, period=29)
    v_of = fac_oracle.Fac(L)
    vs = [v_of.magnitude(x[i * L:(i + 1) * L]) for i in range(3)]
    o = fac_oracle.Fac(L, 0.5, lags, 1.0)
    st = o.update_feed(vs)
    s = FacStmt(L, 0.5, lags, 1.0)
    ss = s.feed_v(vs, **{mistake: True})
    return st.key() == key(ss) and np.array_equal(o.fac.view(np.uint32), s.fac.view(np.uint32))


def test_planted_records_in_power_is_caught():
    assert not _feed_with("record_in_power")


def test_planted_local_max_per_block_is_caught():
    assert not _feed_with("reset_local_per_block")


def test_planted_max_before_block_is_caught():
    assert not _feed_with("max_before")


def test_planted_max_outside_window_is_caught():
    assert not _feed_with("max_outside", lags=(40, 256))


def test_statement_without_mistakes_agrees():
    x = _symbols(3 * 512, 11, period=29)
    v_of = fac_oracle.Fac(512)
    vs = [v_of.magnitude(x[i * 512:(i + 1) * 512]) for i in range(3)]
    o = fac_oracle.Fac(512, 0.5, (2, 256), 1.0)
    s = FacStmt(512, 0.5, (2, 256), 1.0)
    assert o.update_feed(vs).key() == key(s.feed_v(vs))
