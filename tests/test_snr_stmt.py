"""The oracle's SNR meter (oracle/snr.c) against the binary32 statement of SPEC SN (tests/snr_stmt.py), bit for bit,
and its behaviour on synthetic QPSK.  Each planted mistake of the statement is caught by a named case."""
import numpy as np
import pytest

import snr_oracle as O
import snr_stmt as S

F = np.float32


def edge_symbols():
    """v = +-pi, -0, NaN, and moduli at, just under and above 1, plus random symbols"""
    one_minus = np.nextafter(F(1.0), F(0.0))
    one_plus = np.nextafter(F(1.0), F(2.0))
    pts = [complex(-1.0, 0.0), complex(-1.0, -0.0), complex(-0.0, 0.0), complex(0.0, -0.0), complex(-0.0, -0.0),
           complex(1.0, 0.0), complex(0.0, 1.0), complex(0.0, -1.0), complex(np.nan, 0.0), complex(0.0, np.nan),
           complex(one_minus, 0.0), complex(0.0, one_minus), complex(1.0, 0.0), complex(one_plus, 0.0),
           complex(0.0, 2.0), complex(-0.6, 0.8), complex(np.inf, 1.0), complex(-3.0, -1e-30)]
    rng = np.random.default_rng(1)
    r = (rng.standard_normal(4000) + 1j * rng.standard_normal(4000)) * 0.6
    return np.concatenate([np.array(pts, np.complex64), r.astype(np.complex64)])


def status_key(m):
    b = lambda x: int(np.float32(x).view(np.uint32))      # noqa: E731
    return (m.counted, m.steps, m.stepped, b(m.sigma), b(m.snr), b(m.delta))


def assert_same(o, s, where):
    assert np.array_equal(o.h, s.h.astype(np.uint32)), "h differs at %s" % (where,)
    assert np.array_equal(o.model.view(np.uint32), s.model.view(np.uint32)), "model differs at %s" % (where,)
    assert o.status.key() == status_key(s), "status differs at %s: %s vs %s" % (where, o.status.key(), status_key(s))


@pytest.mark.parametrize("L", [16, 100, 256, 1024])
@pytest.mark.parametrize("mode", [0, 1])
def test_bins_match_statement(mode, L):
    x = edge_symbols()
    want = S.bins(x, mode, L)
    got = np.array([O.bin_of(mode, L, v) for v in x])
    assert np.array_equal(got, want)
    if mode == 0:
        assert got[0] == L - 1 and got[1] == L - 1        # v = pi lands in the last bin (M.2 gives pi for y = -0)
        assert got[17] == 0                                # v = -pi in the first
        assert got[8] == -1                                # a NaN v is never counted (M.2 gives pi/2 for x = 0, y = NaN)
    else:
        assert got[10] == L - 1 and got[12] == -1 and got[13] == -1 and got[14] == -1
        assert got[8] == -1 and got[9] == -1


def test_ask_at_or_above_one_is_dropped():
    x = edge_symbols()
    for L in (16, 256):
        got = np.array([O.bin_of(1, L, v) for v in x])
        assert not np.array_equal(got, S.bins(x, 1, L, mistake="ask_clamp"))


def test_bin_expression_matches_spec_d():
    """Arguments within a few ulps of the bin edges, where (v - min) / (max - min) L and (v - min) L / (max - min)
    round to different sides"""
    caught = False
    for L in (100, 256, 1000):
        edges = -np.pi + 2 * np.pi * np.arange(L) / L
        th = (edges[:, None] + np.linspace(-4e-7, 4e-7, 41)[None, :]).ravel()
        x = np.exp(1j * th).astype(np.complex64)
        want = S.bins(x, 0, L)
        differ = np.flatnonzero(want != S.bins(x, 0, L, mistake="bin_scaled"))
        pick = np.concatenate([differ[:200], np.arange(0, len(x), 97)])
        got = np.array([O.bin_of(0, L, v) for v in x[pick]])
        assert np.array_equal(got, want[pick])
        caught |= len(differ) > 0
    assert caught


def feeds(rng, cls, bps, n_feeds=12):
    """soft symbols of a noisy constellation, with zero-symbol feeds in the middle of the run"""
    K = 1 << max(bps, 1)
    out = []
    for f in range(n_feeds):
        n = 0 if f in (3, 4, 8) else int(rng.integers(1, 900))
        k = rng.integers(0, K, n)
        if cls == "ask":
            a = (k + 0.5) / K * 1.1
            x = a * np.exp(1j * rng.uniform(-0.1, 0.1, n)) + 0.05 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
        else:
            x = np.exp(1j * (2 * np.pi * (k + 0.5) / K)) * 0.8 + 0.15 * (rng.standard_normal(n) +
                                                                        1j * rng.standard_normal(n))
        out.append(x.astype(np.complex64))
    return out


@pytest.mark.parametrize("bps", [1, 2, 3])
@pytest.mark.parametrize("L", [16, 100, 256, 1024])
@pytest.mark.parametrize("cls", ["psk", "fsk", "ask"])
def test_runs_match_statement(cls, L, bps):
    rng = np.random.default_rng(100 * L + 10 * bps + len(cls))
    K = 1 << bps
    o, s = O.Meter(cls, L, bps, 1.0, 1.0 / K), S.Meter(cls, L, bps, 1.0, 1.0 / K)
    for f, x in enumerate(feeds(rng, cls, bps)):
        o.feed(x)
        s.feed(x)
        assert_same(o, s, (cls, L, bps, f))


def test_bps_zero_is_read_as_one():
    rng = np.random.default_rng(3)
    o, s = O.Meter("psk", 64, 0, 1.0, 0.5), S.Meter("psk", 64, 0, 1.0, 0.5)
    assert o.m.K == s.K == 2
    for x in feeds(rng, "psk", 1, 4):
        o.feed(x)
        s.feed(x)
        assert_same(o, s, "bps 0")


def test_zero_symbol_feed_does_not_step():
    rng = np.random.default_rng(5)
    xs = feeds(rng, "psk", 2, 6)
    o, s, bad = O.Meter("psk", 256, 2, 1.0, 0.25), S.Meter("psk", 256, 2, 1.0, 0.25), \
        S.Meter("psk", 256, 2, 1.0, 0.25, mistake="step_on_empty")
    diverged = False
    for f, x in enumerate(xs):
        before = o.status.key()
        o.feed(x)
        s.feed(x)
        bad.feed(x)
        assert_same(o, s, f)
        if len(x) == 0:
            assert o.status.stepped == 0 and o.status.key()[:2] == before[:2] and o.status.key()[3:] == before[3:]
        diverged |= status_key(bad) != o.status.key()
    assert diverged


@pytest.mark.parametrize("cls", ["psk", "ask"])
def test_halving_at_two_to_the_31(cls):
    L = 64
    rng = np.random.default_rng(9)
    h0 = rng.integers(0, 1 << 30, L).astype(np.int64)
    x = feeds(rng, cls, 2, 1)[0]
    b = S.bins(x, 1 if cls == "ask" else 0, L)
    top = int(np.bincount(b[b >= 0], minlength=L).argmax())
    h0[top] = (1 << 31) - 1                     # the feed's busiest bin crosses 2^31
    o, s = O.Meter(cls, L, 2, 1.0, 0.25), S.Meter(cls, L, 2, 1.0, 0.25)
    o.seed(h0)
    s.h = h0.copy()
    o.feed(x)
    s.feed(x)
    assert_same(o, s, "halving")
    assert o.h.max() < (1 << 31) and o.h[top] == ((1 << 31) - 1 + np.sum(b == top)) >> 1
    o.feed(x)
    s.feed(x)
    assert_same(o, s, "after halving")


def test_replan_and_reset():
    """SN.3 reset and every SN.4 branch, each with feeds after it"""
    rng = np.random.default_rng(11)
    xs = feeds(rng, "fsk", 2, 16)
    o, s = O.Meter("fsk", 128, 2, 1.0, 0.25), S.Meter("fsk", 128, 2, 1.0, 0.25)
    bad = S.Meter("fsk", 128, 2, 1.0, 0.25, mistake="keep_h_on_change")
    steps = [("feed",)] * 3 + [("reset", 0.5)] + [("feed",)] * 2 + [("replan", True, 2, 0.3)] + [("feed",)] * 2 + \
        [("replan", False, 2, 0.3)] + [("feed",)] * 2 + [("replan", False, 3, 0.125)] + [("feed",)] * 3
    it = iter(xs)
    caught = False
    for i, st in enumerate(steps):
        for m in (o, s, bad):
            if st[0] == "feed":
                pass
            elif st[0] == "reset":
                m.reset(st[1])
            else:
                m.replan(*st[1:])
        if st[0] == "feed":
            x = next(it)
            o.feed(x)
            s.feed(x)
            bad.feed(x)
        elif st[0] == "reset":
            assert o.h.sum() > 0 and o.status.sigma == np.float32(0.5)          # h kept, sigma set
        elif st[0] == "replan" and st[1]:
            assert o.h.sum() > 0                                                # everything kept
        elif st[0] == "replan":
            assert o.h.sum() == 0 and o.status.steps == 0                       # h cleared
            assert o.status.sigma == (np.float32(0.125) if st[2] == 3 else s.sigma)
        assert_same(o, s, (i, st))
        caught |= not np.array_equal(bad.h, s.h)
    assert caught


def qpsk_sigmas(esn0_db, steps, seed):
    rng = np.random.default_rng(seed)
    m = O.Meter("psk", 256, 2, 1.0, 0.25)
    n0 = 10 ** (-esn0_db / 10)
    out = []
    for _ in range(steps):
        sym = np.exp(1j * (np.pi / 4 + np.pi / 2 * rng.integers(0, 4, 1300)))
        x = sym + np.sqrt(n0 / 2) * (rng.standard_normal(1300) + 1j * rng.standard_normal(1300))
        m.feed(x.astype(np.complex64))
        out.append(m.status.snr)
    return np.array(out)


def test_snr_increases_with_esn0_on_qpsk():
    """The fit converges slowly, so only the ordering is asserted: at every step from 10 to 300 the estimate grows
    strictly with Es/N0."""
    snr = np.array([qpsk_sigmas(e, 300, 20 + e) for e in (5, 10, 15, 20, 25)])
    assert np.all(np.diff(snr[:, 9:], axis=0) > 0)
