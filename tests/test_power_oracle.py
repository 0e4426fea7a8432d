"""The power-inspector oracle (oracle/power.c, SPEC PW) against a literal transcription of the RMS tab's raw-mode
integration (Default/RMSInspector/RMSInspector.cpp:538-560, 327-338): bit-identical means for every M, however the
input is split into feeds, and on an input where the Kahan compensation changes the result."""
import numpy as np
import pytest

import power_oracle as P


def noise(n, seed, scale=1.0):
    rng = np.random.default_rng(seed)
    return (scale * (rng.standard_normal(n) + 1j * rng.standard_normal(n))).astype(np.complex64)


def run_oracle(x, M, splits):
    pw, out, pos = P.Power(M), [], 0
    for m in splits:
        out.append(pw.feed(x[pos:pos + m]))
        pos += m
    assert pos == len(x)
    return np.concatenate(out)


def run_gui(x, M, splits):
    st, out, pos = [0.0, 0.0, 0], [], 0
    for m in splits:
        out.append(P.gui_raw_mode(x[pos:pos + m], M, st))
        pos += m
    return np.concatenate(out)


def ragged(n, seed):
    """feed sizes 1 .. 5000, some shorter than any M tested below"""
    rng = np.random.default_rng(seed)
    out = []
    while sum(out) < n:
        out.append(int(rng.integers(1, 5000)))
    out[-1] -= sum(out) - n
    return [m for m in out if m > 0]


@pytest.mark.parametrize("M", [0, 1, 2, 7, 4096, 10**6])
def test_oracle_matches_gui_raw_mode(M):
    n = 2_500_000 if M == 10**6 else 60_000
    # a level that drifts over four decades, so that the sums grow well past the size of one sample
    x = noise(n, 5 + M % 97) * np.exp(np.linspace(0, 4.6, n)).astype(np.float32)
    ref = run_gui(x, M, [n])
    assert len(ref) == n // max(M, 1)
    for splits in ([n], ragged(n, M % 13), [1] * 10 + [n - 10]):
        got = run_oracle(x, M, splits)
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), splits[:4]


def test_group_split_inside_feeds():
    """M = 7 over feeds of 3, 5 and 11 samples: groups straddle every feed boundary"""
    x = noise(7 * 300, 2)
    splits = [3, 5, 11] * 110
    splits[-1] += len(x) - sum(splits)
    assert np.array_equal(run_oracle(x, 7, splits).view(np.uint32), run_gui(x, 7, [len(x)]).view(np.uint32))


def kahan_case(groups):
    """Per group of M = 4 the powers 1, 2^-24, 2^-53, 2^-53.  A binary64 sum drops each 2^-53 (ties to even) and
    stops at 1 + 2^-24, whose quarter is a binary32 tie that rounds down to 1/4; the compensated sum reaches
    1 + 2^-24 + 2^-52, whose quarter rounds up to (1 + 2^-23) / 4."""
    g = np.array([1.0, 2.0 ** -12, 2.0 ** -27 * (1 + 1j), 2.0 ** -27 * (1 + 1j)], np.complex64)
    return np.tile(g, groups)


def plain_sum(x, M):
    re, im = x.real.astype(np.float32), x.imag.astype(np.float32)
    acc, n, out = 0.0, 0, []
    for p in (re * re + im * im).astype(np.float32).tolist():
        acc += p
        n += 1
        if n >= M:
            out.append(acc / n)
            acc, n = 0.0, 0
    return np.array(out, np.float32)


def test_kahan_compensation_changes_the_mean():
    x = kahan_case(3)
    ref = run_gui(x, 4, [len(x)])
    assert np.all(ref == np.float32((1 + 2.0 ** -23) / 4))
    assert not np.array_equal(plain_sum(x, 4), ref)          # an uncompensated statement fails this input
    assert np.array_equal(plain_sum(x, 4), np.full(3, 0.25, np.float32))
    for splits in ([len(x)], [1] * len(x), [3, 2, 7]):
        assert np.array_equal(run_oracle(x, 4, splits).view(np.uint32), ref.view(np.uint32))
