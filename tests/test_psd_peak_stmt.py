"""The statement of SPEC PK (tests/psd_peak_stmt.py) held to known answers, without a GPU."""
import numpy as np
import pytest

from psd_peak_stmt import MISTAKES, group_peaks, same


def _noise(S, F, N, seed):
    """positive per-frame spectra like the main PSD's: |X|^2 / N of complex noise"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((S, F, N, 2)).astype(np.float32)
    return ((x[..., 0] * x[..., 0] + x[..., 1] * x[..., 1]) / np.float32(N)).astype(np.float32)


def _feeds(psd, P, split, mistake=None):
    """group_peaks over the frames of psd split into feeds of `split` frames, the carry passed on"""
    carry, mx, mn, pos = None, [], [], 0
    for f in split:
        a, b, carry = group_peaks(psd[:, pos:pos + f], P, carry, mistake)
        mx.append(a); mn.append(b)
        pos += f
    return np.concatenate(mx, axis=1), np.concatenate(mn, axis=1), carry


@pytest.mark.parametrize("P", [2, 3, 7])
def test_tone_in_one_frame(P):
    """A tone present in one frame of each group is in every max at that frame's level and absent from every min."""
    S, N, G = 2, 64, 5
    floor = np.full((S, G * P, N), 1e-4, np.float32)
    psd = floor.copy()
    for g in range(G):
        f = g * P + (g % P)                                         # a different frame of each group
        psd[:, f, 10 + g] = np.float32(3.5 + g)
    mx, mn, carry = group_peaks(psd, P)
    assert mx.shape == mn.shape == (S, G, N) and carry.count == 0
    for g in range(G):
        want = np.full((S, N), 1e-4, np.float32)
        want[:, 10 + g] = np.float32(3.5 + g)
        assert same(mx[:, g], want)
        assert same(mn[:, g], floor[:, 0])


def test_constant_spectrum():
    """max = min = the spectrum when every frame is the same."""
    S, N, P = 3, 32, 4
    one = _noise(S, 1, N, 1)
    psd = np.repeat(one, 3 * P, axis=1)
    mx, mn, _ = group_peaks(psd, P)
    for g in range(3):
        assert same(mx[:, g], one[:, 0]) and same(mn[:, g], one[:, 0])


def test_extremes_are_input_values():
    """Every output is one of the group's inputs, and equals numpy's reduction of the group."""
    S, N, P = 2, 128, 5
    psd = _noise(S, 4 * P, N, 2)
    mx, mn, _ = group_peaks(psd, P)
    g = psd.reshape(S, 4, P, N)
    assert same(mx, g.max(axis=2)) and same(mn, g.min(axis=2))


def test_nan_rules():
    """NaN operands are ignored, also in the group's first frame; a bin NaN in every frame of its group gives NaN."""
    S, N, P = 1, 8, 3
    psd = _noise(S, 3 * P, N, 3)
    nan = np.float32(np.nan)
    psd[:, 0, :] = nan                                              # group 0: its first frame is NaN
    psd[:, 4, 2] = nan                                              # group 1: one bin NaN in its middle frame
    psd[:, 6:9, 5] = nan                                            # group 2: bin 5 NaN in every frame
    psd[:, 8, 1] = np.float32(np.inf)                               # group 2: +inf wins the max
    mx, mn, _ = group_peaks(psd, P)
    assert same(mx[:, 0], np.fmax(psd[:, 1], psd[:, 2])) and same(mn[:, 0], np.fmin(psd[:, 1], psd[:, 2]))
    assert not np.isnan(mx[:, :2]).any() and not np.isnan(mn[:, :2]).any()
    assert mx[0, 1, 2] == max(psd[0, 3, 2], psd[0, 5, 2]) and mn[0, 1, 2] == min(psd[0, 3, 2], psd[0, 5, 2])
    assert np.isnan(mx[0, 2, 5]) and np.isnan(mn[0, 2, 5])
    assert np.isinf(mx[0, 2, 1]) and mn[0, 2, 1] == min(psd[0, 6, 1], psd[0, 7, 1])
    assert np.isnan(mx[0, 2]).sum() == 1 and np.isnan(mn[0, 2]).sum() == 1


@pytest.mark.parametrize("split", [[24], [1] * 24, [3, 7, 1, 9, 4], [5, 5, 5, 9], [10, 14]])
def test_any_split_gives_the_same_groups(split):
    """PK.3: the partial group carries, so any split of the frames into feeds gives the groups of one feed."""
    S, N, P = 2, 64, 5
    psd = _noise(S, 24, N, 4)
    want_mx, want_mn, want_c = group_peaks(psd, P)
    mx, mn, carry = _feeds(psd, P, split)
    assert mx.shape == (S, 24 // P, N)
    assert same(mx, want_mx) and same(mn, want_mn)
    assert carry.count == want_c.count == 24 % P
    assert same(carry.mx, want_c.mx) and same(carry.mn, want_c.mn)


def test_feed_emits_floor_of_carried_plus_frames():
    S, N, P = 1, 16, 4
    psd = _noise(S, 11, N, 5)
    carry, counts = None, []
    for f0, f1 in ((0, 3), (3, 4), (4, 11)):
        mx, _, carry = group_peaks(psd[:, f0:f1], P, carry)
        counts.append(mx.shape[1])
    assert counts == [0, 1, 1] and carry.count == 3


@pytest.mark.parametrize("mistake", MISTAKES)
def test_statement_rejects_planted_mistakes(mistake):
    """Each planted mistake changes the outputs of the known-answer scenes above."""
    S, N, P = 1, 32, 4
    psd = _noise(S, 4 * P, N, 6)
    psd[:, 0, 3] = np.float32(np.nan)                               # only "max" sees this
    psd[:, P, 7] = np.float32(50.0)                                 # first frame of group 1: only "off_by_one" moves it
    mx, mn, _ = group_peaks(psd, P)
    bad_mx, bad_mn, _ = group_peaks(psd, P, mistake=mistake)
    assert not (same(mx, bad_mx) and same(mn, bad_mn))
