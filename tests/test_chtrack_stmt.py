"""The CPU oracle's channel tracker (sdo_chtrack_update, oracle/chtrack.c) against the exact statement of SPEC KT
(tests/chtrack_stmt.py).

The CUDA tracker is held bit for bit to the oracle (tests/test_gpu_chtrack.py); these tests hold the oracle to the
SPEC over sequences of detector lists at the edges of KT (carriers that vanish within and beyond the hold, splits,
merges, overlap ties, the 256-track cap), over whole detector runs with zero-frame feeds and ragged feed splits, and
show that a statement with one deliberate mistake is rejected by a named case."""
import numpy as np
import pytest

import chdet_stmt as cs
import chtrack_oracle as co
import chtrack_stmt as kt

BETAS = (1.0, 0.5, 0.01)
HOLDS = (0, 1, 7)

# deliberate mistake -> (scene, beta, hold) that must catch it
MISTAKE_CASES = {
    "first_overlap": ("merge", 0.5, 1),
    "insert_first": ("cap_dropped", 0.5, 0),
    "misses_ge": ("appear_vanish_return", 0.5, 1),
    "smooth_unmatched": ("appear_vanish_return", 0.5, 7),
}


def oracle_drive(lists, beta, hold):
    t = co.Tracker(beta, hold)
    out = []
    for lst in lists:
        t.update(lst)
        out.append((t.keys(), t.dropped, t.next_id))
    return out


def scene(name):
    return {n: s for n, s in kt.list_scenes()}[name]


@pytest.mark.parametrize("beta", BETAS)
@pytest.mark.parametrize("hold", HOLDS)
def test_oracle_equals_statement_lists(oracle, beta, hold):
    """Every list scene: ranges, S0 bits, ids, age, present, misses, dropped and next_id, update after update."""
    for name, lists in kt.list_scenes():
        assert oracle_drive(lists, beta, hold) == kt.drive(lists, beta, hold), (name, beta, hold)


def detector_lists(oracle, N, prm, feeds):
    """The oracle's K.4 lists of every feed with frames (KT.1), and the statement's (they are equal: SPEC K)."""
    o = oracle.ChannelDetector(N, prm["alpha"], prm["gamma"], prm["snr"], prm["min_bins"])
    st = cs.Detector(N, prm["alpha"], prm["gamma"], prm["snr"], prm["min_bins"])
    ref, mine = [], []
    try:
        for f in feeds:
            frames = f[0]
            r, _ = o.feed(frames)
            m, _ = st.feed(frames)
            if len(frames) == 0:
                continue
            ref.append([(a, b, np.float32(s0)) for a, b, s0, _n0, _snr in r])
            mine.append([(c.bin_lo, c.bin_hi, c.S0) for c in m])
    finally:
        o.close()
    return ref, mine


def bursty_feeds(N, frames, seed=1):
    """A carrier near the threshold that drops out and returns, a bursty one, and a steady one."""
    rng = np.random.default_rng(seed)
    out = []
    for i, f in enumerate(frames):
        p = rng.exponential(1.0, (1, f, N)).astype(np.float32)
        p[..., N // 8:N // 8 + N // 64] += 30.0
        if i % 3 != 1:
            p[..., N // 3:N // 3 + N // 32] += 12.0 if i % 2 else 3.0
        if i % 4 == 0:
            p[..., 5 * N // 8:5 * N // 8 + N // 16] += 40.0 * (1 + i % 3)
        out.append(p)
    return out


@pytest.mark.parametrize("N", [64, 1024, 16384])
@pytest.mark.parametrize("beta,hold", [(1.0, 0), (0.5, 1), (0.01, 7)])
def test_oracle_equals_statement_detector_runs(oracle, N, beta, hold):
    """K then KT over the detector scenes of tests/chdet_stmt.py (zero-frame feeds included) and a bursty scene."""
    sc = [(n, p, f) for n, p, f in cs.scenes(N)]
    sc.append(("bursty", dict(alpha=0.5, gamma=0.25, snr=4.0, min_bins=2), bursty_feeds(N, [1, 2, 0, 1, 3, 1, 0, 2, 1, 1])))
    for name, prm, feeds in sc:
        ref, mine = detector_lists(oracle, N, prm, feeds)
        assert oracle_drive(ref, beta, hold) == kt.drive(mine, beta, hold), (name, N, beta, hold)


def test_zero_frame_feeds_and_ragged_splits(oracle):
    """KT.1: zero-frame feeds are no-ops wherever they fall; a ragged split changes the tracks only through K's lists."""
    N = 1024
    prm = dict(alpha=0.5, gamma=0.25, snr=4.0, min_bins=2)
    frames = bursty_feeds(N, [1] * 12, seed=3)
    allf = np.concatenate(frames, axis=1)

    def split(sizes):
        out, at = [], 0
        for s in sizes:
            out.append(allf[:, at:at + s])
            at += s
        assert at == allf.shape[1]
        return out
    plain = split([2, 3, 1, 4, 2])
    zeros = split([0, 2, 0, 0, 3, 1, 0, 4, 2, 0])
    ragged = split([1, 1, 5, 2, 3])
    for beta, hold in [(0.5, 1), (0.01, 7)]:
        a = oracle_drive(detector_lists(oracle, N, prm, plain)[0], beta, hold)
        b = oracle_drive(detector_lists(oracle, N, prm, zeros)[0], beta, hold)
        assert a == b
        ref, mine = detector_lists(oracle, N, prm, ragged)
        assert oracle_drive(ref, beta, hold) == kt.drive(mine, beta, hold)
        assert len(ref) == 5


@pytest.mark.parametrize("N", [256, 4096])
def test_beta1_hold0_is_the_detector_list(oracle, N):
    """With beta = 1 and hold = 0 the tracked ranges are the K.4 list, update by update, and S0 is
    S0 + (S0_d - S0) in binary32: S0_d itself for a new track and wherever the difference is exact (Sterbenz,
    S0 / 2 <= S0_d <= 2 S0), one rounding of the difference away otherwise (as K.1 at alpha = 1)."""
    sc = list(cs.scenes(N)) + [("bursty", dict(alpha=0.5, gamma=0.25, snr=4.0, min_bins=2),
                                bursty_feeds(N, [1, 2, 1, 3, 1, 2]))]
    exact = 0
    for name, prm, feeds in sc:
        ref, _ = detector_lists(oracle, N, prm, feeds)
        t = co.Tracker(1.0, 0)
        prev = {}
        for lst in ref:
            got = t.update(lst)
            assert [(a, b) for a, b, *_ in got] == [(a, b) for a, b, _ in lst], name
            for (a, b, s0d), (_, _, bits, id_, *_r) in zip(lst, got):
                s0d = np.float32(s0d)
                old = prev.get(id_)
                want = s0d if old is None else np.float32(old + np.float32(s0d - old))
                assert bits == int(want.view(np.uint32)), name
                if old is None or old / 2 <= s0d <= 2 * old:
                    assert bits == int(s0d.view(np.uint32)), name
                    exact += 1
            prev = {id_: np.uint32(bits).view(np.float32) for _, _, bits, id_, *_r in got}
    assert exact > 100


@pytest.mark.parametrize("mistake", kt.MISTAKES)
def test_statement_mistakes_are_caught(oracle, mistake):
    """Each planted mistake makes its named case disagree with the oracle, which the correct statement matches."""
    name, beta, hold = MISTAKE_CASES[mistake]
    lists = scene(name)
    ref = oracle_drive(lists, beta, hold)
    assert kt.drive(lists, beta, hold) == ref
    assert kt.drive(lists, beta, hold, mistake=mistake) != ref, (mistake, name)


def test_scene_edges_hold():
    """The scenes reach what they are named for (checked on the statement, which equals the oracle above)."""
    t = kt.Tracker(0.5, 1)
    lists = scene("cap_dropped")
    t.update(lists[0])
    assert len(t.tracks) == kt.CAP and t.dropped == 0
    t.update(lists[1])
    assert len(t.tracks) == kt.CAP and t.dropped == kt.CAP and all(x.misses == 1 for x in t.tracks)
    t.update(lists[2])
    assert len(t.tracks) == kt.CAP and [x.id for x in t.tracks] == list(range(kt.CAP + 1, 2 * kt.CAP + 1))
    assert t.dropped == kt.CAP
    # merge: the right track overlaps the merged run more, and wins although it comes second
    t = kt.Tracker(0.5, 1)
    for lst in scene("merge")[:3]:
        t.update(lst)
    assert [(x.a, x.b, x.id, x.misses) for x in t.tracks] == [(100, 130, 1, 1), (100, 200, 2, 0)]
    # ties: equal overlaps go to the smaller a; equal a to the smaller id
    t = kt.Tracker(1.0, 1)
    for lst in scene("tie_a")[:2]:
        t.update(lst)
    assert [(x.a, x.id, x.misses) for x in t.tracks] == [(105, 1, 0), (120, 2, 1)]
    t = kt.Tracker(1.0, 7)
    for lst in scene("tie_id")[:4]:
        t.update(lst)
    assert [(x.a, x.id, x.misses) for x in t.tracks] == [(201, 1, 3), (201, 2, 0)]
    t.update(scene("tie_id")[4])
    assert [(x.a, x.b, x.id, x.misses) for x in t.tracks] == [(201, 205, 1, 0), (201, 205, 2, 1)]
    # a carrier returning within the hold keeps its id; beyond it, it opens a new one
    t = kt.Tracker(0.5, 7)
    ids = set()
    for lst in scene("appear_vanish_return"):
        t.update(lst)
        ids |= {x.id for x in t.tracks if x.a == 300}
    assert len(ids) == 2


def test_statement_known_answers():
    """Hand-checked: smoothing in binary32, age / present / misses, removal one update after the hold."""
    t = kt.Tracker(0.25, 1)
    t.update([(10, 20, np.float32(8.0))])
    t.update([(11, 21, np.float32(16.0))])
    (x,) = t.tracks
    assert (x.a, x.b, float(x.S0), x.id, x.age, x.present, x.misses) == (11, 21, 10.0, 1, 2, 2, 0)
    t.update([])
    (x,) = t.tracks
    assert (x.a, float(x.S0), x.age, x.present, x.misses) == (11, 10.0, 3, 2, 1)
    t.update([])
    assert t.tracks == [] and t.next_id == 2
    t.update([(0, 5, np.float32(1.0)), (30, 40, np.float32(2.0))])
    assert [(x.a, x.id) for x in t.tracks] == [(0, 2), (30, 3)]
    assert kt.snr(t.tracks[1], np.float32(4.0)) == np.float32(0.5)
