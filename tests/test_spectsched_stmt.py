"""The statement of SPEC US (tests/spectsched_stmt.py) against the whole-stream definition, without a GPU: every
emission of the feed-by-feed schedule, with its carried history, equals the oracle's U.1-U.5 over the stream's prefix
up to t_j, bit for bit, for every spectrum kind and both estimators."""
import numpy as np
import pytest

from sigdigger_b200 import synth
from spectsched_stmt import MISTAKES, reference, same, schedule

KINDS = ["psd", "cyclo", "fmspect", "timediff", "abstimediff", "exp_2", "exp_4", "exp_8", "fac"]
FS = 48000.0


def _stream(n, seed):
    sig, _ = synth.psk_signal(n, 8.0, order=4, seed=seed)
    rng = np.random.default_rng(seed)
    return (0.5 * sig + synth.awgn(n, 1e-3, rng)).astype(np.complex64)


def _frame_fn(oracle, ns, kinds):
    def fn(c):
        out = [oracle.spectsrc_frame(k, ns, c) for k in kinds]
        out += [oracle.estimate_baud(e, ns, FS, c) for e in ("baud-fac", "baud-nonlinear")]
        return out
    return fn


def _split(n, how, ns, seed):
    rng = np.random.default_rng(seed)
    if how == "one":
        return [n]
    if how == "ragged":       # 1 ... 3 Ns samples a feed
        hi = 3 * ns
    else:                     # "short": every feed shorter than Ns
        hi = max(2, ns // 3)
    sizes = []
    while sum(sizes) < n:
        sizes.append(int(rng.integers(1, hi + 1)))
    sizes[-1] -= sum(sizes) - n
    return [s for s in sizes if s > 0]


def _run(oracle, ns, I, how, n, kinds, mistake=None, seed=1):
    c = _stream(n, seed)
    fn = _frame_fn(oracle, ns, kinds)
    pos, feeds = 0, []
    for s in _split(n, how, ns, seed + 7):
        feeds.append(c[pos:pos + s])
        pos += s
    got, _ = schedule(feeds, ns, I, fn, mistake)
    return [x for em in got for x in em], reference(c, ns, I, fn)


def _length(ns, I):
    # a few emissions past the first: at most ~24 frames, at least two emission points past Ns + 1
    return ns + 1 + max(2 * I, min(24 * I, 3 * ns)) + 5


@pytest.mark.parametrize("ns", [64, 1024, 4096])
@pytest.mark.parametrize("Ifac", ["1", "ns/2", "ns+1", "3ns+7", "1e5"])
@pytest.mark.parametrize("how", ["one", "ragged", "short"])
def test_schedule_equals_whole_stream(oracle, ns, Ifac, how):
    I = {"1": 1, "ns/2": ns // 2, "ns+1": ns + 1, "3ns+7": 3 * ns + 7, "1e5": 100000}[Ifac]
    n = _length(ns, I)
    got, want = _run(oracle, ns, I, how, n, KINDS)
    assert len(want) >= 2 and want[0][0] >= ns + 1
    assert same(got, want), (ns, I, how)


def test_several_emissions_per_feed_and_none(oracle):
    """A feed of 5 I + 3 samples emits at the four points past Ns + 1, a 27-sample feed between two points emits
    nothing, and the rest emit at every point, all equal to the whole-stream frames."""
    ns, I = 64, 40
    c = _stream(2000, 9)
    fn = _frame_fn(oracle, ns, ["psd"])
    got, _ = schedule([c[:203], c[203:230], c[230:2000]], ns, I, fn)
    assert [len(g) for g in got] == [4, 0, 45]
    assert [t for t, _ in got[0]] == [80, 120, 160, 200]
    assert same([x for g in got for x in g], reference(c, ns, I, fn))


def test_carry_across_replan_and_interval_change(oracle):
    """US.5: carrying the state over gives the uninterrupted result; after a change of I, the points whose frame
    reaches before the kept samples are skipped and every other one is the whole-stream frame."""
    ns, I = 256, 1000
    c = _stream(12000, 3)
    fn = _frame_fn(oracle, ns, ["psd"])
    a, st = schedule([c[:3100]], ns, I, fn)
    b, _ = schedule([c[3100:7000], c[7000:]], ns, I, fn, state=st)
    assert same([x for g in a + b for x in g], reference(c, ns, I, fn))
    # I 1000 -> 300 at t = 3100: the next point of I = 1000 was 4000, whose frame starts at 3743 > 3100, so the
    # history kept nothing (v = 3100); 3300 would need samples from before 3100 and is skipped, 3600 is the first
    a, st = schedule([c[:3100]], ns, I, fn)
    assert st[2] == 3100
    b, _ = schedule([c[3100:]], ns, 300, fn, state=st)
    want = [(t, r) for t, r in reference(c, ns, 300, fn) if t > 3100 and t - ns - 1 >= st[2]]
    assert want[0][0] == 3600 and same(b[0], want)


@pytest.mark.parametrize("mistake,case", [
    ("frame_ends_early", dict(ns=64, I=32, how="ragged")),
    ("emits_before_ns1", dict(ns=64, I=1, how="one")),
    ("history_not_carried", dict(ns=1024, I=1025, how="short")),
])
def test_planted_mistakes_are_rejected(oracle, mistake, case):
    assert mistake in MISTAKES
    ns, I, how = case["ns"], case["I"], case["how"]
    got, want = _run(oracle, ns, I, how, _length(ns, I), ["psd"], mistake)
    assert not same(got, want), mistake
    got, want = _run(oracle, ns, I, how, _length(ns, I), ["psd"])
    assert same(got, want)
