"""CPU: the Analog TV tab on an inspector (oracle/SPEC_TI.md).  The oracle runner (oracle/tvinsp.c) equals the statement
of TI.1-TI.3 (tests/tvinsp_stmt.py, over the exact SPEC TV statement tests/tv_stmt.py) bit for bit after every feed:
the posted frame and the status.  The scenes cover feeds that complete 0, 1 and 6 frames (more than the ring's 4), each
class, invert on and off with dc != 0, a mid-run parameter change, a refused geometry change and feeds without
symbols.  Each planted mistake of the statement is caught by the scene named for it."""
import numpy as np
import pytest

import test_tv_stmt as TS
import tvinsp_oracle as TO
import tvinsp_stmt as ST

FRAME = int(20 * TS.LINE)                  # samples per frame of the toy geometry (20 lines of 400.37 samples)


def symbols(cls, invert, dc, c, seed):
    """soft symbols whose TI.1 conversion is (about) the composite signal c"""
    rng = np.random.default_rng(seed)
    u = (c.astype(np.float64) - dc) / (-1.0 if invert else 1.0)
    if cls == "ask":
        assert u.size == 0 or u.min() >= 0
        return (u * np.exp(2j * np.pi * rng.random(u.size))).astype(np.complex64)
    return (rng.uniform(0.5, 1.5, u.size) * np.exp(1j * np.pi * u)).astype(np.complex64)


def cuts(x, sizes):
    out, a = [], 0
    for n in sizes:
        out.append(x[a:a + n])
        a += n
    return out


# name: (class, interlace, invert, dc, feed sizes, {feed index: (parameter changes, invert, dc)})
SCENES = {
    "ask_0_1_6": ("ask", False, False, -0.1, [0, 3000, FRAME, 6 * FRAME + 500, 0, 2000], {}),
    "psk_inverted": ("psk", False, True, 0.3, [FRAME // 2, 2 * FRAME, 0, 3 * FRAME], {}),
    "fsk_live_change": ("fsk", False, False, 0.2, [FRAME + 100, 2 * FRAME, 2 * FRAME],
                        {1: (dict(enable_agc=0, t_tol=0.15), False, 0.25), 2: (dict(reverse=1), True, 1.2)}),
    "psk_interlaced": ("psk", True, False, -0.05, [3 * FRAME, 0, 5 * FRAME], {}),
}


def scene_feeds(name):
    cls, inter, invert, dc, sizes, changes = SCENES[name]
    c = TS.composite(lines=20, interlace=inter, frames=sum(sizes) // FRAME + 2, amp=0.9, seed=5)
    feeds, inv, d = [], invert, dc
    for i, seg in enumerate(cuts(c, sizes)):
        if i in changes:
            inv, d = changes[i][1], changes[i][2]
        feeds.append(symbols(cls, inv, d, seg, seed=i))
    return cls, TS.base(lines=20, interlace=inter), invert, dc, feeds, changes


def run(name, mistake=None):
    """[(oracle posted, oracle status key, statement posted, statement status key)] per feed"""
    cls, p, invert, dc, feeds, changes = scene_feeds(name)
    o, s = TO.Tab(cls, p, invert, dc), ST.TabStmt(cls, p, invert, dc, mistake)
    out = []
    for i, x in enumerate(feeds):
        if i in changes:
            q = dict(p, **changes[i][0])
            assert o.set_params(q, changes[i][1], changes[i][2]) and s.set_params(q, changes[i][1], changes[i][2])
        o.feed(x)
        s.feed(x)
        out.append((o.posted, o.status.key(), s.posted, s.status_key()))
    return out


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("name", sorted(SCENES))
def test_oracle_equals_statement(name):
    completed = []
    for i, (op, ok, sp, sk) in enumerate(run(name)):
        assert ok == sk, (name, i, ok, sk)
        assert np.array_equal(bits(op), bits(sp)), (name, i)
        completed.append(ok[2])
    if name == "ask_0_1_6":
        assert completed == [0, 0, 1, 6, 0, 0], completed


def test_six_frames_post_the_first():
    """the 6-frame feed posts frame 2 (the feed's first), which the ring no longer holds after the feed"""
    cls, p, invert, dc, feeds, _ = scene_feeds("ask_0_1_6")
    o = TO.Tab(cls, p, invert, dc)
    for x in feeds[:4]:
        o.feed(x)
    st = o.status
    assert (st.frames, st.posted_no, st.completed) == (7, 2, 6)
    assert np.any(o.posted != 0)


def test_geometry_change_refused():
    cls, p, invert, dc, feeds, _ = scene_feeds("fsk_live_change")
    o, s = TO.Tab(cls, p, invert, dc), ST.TabStmt(cls, p, invert, dc)
    for q in (dict(p, frame_lines=22), dict(p, line_len=TS.LINE + 1), dict(p, interlace=1)):
        assert not o.set_params(q) and not s.set_params(q)


def test_invalid_parameters_and_classes_refused():
    with pytest.raises(ValueError):
        TO.Tab("ask", dict(TS.base(), line_len=4.0))
    with pytest.raises(KeyError):
        TO.Tab("audio", TS.base())


@pytest.mark.parametrize("mistake,name", [("post_last", "ask_0_1_6"), ("psk_modulus", "psk_inverted")])
def test_planted_mistake_is_caught(mistake, name):
    differs = any(ok != sk or not np.array_equal(bits(op), bits(sp)) for op, ok, sp, sk in run(name, mistake))
    assert differs, "%s: the planted mistake went unnoticed" % mistake
