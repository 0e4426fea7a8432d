"""-m gpu: the analog-TV processor batch on the GPU (k_tv_feed, one warp per processor) against the oracle, bit for
bit: frame counts, every frame still in the ring, the picture in progress, the loop estimates; block-size independence;
the TV tab's input conversion.  Through the C-ABI (sdb_tv_processor_*)."""
import ctypes as C

import numpy as np
import pytest

import test_oracle_tv as T
import sigdigger_b200 as sdb_mod

pytestmark = pytest.mark.gpu


def _params(lines, interlace, trigger, comb):
    o = T.toy_params(lines, interlace, trigger, comb=comb)
    p = sdb_mod.TvParams()
    for name, _ in sdb_mod.TvParams._fields_:
        setattr(p, name, getattr(o, name))
    return o, p


@pytest.mark.parametrize("interlace,lines,comb", [(False, 40, False), (True, 61, True)])
def test_tv_batch_bit_exact(sdb, oracle, interlace, lines, comb):
    o, p = _params(lines, interlace, 4, comb)
    B = 5
    sigs = []
    for b in range(B):
        x, _, _ = T.toy_signal(lines, interlace, frames=10, start=3.1 + 4.7 * b, amp=0.3 + 0.1 * b, noise=0.002 * (b + 1),
                               seed=10 + b)
        sigs.append(x)
    n = min(len(s) for s in sigs)
    X = np.stack([s[:n] for s in sigs])
    tv = sdb.TvProcessor(p, batch=B)
    assert (tv.width, tv.height) == (int(np.floor(T.LINE)), lines)
    done = tv.feed(X)
    counts = tv.frames()
    for b in range(B):
        t = T.OracleTv(o)
        assert t.feed(X[b]) == int(done[b]) == int(counts[b]) and done[b] >= 8
        for f in range(max(0, t.frames - 3), t.frames + 1):          # three completed frames + the one in progress
            assert np.array_equal(tv.read_frame(b, f).view(np.uint32), t.frame(f).view(np.uint32)), (b, f)
        assert np.array_equal(np.float32(tv.estimates(b)).view(np.uint32), np.float32(t.estimates()).view(np.uint32))
        t.close()
    with pytest.raises(sdb.SdbError):
        tv.read_frame(0, int(counts[0]) + 1)
    tv.close()


def test_tv_block_size_independence_and_live_params(sdb, oracle):
    lines = 40
    o, p = _params(lines, False, 4, True)
    x, _, _ = T.toy_signal(lines, False, frames=8)
    one = sdb.TvProcessor(p, batch=1)
    one.feed(x[None, :])
    ragged = sdb.TvProcessor(p, batch=1)
    pos, rng, total = 0, np.random.default_rng(4), 0
    while pos < x.size:
        k = int(rng.integers(1, 9000))
        total += int(ragged.feed(x[None, pos:pos + k])[0])
        pos += k
    assert total == int(one.frames()[0]) == int(ragged.frames()[0])
    f = int(one.frames()[0])
    for no in (f - 1, f):
        assert np.array_equal(one.read_frame(0, no).view(np.uint32), ragged.read_frame(0, no).view(np.uint32))
    # a live parameter change takes effect at the next sample, on both sides alike
    t = T.OracleTv(o)
    t.feed(x)
    o.l_tol, p.l_tol = 0.15, 0.15
    o.hsync_fast_track_tau = p.hsync_fast_track_tau = 5.0
    assert T.tv_lib().sdo_tv_set_params(t.h, C.byref(o)) == 1
    one.set_params(p)
    x2, _, _ = T.toy_signal(lines, False, frames=4, start=0.4, seed=9)
    one.feed(x2[None, :])
    t.feed(x2)
    assert int(one.frames()[0]) == t.frames
    assert np.array_equal(one.read_frame(0, t.frames - 1).view(np.uint32), t.frame(t.frames - 1).view(np.uint32))
    p.frame_lines = 50
    with pytest.raises(sdb.SdbError):
        one.set_params(p)
    bad = sdb_mod.TvParams.from_buffer_copy(p)
    bad.frame_lines, bad.hsync_len = 40, 0.4
    with pytest.raises(sdb.SdbError):
        sdb.TvProcessor(bad)
    for h in (one, ragged):
        h.close()
    t.close()


def test_tv_pal_preset_full_size(sdb, oracle):
    """625-line PAL at 8 MS/s (512 samples per line), 4 frames: the preset geometry end to end"""
    o = T.OL.TvParams()
    T.tv_lib().sdo_tv_params_pal(C.byref(o), 8e6)
    p = sdb.tv_params("pal", 8e6)
    assert bytes(o) == bytes(p)
    from sigdigger_b200 import synth
    rng = np.random.default_rng(5)
    pic = rng.random((625, 32)).repeat(4, axis=1)
    x, _ = synth.tv_composite(512.0, 32.0, 16.0, 625, True, 4, pic, amp=0.6, noise=0.003)
    tv = sdb.TvProcessor(p, batch=2)
    X = np.stack([x, x[::-1].copy()])
    done = tv.feed(X)
    t = T.OracleTv(o)
    assert t.feed(X[0]) == int(done[0]) >= 2
    assert np.array_equal(tv.read_frame(0, t.frames - 1).view(np.uint32), t.frame(t.frames - 1).view(np.uint32))
    t.close()
    tv.close()


def test_tv_feed_transform_bit_exact(sdb, oracle):
    L = T.tv_lib()
    rng = np.random.default_rng(6)
    x = (rng.standard_normal(100003) + 1j * rng.standard_normal(100003)).astype(np.complex64)
    ref = np.empty(x.size, np.float32)
    for mode, name, k, dc in ((0, "modulus", -1.0, 0.3), (1, "argument", 1.0, -0.05)):
        L.sdo_tv_feed_transform(x.ctypes.data, x.size, mode, k, dc, ref.ctypes.data)
        assert np.array_equal(sdb.tv_feed_transform(x, name, k, dc).view(np.uint32), ref.view(np.uint32))
