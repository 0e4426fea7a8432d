"""-m gpu: the analog-TV processor batch on the GPU (k_tv_feed, one warp per processor) against the oracle, bit for
bit: frame counts, every frame still in the ring, the picture in progress, the loop estimates; block-size independence;
the TV tab's input conversion.  Through the C-ABI (sdb_tv_processor_*).  Every scene of tests/test_tv_stmt.py runs as
one batch with its live parameter changes, against the oracle and the statement; the geometry edges (line_len 8,
8.5, 4096, 4096.5, H = 2, an interlaced 2049-line picture, the NTSC preset) are scenes of that table; a batch larger
than a wave of SMs; feed splits around the kernel's 32-sample loads; the device feed and its stride check."""
import ctypes as C

import numpy as np
import pytest

import test_oracle_tv as T
import test_tv_stmt as TS
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


# ---- the scene table of tests/test_tv_stmt.py through k_tv_feed ----------------------------------------------------

def _sdb_params(d):
    p = sdb_mod.TvParams()
    for name, _ in sdb_mod.TvParams._fields_:
        setattr(p, name, d[name])
    return p


def _batch(scene, B):
    sigs = [scene.signal(v) for v in range(B)]
    n = min(s.size for s in sigs)
    return np.stack([s[:n] for s in sigs])


def _check_window(tv, b, frames, pics):
    """frames - 3 ... frames readable and equal; frames - 4 and frames + 1 refused"""
    assert set(pics) == set(TS.readable(frames))
    for f, pic in pics.items():
        assert np.array_equal(tv.read_frame(b, f).view(np.uint32), TS.bits(pic)), (b, f)
    for f in (frames - 4, frames + 1):
        if f >= 0:
            with pytest.raises(sdb_mod.SdbError):
                tv.read_frame(b, f)


@pytest.mark.parametrize("name", [s.name for s in TS.SCENES])
def test_tv_scene_batch_bit_exact(sdb, oracle, name):
    """one batch per scene, a different signal per processor, live parameter changes between feeds on both sides:
    after every feed, frame counts, the readable window and the estimates equal the oracle's (and, for the scenes short
    enough, the statement's on processor 0)"""
    scene = TS.BY_NAME[name]
    B = 2 if scene.long else 3
    X = _batch(scene, B)
    refs = [TS.run_oracle(scene, X[b]) for b in range(B)]
    stmt = None if scene.long else TS.run_stmt(scene, X[0])[0]
    p = dict(scene.params)
    tv = sdb.TvProcessor(_sdb_params(p), batch=B)
    pos = 0
    for i, (k, ch) in enumerate(TS.plan(scene, X.shape[1])):
        if ch:
            p.update(ch)
            tv.set_params(_sdb_params(p))
        if k:
            tv.feed(X[:, pos:pos + k])
        pos += k
        counts = tv.frames()
        for b in range(B):
            frames, pics, est = refs[b][i]
            assert int(counts[b]) == frames, (i, b)
            _check_window(tv, b, frames, pics)
            assert np.array_equal(np.float32(tv.estimates(b)).view(np.uint32), TS.bits(est)), (i, b)
        if stmt is not None:
            assert TS.same([refs[0][i]], [stmt[i]]), i
    assert refs[0][-1][0] >= 1
    tv.close()


def test_tv_batch_of_300(sdb, oracle):
    """more processors than a wave of SMs, each with its own signal"""
    scene = TS.BY_NAME["acquire"]
    B = 300
    X = _batch(scene, B)[:, :12000]
    tv = sdb.TvProcessor(_sdb_params(scene.params), batch=B)
    done = tv.feed(X)
    for b in range(B):
        t = T.OracleTv(TS._struct(scene.params))
        assert t.feed(X[b]) == int(done[b]) == int(tv.frames()[b])
        for f in TS.readable(t.frames):
            assert np.array_equal(tv.read_frame(b, f).view(np.uint32), t.frame(f).view(np.uint32)), (b, f)
        assert np.array_equal(np.float32(tv.estimates(b)).view(np.uint32), np.float32(t.estimates()).view(np.uint32))
        t.close()
    tv.close()


def test_tv_feed_splits_equal_one_feed(sdb, oracle):
    """feeds of 1, 31, 32 and 33 samples (around the kernel's 32-sample load), then a random split"""
    scene = TS.BY_NAME["interlaced_odd"]
    X = _batch(scene, 2)
    p = _sdb_params(scene.params)
    whole, split = sdb.TvProcessor(p, batch=2), sdb.TvProcessor(p, batch=2)
    whole.feed(X)
    pos, rng = 0, np.random.default_rng(11)
    for k in (1, 31, 32, 33, 1, 1, 33):
        split.feed(X[:, pos:pos + k])
        pos += k
    while pos < X.shape[1]:
        k = int(rng.integers(1, 20000))
        split.feed(X[:, pos:pos + k])
        pos += k
    assert np.array_equal(whole.frames(), split.frames())
    f = int(whole.frames()[0])
    for b in range(2):
        for no in TS.readable(int(whole.frames()[b])):
            assert np.array_equal(whole.read_frame(b, no).view(np.uint32), split.read_frame(b, no).view(np.uint32))
        assert whole.estimates(b) == split.estimates(b)
    assert f >= 2
    whole.close()
    split.close()


def test_tv_device_feed_equals_host_feed(sdb, oracle):
    """sdb_tv_processor_feed_device from a torch tensor whose rows are longer than the feed; stride < n refused"""
    import torch
    scene = TS.BY_NAME["acquire"]
    X = _batch(scene, 3)
    n, stride = X.shape[1] - 1000, X.shape[1]
    p = _sdb_params(scene.params)
    host, dev = sdb.TvProcessor(p, batch=3), sdb.TvProcessor(p, batch=3)
    host.feed(X[:, :n])
    xd = torch.from_numpy(X).cuda()
    L = sdb.load_library()
    done = np.zeros(3, np.uint32)
    got = L.sdb_tv_processor_feed_device(dev._h, C.c_void_p(xd.data_ptr()), stride, n, done.ctypes.data)
    assert got == int(done.sum()) == int(host.frames().sum()) > 0
    for b in range(3):
        f = int(host.frames()[b])
        assert int(dev.frames()[b]) == f
        for no in TS.readable(f):
            assert np.array_equal(host.read_frame(b, no).view(np.uint32), dev.read_frame(b, no).view(np.uint32))
        assert host.estimates(b) == dev.estimates(b)
    before = dev.frames().copy()
    assert L.sdb_tv_processor_feed_device(dev._h, C.c_void_p(xd.data_ptr()), 100, 101, done.ctypes.data) < 0
    assert "stride" in sdb.last_error()
    assert np.array_equal(dev.frames(), before)
    host.close()
    dev.close()
