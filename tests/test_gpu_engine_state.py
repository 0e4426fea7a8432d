"""-m gpu: the engine's committed state and its feed-parity slots.

A commit that fails leaves nothing behind, so a corrected commit runs exactly what an engine configured correctly from
the start runs.  Host and device feeds may be mixed with asynchronous reads: host-input staging keeps its own parity
beside the feed parity of the result slots.  The device-pointer accessors return the slot of the latest feed, slot 0
before the first."""
import numpy as np
import pytest
import torch

from sigdigger_b200 import synth

pytestmark = pytest.mark.gpu

SPECS = [("qpsk", 0.10, 1 / 128.), ("qpsk", 0.30, 1 / 160.)]


def _signal(S, n, seed):
    xs = [synth.multi_carrier(n, 1.0, [(k, f, b, -14.0, {}) for k, f, b in SPECS], noise_db=-50.0, seed=seed + s)[0]
          for s in range(S)]
    return np.ascontiguousarray(np.stack(xs).astype(np.complex64))


def _engine(sdb, S, N, n, costas_order_1=2):
    e = sdb.Engine(n_streams=S, psd_size=N, psd_window="hann", max_feed=n)
    hs = []
    for i, (_, f, baud) in enumerate(SPECS):
        h = e.open_channel(2 * np.pi * f, 2 * np.pi * 3 * baud, 1.0)
        e.set_inspector(h, "psk", baud=baud, costas_order=costas_order_1 if i == 1 else 2, bits_per_symbol=2,
                        loop_bw=e.channel_rate(h) * 2e-3, mf_type=1, clock_type=1, clock_gain=0.1)
        hs.append(h)
    return e, hs


def _symbols(e, chains):
    cap = e.symbol_capacity
    cnt = np.zeros(chains, np.uint32)
    soft = np.zeros((chains, cap), np.complex64)
    hard = np.zeros((chains, cap), np.uint8)
    e.read_all_symbols(cnt, soft, hard, cap)
    return cnt, [soft[c, :m].copy() for c, m in enumerate(cnt)], [hard[c, :m].copy() for c, m in enumerate(cnt)]


@pytest.mark.parametrize("N", [16384, 65536])
def test_failed_commit_then_corrected_commit(sdb, N):
    """An invalid inspector configuration (costas_order 4) fails the commit after the transforms, the channel plan
    and the streams have been built.  Corrected and committed again, the engine gives bit for bit what an engine
    configured correctly from the start gives, over three feeds: PSD, channel samples and symbols.  N = 16384 runs the
    two-kernel transforms with the PSD on its own stream, N = 65536 the cluster transform."""
    S, feeds = 2, 3
    n = 4 * N if N < 65536 else 2 * N
    x = _signal(S, feeds * n, 40)
    retried, hs = _engine(sdb, S, N, n, costas_order_1=4)
    with pytest.raises(sdb.SdbError, match="invalid inspector configuration"):
        retried.commit()
    _, f, baud = SPECS[1]
    retried.set_inspector(hs[1], "psk", baud=baud, costas_order=2, bits_per_symbol=2,
                          loop_bw=retried.channel_rate(hs[1]) * 2e-3, mf_type=1, clock_type=1, clock_gain=0.1)
    retried.commit()
    fresh, _ = _engine(sdb, S, N, n)
    fresh.commit()
    chains = S * len(hs)
    total = 0
    for i in range(feeds):
        outs = []
        for e in (retried, fresh):
            e.feed(x[:, i * n:(i + 1) * n])
            chans = [e.read_channel(s, h) for s in range(S) for h in hs]
            outs.append((e.read_psd().copy(), chans, _symbols(e, chains)))
        (pa, ca, (na, sa, ha)), (pb, cb, (nb, sb, hb)) = outs
        assert np.array_equal(pa.view(np.uint32), pb.view(np.uint32)), "PSD of feed %d" % i
        for j, (a, b) in enumerate(zip(ca, cb)):
            assert len(a) == len(b) > 0 and np.array_equal(a.view(np.uint32), b.view(np.uint32)), \
                "feed %d, stream %d, channel %d" % (i, j // len(hs), j % len(hs))
        assert np.array_equal(na, nb), "symbol counts of feed %d" % i
        for c in range(chains):
            assert np.array_equal(sa[c].view(np.uint32), sb[c].view(np.uint32)) and np.array_equal(ha[c], hb[c]), (i, c)
        total += int(nb.sum())
    assert total > 0
    retried.close()
    fresh.close()


def test_host_and_device_feeds_with_async_reads(sdb):
    """Host, device, host, host, device feeds, each followed by read_psd_async and read_symbols_packed_async, with one
    sync at the end: the staging parity (host feeds only) and the feed parity come apart.  Every result equals the
    blocking reads of an identical engine fed synchronously."""
    S, N, kinds = 3, 16384, ["host", "device", "host", "host", "device"]
    n = 4 * N
    x = _signal(S, len(kinds) * n, 50)
    segs = [np.ascontiguousarray(x[:, i * n:(i + 1) * n]) for i in range(len(kinds))]
    dev = [torch.from_numpy(s).cuda() if k == "device" else None for s, k in zip(segs, kinds)]
    torch.cuda.synchronize()
    pin = lambda shape, dt: torch.zeros(shape, dtype=dt, pin_memory=True).numpy()

    def bufs(e):
        chains, cap = S * len(SPECS), e.symbol_capacity
        total_cap = chains * ((cap + 15) // 16 * 16)
        return dict(psd=pin((S, n // N, N), torch.float32), cnt=pin((chains,), torch.int32).view(np.uint32),
                    off=pin((chains + 1,), torch.int64).view(np.uint64), soft=pin((total_cap,), torch.complex64),
                    hard=pin((total_cap,), torch.uint8)), total_cap

    ref_e, _ = _engine(sdb, S, N, n)
    ref_e.commit()
    ref = []
    for s in segs:
        ref_e.feed(s)
        o, total_cap = bufs(ref_e)
        ref_e.read_psd(o["psd"])
        ref_e.read_symbols_packed(o["cnt"], o["off"], o["soft"], o["hard"], total_cap)
        ref.append(o)
    e, _ = _engine(sdb, S, N, n)
    e.commit()
    outs = []
    for s, d, k in zip(segs, dev, kinds):
        if k == "host":
            e.feed_host_ptr(s.ctypes.data, n, n)
        else:
            e.feed_device_ptr(d.data_ptr(), n, n)
        o, total_cap = bufs(e)
        e.read_psd_async(o["psd"])
        e.read_symbols_packed_async(o["cnt"], o["off"], o["soft"], o["hard"], total_cap)
        outs.append(o)
    e.sync()
    for i, (o, r) in enumerate(zip(outs, ref)):
        assert np.array_equal(o["psd"].view(np.uint32), r["psd"].view(np.uint32)), "PSD of feed %d" % i
        assert np.array_equal(o["cnt"], r["cnt"]) and np.array_equal(o["off"], r["off"]), "counts of feed %d" % i
        end = int(r["off"][-1])
        assert np.array_equal(o["soft"][:end].view(np.uint32), r["soft"][:end].view(np.uint32)), "soft of feed %d" % i
        assert np.array_equal(o["hard"][:end], r["hard"][:end]), "hard of feed %d" % i
    assert sum(int(r["cnt"].sum()) for r in ref) > 0
    e.close()
    ref_e.close()


def test_slot_accessors(sdb):
    """Before its commit an engine has no slots: psd_device is null and reading a channel or its symbols fails.  After
    the commit, psd_device and the symbol-count pointer name slot 0 until the first feed, then the slot of the latest
    feed: slot 0 after the first, and alternating from there."""
    S, N = 1, 16384
    n = 2 * N
    x = _signal(S, 4 * n, 60)
    e, hs = _engine(sdb, S, N, n)
    assert e.psd_device_ptr is None
    with pytest.raises(sdb.SdbError, match="engine not committed"):
        e.read_channel(0, hs[0])
    with pytest.raises(sdb.SdbError, match="engine not committed"):
        e.read_symbols(0, hs[0])
    e.commit()
    counts = lambda: e._L.sdb_engine_symbol_counts_device(e._h)
    p0, c0 = e.psd_device_ptr, counts()
    assert p0 and c0
    seen = []
    for i in range(4):
        e.feed(x[:, i * n:(i + 1) * n])
        seen.append((e.psd_device_ptr, counts()))
    assert seen[0] == (p0, c0)                                    # the first feed fills slot 0
    assert seen[1][0] != p0 and seen[1][1] != c0
    assert seen[2] == (p0, c0) and seen[3] == seen[1]
    e.close()
