"""Every path k_inspectors selects, against the oracle bit for bit, and a subset against the exact statement
(tests/chain_stmt.py).

The kernel picks its shared-memory lines and its loop variants per plan (`sdb_insp_dyn`, chain_kernels.cu); PATHS below
maps each selection rule to the scene that reaches it, and `test_path_table_is_covered` (CPU) checks that every scene
satisfies its rule.  Offline runs use batches of 33 (the second CTA holds one valid lane) and lengths of 16k + 1 and
16k + 15 samples, so the last 16-sample pipeline chunk is partial.  Engine scenes put 36 or more channels of one class
in one stream, so that one CTA holds lanes that differ in Costas kind, AGC, matched-filter length, channel size, CMA
and clock.running, and feed three feeds of different lengths so that the lines carry state across feeds."""
import types

import numpy as np
import pytest

import chain_cases as cc
import chain_stmt as cs

MF_RING_MAX = 209        # SDB_INSP_MF_RING_MAX
AGC_SMEM_ROWS = 160      # 2 dl_size + mh_size above this -> the AGC lines live in the global pool
DL_PRE_MIN = 16          # dl_size >= 16 (and in shared memory) -> the delay line is served by the pre warps
BATCH = 33
N_PSD = 4096

# path -> (scene, the rule's condition on that scene: its AGC design d, matched-filter span mf, bnor, baud, fs and
# length n in samples)
PATHS = {
    "agc lines in shared memory": ("ladder_T13.8", lambda c: 2 * c.d.dl_size + c.d.mh_size <= AGC_SMEM_ROWS),
    "agc lines in the global pool": ("ladder_T13.9", lambda c: 2 * c.d.dl_size + c.d.mh_size > AGC_SMEM_ROWS),
    "delay line in the track warp": ("ladder_T4.09", lambda c: c.d.dl_size < DL_PRE_MIN),
    "delay line in the pre warps": ("ladder_T4.1", lambda c: DL_PRE_MIN <= c.d.dl_size
                                    and 2 * c.d.dl_size + c.d.mh_size <= AGC_SMEM_ROWS),
    "matched filter in the ring": ("ladder_T34.8", lambda c: c.mf <= MF_RING_MAX),
    "matched filter in the global pool": ("ladder_T34.9", lambda c: c.mf > MF_RING_MAX),
    "matched-filter span cap 1024": ("ladder_T171", lambda c: c.mf == 1024 and c.n > 4 * c.mf),
    "agc line cap 4096": ("ladder_T1100", lambda c: c.d.dl_size == 4096 and c.n > 2 * c.d.dl_size),
    "bnor = 1": ("ladder_T1", lambda c: c.bnor == 1 and c.baud == c.fs),
    "bnor clamped to 1 (baud > fs)": ("psk_baud_above_fs", lambda c: c.bnor == 1 and c.baud > c.fs),
    "general Costas loop": ("engine:psk_mixed", "costas_order"),
    "general fsk loop": ("engine:fsk_mixed", "fsk_quad_demod"),
    "role_post general path": ("engine:psk_mixed", "agc_enabled"),
    "lanes of one CTA with different lengths": ("engine:psk_mixed", "size"),
    "a CTA with one valid lane": ("offline batch 33", None),
    "CMA in some lanes only": ("engine:psk_mixed", "eq_type"),
    "clock.running = 0 beside running lanes": ("engine:psk_mixed", "clock_running"),
    "clock.running toggled on a live chain": ("engine toggle", None),
    "matched filters from 19 to past 209 in one CTA": ("engine:psk_mixed", "mf"),
}

CASES = {c[0]: c[1:] for c in cc.cases() + cc.audio_cases()}
# raw channels are read from the channeliser, not run through k_inspectors
GPU_CASES = [name for name, c in CASES.items() if c[0] != "raw"]
# cases also held to the statement on the GPU (the four base inputs)
STMT_CASES = ("psk_qpsk_T4", "psk_8psk_T5", "psk_cma_T4", "fsk_quad_T5", "ask_pll1_ch2_T6.25", "ladder_T4.09",
              "ladder_T13.9", "ladder_T34.9", "audio_usb_sq1")


def case_cfg(name):
    cls, fs, kw, n = CASES[name]
    cfg = dict(insp_class=cs.INSP[cc.insp_class(cls)], fs=np.float32(fs), **kw)
    cfg["baud"] = np.float32(cfg["baud"])
    bnor = cs.bnor_of(cfg)
    T = np.float32(1.0) / bnor
    return types.SimpleNamespace(d=cs.AgcDesign(T), mf=cs.mf_span(T), bnor=bnor, baud=cfg["baud"], fs=cfg["fs"],
                                 n=16 * (n // 16) + 1)


# ---- engine scenes --------------------------------------------------------------------------------------------------
def psk_mixed_lanes():
    """36 psk lanes; every warp mixes Costas kinds 1-3, AGC on / off, matched filters of 19 to 240 taps (T 3.1 ... 40,
    across the 209-tap ring limit), 64- and 128-point channels; CMA on lanes 5 and 22; clock.running = 0 on lane 9"""
    Ts = (3.1, 4.5, 13.9, 34.8, 40.0, 6.0)
    out = []
    for k in range(36):
        kind = 1 + k % 3
        out.append(dict(size=64 if k % 4 < 3 else 128, T=Ts[k % len(Ts)],
                        kw=dict(costas_order=kind, bits_per_symbol=kind, mf_type=1 if k % 7 else 0,
                                agc_enabled=0 if k % 5 == 2 else 1, agc_gain_db=3.0, clock_type=1 if k % 6 else 0,
                                clock_gain=0.1, clock_phase=0.25, eq_type=1 if k in (5, 22) else 0, eq_rate=1e-2,
                                clock_running=0 if k == 9 else 1)))
    return out


def fsk_mixed_lanes():
    """34 fsk lanes with quad-demod alternating, two channel sizes"""
    return [dict(size=64 if k % 3 else 128, T=5.0 + (k % 4),
                 kw=dict(bits_per_symbol=1, fsk_quad_demod=k % 2, fsk_phase=0.1 * (k % 5), mf_type=1, clock_type=1,
                         clock_gain=0.2)) for k in range(34)]


ENGINE_SCENES = {"psk_mixed": ("psk", psk_mixed_lanes), "fsk_mixed": ("fsk", fsk_mixed_lanes)}


def scene_input(n, seed=0):
    from sigdigger_b200 import synth
    rng = np.random.default_rng(seed)
    x = synth.awgn(n, 0.05, rng)
    for f, sps in ((-0.31, 300.0), (0.07, 260.0), (0.33, 512.0)):
        s, _ = synth.psk_signal(n, sps, order=4, seed=int(sps))
        x = x + 0.3 * synth.mix(s, f)
    return x.astype(np.complex64)


def test_path_table_is_covered():
    """Every row of the path table has a scene, and the scene satisfies the selection rule it stands for."""
    for path, (scene, rule) in PATHS.items():
        if scene.startswith("engine:"):
            cls, lanes = ENGINE_SCENES[scene.split(":")[1]]
            lanes = lanes()
            warp = lanes[:32]
            if rule == "mf":
                mfs = {cs.mf_span(l["T"]) for l in warp if l["kw"]["mf_type"] == 1}
                assert min(mfs) == 19 and any(m <= MF_RING_MAX for m in mfs) and max(mfs) > MF_RING_MAX, path
            elif rule == "size":
                assert len({l["size"] for l in warp}) > 1, path
            elif rule in ("eq_type", "clock_running"):
                vals = [l["kw"][rule] for l in warp]
                assert 0 < sum(vals) < len(vals) or 0 < len(vals) - sum(vals) < len(vals), path
                assert len(set(vals)) == 2, path
            else:
                assert len({l["kw"].get(rule) for l in warp}) > 1, path
            assert len(lanes) >= 33
        elif scene == "offline batch 33":
            assert BATCH % 32 == 1
        elif scene == "engine toggle":
            assert [r for _, r in TOGGLE_FEEDS] == [1, 0, 1]
        else:
            assert scene in CASES, path
            assert rule(case_cfg(scene)), path
    rows = {"agc lines in the global pool", "delay line in the track warp", "delay line in the pre warps",
            "matched filter in the global pool", "matched-filter span cap 1024", "agc line cap 4096", "bnor = 1",
            "general Costas loop", "general fsk loop", "role_post general path",
            "lanes of one CTA with different lengths", "a CTA with one valid lane", "CMA in some lanes only",
            "clock.running = 0 beside running lanes"}
    assert rows <= set(PATHS)


# ---- offline task ---------------------------------------------------------------------------------------------------
def batch_inputs(cls, fs, kw, n):
    """[33, n]: the four base inputs, then the capture and the noise at further seeds"""
    xs = [cc.case_inputs(cls, fs, kw, n, seed=0)]
    seed = 1
    while sum(len(x) for x in xs) < BATCH:
        xs.append(cc.case_inputs(cls, fs, kw, n, seed=seed)[[1, 0, 3]])
        seed += 1
    return np.concatenate(xs)[:BATCH]


def _equal(soft, hard, rs, rh, audio=False):
    """soft (bits), counts and, except for audio (samples, not symbols), hard symbols"""
    return len(soft) == len(rs) and np.array_equal(soft.view(np.uint64), rs.view(np.uint64)) and \
        (audio or np.array_equal(hard, rh))


@pytest.mark.gpu
@pytest.mark.parametrize("tail", [1, 15])
@pytest.mark.parametrize("name", GPU_CASES)
def test_offline_chain_bit_exact(sdb, oracle, name, tail):
    cls, fs, kw, n = CASES[name]
    n = 16 * (n // 16) + tail
    x = batch_inputs(cls, fs, kw, n)
    got = sdb.inspector_run(cc.insp_class(cls), fs, x, **kw)
    cfg = oracle.insp_config(cc.insp_class(cls), fs, **kw)
    audio = cls == "audio"
    bad = [b for b in range(BATCH) if not _equal(*got[b], *oracle.inspector_run(cfg, x[b]), audio=audio)]
    assert bad == [], (name, n, bad)
    if name in STMT_CASES and tail == 15:
        st = cs.run({k: getattr(cfg, k) for k, _ in oracle.InspConfig._fields_}, x[:4])
        assert [b for b in range(4) if not _equal(*got[b], *st[b], audio=audio)] == [], name


# ---- engine scenes --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("scene", list(ENGINE_SCENES))
def test_engine_mixed_lanes(sdb, oracle, scene):
    cls, lanes = ENGINE_SCENES[scene]
    lanes = lanes()
    feeds = (40, 23, 61)
    x = scene_input(sum(feeds) * N_PSD, seed=len(lanes))
    e = sdb.Engine(n_streams=1, psd_size=N_PSD, psd_window="hann", max_feed=max(feeds) * N_PSD)
    hs, cfgs = [], []
    for k, l in enumerate(lanes):
        f = 0.05 + 0.9 * k / len(lanes)
        h = e.open_channel(2 * np.pi * f, 2 * np.pi * l["size"] / N_PSD, 1.0)
        assert e.channel_info(h).size == l["size"]
        fs_ch = e.channel_rate(h)
        kw = dict(l["kw"], baud=fs_ch / l["T"], loop_bw=fs_ch * 2e-3)
        e.set_inspector(h, cls, **kw)
        hs.append(h)
        cfgs.append(oracle.insp_config(cls, fs_ch, **kw))
    e.commit()
    chan = [[] for _ in hs]
    soft = [[] for _ in hs]
    hard = [[] for _ in hs]
    off = 0
    for m in feeds:
        e.feed(x[None, off:off + m * N_PSD])
        off += m * N_PSD
        for i, h in enumerate(hs):
            chan[i].append(e.read_channel(0, h))
            a, b = e.read_symbols(0, h)
            soft[i].append(a)
            hard[i].append(b)
    e.close()
    bad = []
    for i, cfg in enumerate(cfgs):
        rs, rh = oracle.inspector_run(cfg, np.concatenate(chan[i]))
        if not _equal(np.concatenate(soft[i]), np.concatenate(hard[i]), rs, rh):
            bad.append(i)
        if cfg.clock_running:
            assert len(rs) > 20, i
    assert bad == [], (scene, bad)


# ---- clock.running toggled on a live chain --------------------------------------------------------------------------
# (feed length in PSD frames, clock.running during that feed)
TOGGLE_FEEDS = ((40, 1), (23, 0), (31, 1))


def oracle_per_feed(oracle, cfg, chunks):
    """one oracle inspector fed chunk by chunk -> [(soft, hard)] per chunk"""
    import ctypes as C
    L = oracle.lib()
    h = L.sdo_inspector_new(C.byref(cfg))
    d = oracle.Decider()
    L.sdo_inspector_decider(C.byref(cfg), C.byref(d))
    out = []
    for x in chunks:
        x = np.ascontiguousarray(x, np.complex64)
        soft = np.empty(len(x) + 16, np.complex64)
        k = L.sdo_inspector_feed(h, oracle.ptr(x), len(x), oracle.ptr(soft), len(soft))
        soft = soft[:k].copy()
        hard = np.empty(k, np.uint8)
        if k:
            L.sdo_decider_decide(C.byref(d), oracle.ptr(soft), oracle.ptr(hard), k)
        out.append((soft, hard))
    L.sdo_inspector_destroy(h)
    return out


@pytest.mark.gpu
def test_engine_clock_running_toggle(sdb, oracle):
    """SPEC X: while clock.running = 0 the clock recovery and the CMA keep running and only the emission is dropped.
    The flag goes 1 -> 0 -> 1 on live chains (a migration between engines keeps their state); the symbols of the running feeds must
    equal those an always-running oracle chain emits during the same feeds.  A chain that froze its clock or its CMA
    while stopped, or restarted on the toggle, would emit different symbols in the last feed."""
    lanes = [dict(T=4.5, kw=dict(costas_order=2, bits_per_symbol=2, mf_type=1, clock_type=1, clock_gain=0.1,
                                 eq_type=1, eq_rate=1e-2)),
             dict(T=13.9, kw=dict(costas_order=3, bits_per_symbol=3, mf_type=1, clock_type=1, clock_gain=0.1)),
             dict(T=6.0, kw=dict(costas_order=1, bits_per_symbol=1, mf_type=0, clock_type=0, clock_phase=0.25,
                                 eq_type=1, eq_rate=2e-2))]
    import ctypes as C
    n = sum(m for m, _ in TOGGLE_FEEDS) * N_PSD
    x = scene_input(n, seed=5)
    L = sdb.load_library()

    def engine(running):
        e = sdb.Engine(n_streams=1, psd_size=N_PSD, psd_window="hann",
                       max_feed=max(m for m, _ in TOGGLE_FEEDS) * N_PSD)
        hs, kws = [], []
        for k, l in enumerate(lanes):
            h = e.open_channel(2 * np.pi * (0.05 + 0.3 * k), 2 * np.pi * 64 / N_PSD, 1.0)
            fs_ch = e.channel_rate(h)
            kw = dict(l["kw"], baud=fs_ch / l["T"], loop_bw=fs_ch * 2e-3)
            e.set_inspector(h, "psk", clock_running=running, **kw)
            hs.append(h)
            kws.append((fs_ch, kw))
        e.commit()
        return e, hs, kws

    cfgs = None
    chan = [[] for _ in lanes]
    got = [[] for _ in lanes]
    off, cur, hs, keep = 0, None, None, []
    for m, r in TOGGLE_FEEDS:
        e, hn, kws = engine(r)
        if cur is not None:                     # the re-plan that carries every chain's state into the new engine
            omap = (C.c_int32 * len(hn))(*hs)
            sdb._check(L.sdb_engine_migrate_map(e._h, cur._h, omap, len(hn)))
            keep.append(cur)
        cur, hs = e, hn
        if cfgs is None:
            cfgs = [oracle.insp_config("psk", fs_ch, clock_running=1, **kw) for fs_ch, kw in kws]
        cur.feed(x[None, off:off + m * N_PSD])
        off += m * N_PSD
        for i, h in enumerate(hs):
            chan[i].append(cur.read_channel(0, h))
            got[i].append(cur.read_symbols(0, h))
    for eng in keep + [cur]:
        eng.close()
    for i, cfg in enumerate(cfgs):
        ref = oracle_per_feed(oracle, cfg, chan[i])
        for f, (_, r) in enumerate(TOGGLE_FEEDS):
            soft, hard = got[i][f]
            if not r:
                assert len(soft) == 0, (i, f)
                assert len(ref[f][0]) > 20, (i, f)      # the always-running chain did emit here
            else:
                assert len(ref[f][0]) > 20 and _equal(soft, hard, *ref[f]), (i, f)
