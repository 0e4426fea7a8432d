"""Inputs and configurations for the inspector-chain tests (tests/test_chain_stmt.py on the CPU, tests/test_gpu_chains.py
on the GPU).  TEST INFRASTRUCTURE ONLY.

Every case is (name, class, fs, config keywords, n): the chain runs over a batch of inputs of n samples.  The inputs
are noise, a capture of the class's own modulation from `synth`, all zeros, and a 30 dB step (loud, then 30 dB down,
then loud again) that makes the AGC's slow level hold for hang_max samples and then fall."""
import numpy as np

from sigdigger_b200 import synth

# symbol periods T = fs / baud at the edges of the kernel's plan-dependent paths (see test_gpu_chains.PATHS)
T_LADDER = (1.0, 2.5, 3.125, 4.09, 4.10, 13.8, 13.9, 34.8, 34.9, 171.0, 1100.0)


def inputs(cls, T, n, seed=0):
    """[4, n] complex64: noise, a capture of the class at T samples per symbol, zeros, a 30 dB step"""
    rng = np.random.default_rng(seed)
    sps = max(float(T), 1.0)
    if cls == "fsk":
        s, _ = synth.fsk_signal(n, sps, h=1.0, seed=seed + 2)
        cap = 0.3 * s
    elif cls == "ask":
        s, _ = synth.ask_signal(n, sps, levels=4, seed=seed + 3)
        cap = 0.4 * synth.mix(s, 1e-4, 0.5)
    else:
        s, _ = synth.psk_signal(n, sps, order=8 if cls == "psk8" else 4, seed=seed + 1)
        cap = 0.2 * synth.mix(s, 2e-4, 0.3)
    cap = cap + synth.awgn(n, 1e-2, rng)
    noise = synth.awgn(n, 0.3, rng)
    step = synth.awgn(n, 1.0, rng)
    step[n // 3:2 * n // 3] *= 10 ** (-30 / 20)
    return np.stack([noise, cap, np.zeros(n), step]).astype(np.complex64)


def audio_inputs(fs, n, demod, seed=0):
    """[4, n] complex64: noise, an AM / FM / SSB tone, zeros, a 30 dB step"""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / fs
    tone = np.cos(2 * np.pi * 0.01 * fs * t)
    if demod == "am":
        s = (1 + 0.5 * tone) * np.exp(1j * 0.4)
    elif demod == "fm":
        s = np.exp(1j * 2 * np.pi * 0.02 * fs * np.cumsum(tone) / fs)
    else:
        sg = 1 if demod == "usb" else -1
        s = np.exp(2j * np.pi * sg * 0.004 * fs * t) + 0.5 * np.exp(2j * np.pi * sg * 0.011 * fs * t)
    step = synth.awgn(n, 1.0, rng)
    step[n // 3:2 * n // 3] *= 10 ** (-30 / 20)
    return np.stack([synth.awgn(n, 0.1, rng), 0.2 * s + synth.awgn(n, 1e-3, rng), np.zeros(n), step]) \
        .astype(np.complex64)


def _psk(T, **kw):
    base = dict(baud=1.0 / T, costas_order=2, bits_per_symbol=2, loop_bw=2e-3, mf_type=1, clock_type=1,
                clock_gain=0.1)
    base.update(kw)
    return base


def _n(T, short=3000):
    """long enough for a few dozen symbols, short enough for the statement"""
    return int(min(max(short, 40 * T), 7000))


def cases():
    out = []
    # psk: the three Costas kinds, manual offset, MF on / off, Gardner / manual, CMA unlocked / locked, AGC on / off,
    # clock.running 0 / 1
    out.append(("psk_bpsk_T4", "psk", 1.0, _psk(4.0, costas_order=1, bits_per_symbol=1), 3000))
    out.append(("psk_qpsk_T4", "psk", 1.0, _psk(4.0), 3000))
    out.append(("psk_8psk_T5", "psk8", 1.0, _psk(5.0, costas_order=3, bits_per_symbol=3), 3000))
    out.append(("psk_offset_manual_T4.5", "psk", 1.0, _psk(4.5, costas_order=0, offset=1e-3, clock_type=0,
                                                          clock_phase=0.3), 3000))
    out.append(("psk_nomf_agcoff_T3.3", "psk", 1.0, _psk(3.3, mf_type=0, agc_enabled=0, agc_gain_db=6.0), 3000))
    out.append(("psk_cma_T4", "psk", 1.0, _psk(4.0, eq_type=1, eq_rate=2e-2), 3000))
    out.append(("psk_cma_locked_T4", "psk", 1.0, _psk(4.0, eq_type=1, eq_rate=2e-2, eq_locked=1), 3000))
    # a run with clock.running = 0 throughout emits nothing; that the clock and the CMA keep running under it is
    # observable only when the flag changes on a live chain (test_gpu_chains.test_engine_clock_running_toggle)
    out.append(("psk_not_running_T4", "psk", 1.0, _psk(4.0, clock_running=0, eq_type=1), 2000))
    # fsk: quad-demod 0 / 1
    out.append(("fsk_rot_T5", "fsk", 1.0, dict(baud=0.2, bits_per_symbol=1, fsk_phase=0.2, mf_type=1, clock_type=1,
                                               clock_gain=0.2), 3000))
    out.append(("fsk_quad_T5", "fsk", 1.0, dict(baud=0.2, bits_per_symbol=1, fsk_quad_demod=1, mf_type=1, clock_type=1,
                                                clock_gain=0.2), 3000))
    # ask: PLL on / off, channel 0 / 1 / 2
    for pll, ch in ((0, 0), (1, 0), (1, 1), (1, 2), (0, 2)):
        out.append(("ask_pll%d_ch%d_T6.25" % (pll, ch), "ask", 1.0,
                    dict(baud=0.16, bits_per_symbol=2, ask_use_pll=pll, ask_channel=ch, loop_bw=5e-3, offset=1e-4,
                         mf_type=1, clock_type=1, clock_gain=0.2), 3000))
    # ask without AGC at a manual gain that carries |x| past 1, where the decider's clamp acts
    out.append(("ask_agcoff_gain12_T6.25", "ask", 1.0,
                dict(baud=0.16, bits_per_symbol=2, agc_enabled=0, agc_gain_db=12.0, ask_channel=0, offset=1e-4,
                     mf_type=1, clock_type=1, clock_gain=0.2), 3000))
    # raw
    out.append(("raw", "raw", 1.0, dict(), 1000))
    # the T ladder: psk with AGC, Costas, MF and Gardner.  At T = 1100 the AGC delay line holds 4096 samples, so the
    # input is several times that long: the capped line, the 1024-tap filter and Gardner all carry signal.
    for T in T_LADDER:
        n = 12000 if T > 1000 else _n(T)
        out.append(("ladder_T%g" % T, "psk", 1.0, _psk(T), n))
    # baud above the channel rate: bnor = baud / fs clamps to 1
    out.append(("psk_baud_above_fs", "psk", 1.0, _psk(1.0, baud=1.3), 3000))
    return out


def audio_cases():
    """audio: AM / FM / USB / LSB, squelch on / off; one case asks for an audio rate above the channel rate.  The
    resampler emits at most one sample per channel sample, so there its phase grows without bound, al clamps to 1
    and the output is volume * the previous filter output at the channel rate: the rate cannot be raised."""
    out = []
    for demod, sq in (("am", 1), ("fm", 0), ("usb", 1), ("lsb", 0)):
        out.append(("audio_%s_sq%d" % (demod, sq), "audio", 200000.0,
                    dict(audio_demod={"am": 1, "fm": 2, "usb": 3, "lsb": 4}[demod], audio_cutoff=5000.0,
                         audio_sample_rate=44100, agc_ts=0.001, offset=1500.0, audio_squelch=sq,
                         audio_squelch_level=1e-3), 3000))
    out.append(("audio_fm_rate_above_fs", "audio", 8000.0,
                dict(audio_demod=2, audio_cutoff=3000.0, audio_sample_rate=44100, agc_ts=0.01, audio_squelch=0), 1500))
    return out


def case_inputs(cls, fs, kw, n, seed=0):
    if cls == "audio":
        demod = {1: "am", 2: "fm", 3: "usb", 4: "lsb"}[kw["audio_demod"]]
        return audio_inputs(fs, n, demod, seed)
    return inputs(cls, fs / kw.get("baud", 0.25) if cls != "raw" else 4.0, n, seed)


def insp_class(cls):
    return "psk" if cls == "psk8" else cls
