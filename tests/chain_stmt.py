"""Exact binary32 statement of the inspector chains, SPEC.md sections M, I, N, A, C, G, E, D and X.  TEST INFRASTRUCTURE
ONLY.

Written from the SPEC text alone, independently of oracle/ and of the CUDA kernels.  The chains hold discontinuous
recurrences (the AGC hang reset, Gardner's phi >= 0.5, the decider's interval edges), so a tolerance cannot follow a
run past its first such event; the statement is therefore exact: numpy binary32 element-wise operations in SPEC's
stated order, binary64 only where SPEC says "binary64, rounded once" (the tap and loop designs, evaluated with the
platform libm through `math`).

Structure: feed-forward stages work on whole [B, n] arrays (the matched filter loops over taps, not samples); the
recurrences (AGC levels, NCQO, Costas, PLL, Gardner, sampler, CMA, audio IIR and resampler) loop over samples in
lockstep over a batch of B chains that share one configuration.

A binary32 fused multiply-add (SPEC I.1) is `fma32`: the product is exact in binary64, the sum is formed with TwoSum,
rounded to odd in binary64 and then rounded once to binary32, which gives the correctly rounded result.

`mistake` plants one deliberate error, so that the tests can show the comparison would catch it:
    "gardner_gt"     Gardner samples on phi > 0.5 instead of phi >= 0.5
    "hang_gt"        the AGC slow level falls once hang > hang_max instead of hang >= hang_max
    "8psk_larger"    the 8PSK Costas error weights the larger component by sqrt(2) - 1
    "pll_phase_pre"  the PLL error against the NCO phase before read() advanced it
    "mf_rounded"     the matched filter with a rounded product and a rounded add instead of fma
    "cma_unshifted"  the CMA gradient against the line before this symbol was shifted in
    "no_clamp"       the decider without its clamp to [0, 2^bps - 1]
    "rs_no_clamp"    the audio resampler without the al <= 1 clamp
"""
import math

import numpy as np

F = np.float32
MISTAKES = ("gardner_gt", "hang_gt", "8psk_larger", "pll_phase_pre", "mf_rounded", "cma_unshifted", "no_clamp",
            "rs_no_clamp")

PI_F = F(3.14159265358979323846)
TWO_PI_F = F(6.28318530717958647692)
INSP = {"psk": 0, "fsk": 1, "ask": 2, "audio": 3, "raw": 4}
AUDIO = {"am": 1, "fm": 2, "usb": 3, "lsb": 4}
AGC_MAX_LINE = 4096
MF_MAX_SPAN = 1024
EQ_LEN = 10


# ---- binary32 fused multiply-add ------------------------------------------------------------------------------------
def fma32(a, b, c):
    """round32(a * b + c) with a single rounding, element-wise"""
    a, b, c = (np.asarray(v, np.float32).astype(np.float64) for v in (a, b, c))
    p = a * b                                   # exact: 24 + 24 bits
    s = p + c
    bp = s - c
    err = (p - bp) + (c - (s - bp))             # TwoSum: p + c = s + err exactly
    bits = np.atleast_1d(s).view(np.int64).copy()
    e = np.atleast_1d(err)
    inexact = e != 0
    toward_zero = inexact & ((e < 0) != (np.atleast_1d(s) < 0))
    bits[toward_zero] -= 1                      # truncate toward zero ...
    bits[inexact] |= 1                          # ... and make it odd
    r = bits.view(np.float64).astype(np.float32)
    return r.reshape(np.shape(s)) if np.ndim(s) else r[0]


# ---- M: elementary functions ----------------------------------------------------------------------------------------
def sincos(x):
    """M.1 -> (sin, cos)"""
    x = np.asarray(x, np.float32)
    q = np.rint(x * F(0.636619772367581343))
    r = x - q * F(1.5703125)
    r = r - q * F(4.837512969970703125e-4)
    r = r - q * F(7.54978995489188e-8)
    z = r * r
    sp = ((F(-1.9515295891e-4) * z + F(8.3321608736e-3)) * z - F(1.6666654611e-1)) * z * r + r
    cp = ((F(2.443315711809948e-5) * z - F(1.388731625493765e-3)) * z + F(4.166664568298827e-2)) * z * z \
        - F(0.5) * z + F(1.0)
    with np.errstate(invalid="ignore"):
        n = q.astype(np.int32) & 3
    s = np.select([n == 0, n == 1, n == 2], [sp, cp, -sp], -cp).astype(np.float32)
    c = np.select([n == 0, n == 1, n == 2], [cp, -sp, -cp], sp).astype(np.float32)
    return s, c


def _atan_pos(t):
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        big = t > F(2.414213562373095)
        mid = ~big & (t > F(0.4142135623730950))
        y0 = np.where(big, F(1.5707963267948966), np.where(mid, F(0.7853981633974483), F(0.0))).astype(np.float32)
        t = np.where(big, F(-1.0) / t, np.where(mid, (t - F(1.0)) / (t + F(1.0)), t)).astype(np.float32)
        z = t * t
        y = (((F(8.05374449538e-2) * z - F(1.38776856032e-1)) * z + F(1.99777106478e-1)) * z
             - F(3.33329491539e-1)) * z * t + t
    return y0 + y


def atan2(y, x):
    """M.2"""
    y, x = np.asarray(y, np.float32), np.asarray(x, np.float32)
    ax, ay = np.abs(x), np.abs(y)
    with np.errstate(divide="ignore", invalid="ignore"):
        a = np.where(ax == F(0), F(1.5707963267948966), _atan_pos(ay / ax)).astype(np.float32)
    a = np.where(x < F(0), PI_F - a, a)
    a = np.where(y < F(0), -a, a)
    return np.where((ax == F(0)) & (ay == F(0)), F(0), a).astype(np.float32)


LOG_POLY = (7.0376836292e-2, -1.1514610310e-1, 1.1676998740e-1, -1.2420140846e-1, 1.4249322787e-1,
            -1.6668057665e-1, 2.0000714765e-1, -2.4999993993e-1, 3.3333331174e-1)
EXP10_POLY = (2.063216740311022e-1, 5.420251702225484e-1, 1.171292686296281, 2.034649854009453, 2.650948748208892,
              2.302585167056758)


def log10(x):
    """M.3, x > 0"""
    x = np.asarray(x, np.float32)
    sub = x < F(1.17549435e-38)
    with np.errstate(over="ignore"):
        x = np.where(sub, x * F(8388608.0), x).astype(np.float32)
    ix = x.view(np.uint32)
    e = np.where(sub, -23, 0) + (ix >> 23).astype(np.int64) - 127
    m = ((ix & np.uint32(0x007FFFFF)) | np.uint32(0x3F800000)).view(np.float32)
    big = m > F(1.41421356)
    m = np.where(big, m * F(0.5), m).astype(np.float32)
    e = e + big
    f = m - F(1.0)
    z = f * f
    y = F(LOG_POLY[0]) * f
    for c in LOG_POLY[1:]:
        y = y + F(c)
        y = y * f
    y = y * z
    y = y - F(0.5) * z
    L = F(4.3429448190325176e-1)
    r = y * L
    r = r + f * L
    return (r + e.astype(np.float32) * F(3.0102999566398120e-1)).astype(np.float32)


def exp10(x):
    """M.4"""
    x = np.asarray(x, np.float32)
    x = np.where(x > F(38.0), F(38.0), x)
    x = np.where(x < F(-37.0), F(-37.0), x).astype(np.float32)
    px = np.floor(F(3.32192809488736234787) * x + F(0.5))
    n = px.astype(np.int32)
    x = x - px * F(3.00781250000000000000e-1)
    x = x - px * F(2.48745663981195213739e-4)
    p = F(EXP10_POLY[0]) * x
    for c in EXP10_POLY[1:-1]:
        p = (p + F(c)) * x
    p = p + F(EXP10_POLY[-1])
    p = p * x + F(1.0)
    sc = ((n + 127).astype(np.uint32) << np.uint32(23)).view(np.float32)
    return (p * sc).astype(np.float32)


def cabs(re, im):
    """M.5"""
    return np.sqrt(re * re + im * im)


def db_to_mag(d):
    return exp10(np.asarray(d, np.float32) * F(0.05))


# ---- I: tap and loop designs (binary64, rounded once) ---------------------------------------------------------------
def mf_span(T):
    """I.2: ceil(6 T) in binary64, clamped to [1, 1024]"""
    return int(min(max(math.ceil(6.0 * float(F(T))), 1.0), float(MF_MAX_SPAN)))


def hamming(i, n):
    return 0.54 - 0.46 * math.cos(2.0 * math.pi * i / (n - 1)) if n > 1 else 1.0


def taps_rrc(n, T, beta):
    """I.2"""
    b, Td = float(F(beta)), float(F(T))
    h = np.empty(n, np.float32)
    for i in range(n):
        t = (i - n / 2.0) / Td
        f = 4.0 * b * t
        dem = math.pi * t * (1.0 - f * f)
        if abs(t) < 1e-9:
            v = 1.0 - b + 4.0 * b / math.pi
        elif abs(dem) < 1e-9:
            v = b / math.sqrt(2.0) * ((1.0 + 2.0 / math.pi) * math.sin(math.pi / (4.0 * b))
                                      + (1.0 - 2.0 / math.pi) * math.cos(math.pi / (4.0 * b)))
        else:
            v = (math.sin(math.pi * t * (1.0 - b)) + 4.0 * b * t * math.cos(math.pi * t * (1.0 + b))) / dem
        v /= Td
        v *= hamming(i, n)
        h[i] = v
    return h


def butter_lp(order, fc):
    """I.4 -> (b, a), order + 1 coefficients each, descending powers of z"""
    fc = float(F(fc))
    warped = 4.0 * math.tan(math.pi * fc / 2.0)
    poles, kden = [], complex(1.0, 0.0)
    for k in range(order):
        th = math.pi * (2.0 * k + order + 1.0) / (2.0 * order)
        s = warped * complex(math.cos(th), math.sin(th))
        poles.append((4.0 + s) / (4.0 - s))
        kden *= (4.0 - s)
    gain = math.pow(warped, order) * (1.0 / kden).real
    pa = [complex(1.0, 0.0)] + [complex(0.0, 0.0)] * order
    pb = [1.0] + [0.0] * order
    for k in range(order):
        for j in range(k + 1, 0, -1):
            pa[j] = pa[j] - poles[k] * pa[j - 1]
            pb[j] = pb[j] + pb[j - 1]
    return (np.array([gain * v for v in pb], np.float32), np.array([v.real for v in pa], np.float32))


def alpha_of(t):
    """A: (float)(1 - exp(-1/t)) in binary64"""
    return F(1.0 - math.exp(-1.0 / float(F(t))))


class AgcDesign:
    """A: the derived sizes and time constants from the symbol period tau, all binary32 in SPEC's order"""

    def __init__(self, tau, s=1.0):
        tau, rise = F(tau), F(s) * F(3.9062e-1)
        self.fast_rise_t = tau * rise
        self.fast_fall_t = tau * (F(2.0) * rise)
        self.slow_rise_t = tau * (F(10.0) * rise)
        self.slow_fall_t = tau * (F(10.0) * (F(2.0) * rise))
        self.hang_max = int(tau * (rise * F(5.0)))
        line = int(tau * (rise * F(10.0)))
        self.dl_size = self.mh_size = min(max(line, 1), AGC_MAX_LINE)
        self.knee = F(-100.0)
        self.gain_slope = F(6.0) * F(1e-2)
        self.fixed_gain = db_to_mag(self.knee * (self.gain_slope - F(1.0)))
        self.far, self.faf = alpha_of(self.fast_rise_t), alpha_of(self.fast_fall_t)
        self.sar, self.saf = alpha_of(self.slow_rise_t), alpha_of(self.slow_fall_t)


def pll_design(fc):
    """C: (alpha, beta) of a PLL at normalised bandwidth fc"""
    fc = PI_F * F(fc)
    dinv = F(1.0) / (F(1.0) + F(2.0) * F(0.707) * fc + fc * fc)
    return F(4.0) * fc * fc * dinv, F(4.0) * F(0.707) * fc * dinv


def costas_design(loop_bw):
    """C: (a, b) of a Costas loop"""
    a = PI_F * F(loop_bw)
    return a, F(0.5) * a * a


# ---- stages ---------------------------------------------------------------------------------------------------------
def wrap(phi):
    """N: one subtraction of 2 pi when >= 2 pi, one addition when < 0"""
    return np.where(phi >= TWO_PI_F, phi - TWO_PI_F, np.where(phi < F(0), phi + TWO_PI_F, phi)).astype(np.float32)


def ncqo_phases(B, n, omega):
    """N: the phases read() sees at each of n samples, starting from 0, for a constant omega"""
    ph = np.empty((B, n), np.float32)
    phi = np.zeros(B, np.float32)
    for t in range(n):
        ph[:, t] = phi
        phi = wrap(phi + omega)
    return ph


def mix_conj(xr, xi, cr, ci):
    """x * conj(c)"""
    return xr * cr + xi * ci, xi * cr - xr * ci


def discriminator(xr, xi):
    """X: d = y conj(prev) over [B, n], prev starting at 0 (fsk and the FM demodulator)"""
    B = xr.shape[0]
    pr = np.concatenate([np.zeros((B, 1), np.float32), xr[:, :-1]], axis=1)
    pi = np.concatenate([np.zeros((B, 1), np.float32), xi[:, :-1]], axis=1)
    return mix_conj(xr, xi, pr, pi)


def agc(xr, xi, d, mistake=None):
    """A over [B, n]: the delay line, magnitudes and history rescans are feed-forward; the levels loop"""
    B, n = xr.shape
    L, M = d.dl_size, d.mh_size
    m = F(10.0) * log10(xr * xr + xi * xi + F(1e-16))
    mp = np.concatenate([np.full((B, M), F(-160.0)), m], axis=1)
    m_old = mp[:, :n]                                       # the history entry each sample replaces
    wmax = np.maximum(F(-160.0), np.lib.stride_tricks.sliding_window_view(mp, M, axis=1)[:, 1:n + 1].max(axis=-1))
    peak = np.full(B, F(-160.0))
    fast, slow = peak.copy(), peak.copy()
    hang = np.zeros(B, np.int64)
    lvl = np.empty((B, n), np.float32)
    hm = d.hang_max + (1 if mistake == "hang_gt" else 0)
    for t in range(n):
        mt = m[:, t]
        peak = np.where(mt > peak, mt, np.where(peak == m_old[:, t], wmax[:, t], peak))
        dd = peak - fast
        fast = fast + np.where(dd > F(0), d.far, d.faf) * dd
        dd = peak - slow
        rise = dd > F(0)
        fall = ~rise & (hang >= hm)
        slow = np.where(rise, slow + d.sar * dd, np.where(fall, slow + d.saf * dd, slow))
        hang = np.where(rise, 0, np.where(fall, hang, hang + 1))
        lvl[:, t] = np.where(fast > slow, fast, slow)
    g = np.where(lvl < d.knee, d.fixed_gain, db_to_mag(lvl * (d.gain_slope - F(1.0)))) * F(0.7)
    pad = np.zeros((B, L), np.float32)
    xdr = np.concatenate([pad, xr], axis=1)[:, :n]
    xdi = np.concatenate([pad, xi], axis=1)[:, :n]
    return xdr * g, xdi * g


class Iir:
    """I.1 on a [2, B] complex state (re, im stacked), every term one fma"""

    def __init__(self, b, a, B):
        self.b, self.na = np.asarray(b, np.float32), len(a)
        self.na_coef = -np.asarray(a, np.float32)
        self.x = [np.zeros((2, B), np.float32) for _ in self.b]
        self.y = [np.zeros((2, B), np.float32) for _ in range(max(self.na - 1, 0))]

    def feed(self, v):
        self.x = [v] + self.x[:-1]
        acc = np.zeros_like(v)
        for bi, xv in zip(self.b, self.x):
            acc = fma32(bi, xv, acc)
        for ai, yv in zip(self.na_coef[1:], self.y):
            acc = fma32(ai, yv, acc)
        if self.na > 1:
            self.y = [acc] + self.y[:-1]
        return acc


def fir(xr, xi, h, mistake=None):
    """I.1 feed-forward over [B, n]: taps in ascending order, one fma each, the line starts at zero"""
    B, n = xr.shape
    ar, ai = np.zeros((B, n), np.float32), np.zeros((B, n), np.float32)
    for i, hi in enumerate(np.asarray(h, np.float32)):
        if i >= n:
            break
        sr, si = np.zeros((B, n), np.float32), np.zeros((B, n), np.float32)
        sr[:, i:], si[:, i:] = xr[:, :n - i], xi[:, :n - i]
        if mistake == "mf_rounded":
            ar, ai = ar + hi * sr, ai + hi * si
        else:
            ar, ai = fma32(hi, sr, ar), fma32(hi, si, ai)
    return ar, ai


def costas(xr, xi, kind, a, b, af_b, af_a, mistake=None):
    """C: Costas loop over [B, n], fhint 0, gain 1, y_alpha 1"""
    B, n = xr.shape
    phi, om = np.zeros(B, np.float32), np.zeros(B, np.float32)
    af = Iir(af_b, af_a, B)
    yr, yi = np.zeros(B, np.float32), np.zeros(B, np.float32)
    outr, outi = np.empty((B, n), np.float32), np.empty((B, n), np.float32)
    k8 = F(0.41421356237309504)
    for t in range(n):
        s, c = sincos(phi)
        phi = wrap(phi + om)
        z = af.feed(np.stack(mix_conj(xr[:, t], xi[:, t], c, s)))
        zr, zi = z[0], z[1]
        if kind == 1:
            e = -(zr * zi)
        else:
            lr, li = np.sign(zr).astype(np.float32), np.sign(zi).astype(np.float32)
            if kind == 2:
                e = lr * zi - li * zr
            else:
                ge = np.abs(zr) >= np.abs(zi)
                if mistake == "8psk_larger":
                    ge = ~ge
                e = np.where(ge, lr * zi - li * zr * k8, lr * zi * k8 - li * zr)
        yr = yr + F(1.0) * (zr - yr)
        yi = yi + F(1.0) * (zi - yi)
        om = om + b * e
        phi = wrap(phi + a * e)
        outr[:, t], outi[:, t] = yr, yi
    return outr, outi


def pll(xr, xi, alpha, beta, mistake=None):
    """C: PLL over [B, n], fhint 0; the error uses the NCO phase after read() advanced it"""
    B, n = xr.shape
    ang = atan2(xi, xr)
    phi, om = np.zeros(B, np.float32), np.zeros(B, np.float32)
    outr, outi = np.empty((B, n), np.float32), np.empty((B, n), np.float32)
    for t in range(n):
        s, c = sincos(phi)
        pre = phi
        phi = wrap(phi + om)
        outr[:, t], outi[:, t] = mix_conj(xr[:, t], xi[:, t], c, s)
        e = ang[:, t] - (pre if mistake == "pll_phase_pre" else phi)
        e = np.where(e > PI_F, e - TWO_PI_F, np.where(e < -PI_F, e + TWO_PI_F, e)).astype(np.float32)
        om = om + alpha * e
        phi = wrap(phi + beta * e)
    return outr, outi


def gardner(xr, xi, bnor, gain, mistake=None):
    """G: Gardner clock recovery over [B, n] -> (sr, si, mask [B, n] of emitted samples)"""
    B, n = xr.shape
    alpha = F(2e-1)
    beta = F(6e-4) * alpha
    gain = F(gain)
    phi, bn = np.full(B, F(0.25)), np.full(B, F(bnor))
    half = np.zeros(B, bool)
    x0r, x0i, x1r, x1i, x2r, x2i, pr, pi = (np.zeros(B, np.float32) for _ in range(8))
    sr, si, emit = np.zeros((B, n), np.float32), np.zeros((B, n), np.float32), np.zeros((B, n), bool)
    for t in range(n):
        vr, vi = xr[:, t], xi[:, t]
        phi = phi + bn
        hit = phi > F(0.5) if mistake == "gardner_gt" else phi >= F(0.5)
        al = bn * (phi - F(0.5))
        om = F(1.0) - al
        p_r, p_i = om * vr + al * pr, om * vi + al * pi
        half = np.where(hit, ~half, half)
        phi = np.where(hit, phi - F(0.5), phi)
        full = hit & ~half
        part = hit & half
        x2r, x2i = np.where(full, x0r, x2r), np.where(full, x0i, x2i)
        x0r, x0i = np.where(full, p_r, x0r), np.where(full, p_i, x0i)
        e = gain * (x1r * (x0r - x2r) + x1i * (x0i - x2i))
        phi = np.where(full, phi + alpha * e, phi)
        b2 = bn + beta * e
        b2 = np.where(b2 > F(1.0), F(1.0), b2)
        b2 = np.where(b2 < F(0.0), F(0.0), b2)
        bn = np.where(full, b2, bn).astype(np.float32)
        x1r, x1i = np.where(part, p_r, x1r), np.where(part, p_i, x1i)
        sr[:, t], si[:, t], emit[:, t] = p_r, p_i, full
        pr, pi = vr, vi
    return sr, si, emit


def sampler(xr, xi, bnor, clock_phase):
    """G: manual sampler over [B, n]; the phase walk is the same for every lane"""
    B, n = xr.shape
    bnor = F(bnor)
    period = F(1.0) / bnor if bnor > F(0) else F(0)
    phase0 = F(clock_phase) * period
    emit = np.zeros(n, bool)
    al = np.zeros(n, np.float32)
    if period >= F(1.0):
        phase = F(0.0)
        for t in range(n):
            phase = phase + F(1.0)
            if phase >= period:
                phase = phase - period
            ph = phase - phase0
            if ph < F(0):
                ph = ph + period
            fl = np.floor(ph)
            if fl == F(0):
                emit[t], al[t] = True, ph - fl
    prr = np.concatenate([np.zeros((B, 1), np.float32), xr[:, :-1]], axis=1)
    pri = np.concatenate([np.zeros((B, 1), np.float32), xi[:, :-1]], axis=1)
    om = F(1.0) - al
    return om * prr + al * xr, om * pri + al * xi, np.broadcast_to(emit, (B, n))


def cma(symbols, mu, locked, mistake=None):
    """E: one list of complex64 symbol arrays per lane -> equalised arrays, lanes in lockstep"""
    B = len(symbols)
    cnt = np.array([len(s) for s in symbols])
    n = int(cnt.max()) if B else 0
    sr, si = np.zeros((B, n), np.float32), np.zeros((B, n), np.float32)
    for b, s in enumerate(symbols):
        sr[b, :len(s)], si[b, :len(s)] = s.real, s.imag
    wr, wi = np.zeros((B, EQ_LEN), np.float32), np.zeros((B, EQ_LEN), np.float32)
    wr[:, 0] = 1.0
    xr, xi = np.zeros((B, EQ_LEN), np.float32), np.zeros((B, EQ_LEN), np.float32)
    outr, outi = np.zeros((B, n), np.float32), np.zeros((B, n), np.float32)
    mu = F(mu)
    for t in range(n):
        live = (t < cnt)[:, None]
        gr_line, gi_line = xr, xi
        xr = np.where(live, np.concatenate([sr[:, t:t + 1], xr[:, :-1]], axis=1), xr)
        xi = np.where(live, np.concatenate([si[:, t:t + 1], xi[:, :-1]], axis=1), xi)
        if mistake != "cma_unshifted":
            gr_line, gi_line = xr, xi
        yr, yi = np.zeros(B, np.float32), np.zeros(B, np.float32)
        tr, ti = wr * xr - wi * xi, wr * xi + wi * xr
        for i in range(EQ_LEN):
            yr, yi = yr + tr[:, i], yi + ti[:, i]
        if not locked:
            y2 = yr * yr + yi * yi
            er, ei = (yr * (y2 - F(1.0)))[:, None], (yi * (y2 - F(1.0)))[:, None]
            gr = gr_line * er + gi_line * ei
            gi = gr_line * ei - gi_line * er
            wr = np.where(live, wr - mu * gr, wr)
            wi = np.where(live, wi - mu * gi, wi)
        outr[:, t], outi[:, t] = yr, yi
    return [(outr[b, :cnt[b]] + 1j * outi[b, :cnt[b]]).astype(np.complex64) for b in range(B)]


def decide(soft, mode, bps, mistake=None):
    """D: mode 0 ARGUMENT on [-pi, pi], 1 MODULUS on [0, 1]"""
    soft = np.asarray(soft, np.complex64)
    re, im = soft.real.copy(), soft.imag.copy()
    if mode == 0:
        v, vmin, vmax = atan2(im, re), -PI_F, PI_F
    else:
        v, vmin, vmax = cabs(re, im), F(0.0), F(1.0)
    q = 1 << bps
    s = np.floor((v - vmin) / (vmax - vmin) * F(q))
    with np.errstate(invalid="ignore"):
        k = np.where(s >= F(0), s, F(0)).astype(np.int64)
    if mistake != "no_clamp":
        k = np.minimum(k, q - 1)
    return k.astype(np.uint8)


# ---- X: the chains --------------------------------------------------------------------------------------------------
def bnor_of(cfg):
    """X: baud / fs in binary32, clamped to 1, 1e-6 when not positive"""
    b = F(cfg["baud"]) / F(cfg["fs"])
    if b > F(1.0):
        b = F(1.0)
    if not b > F(0.0):
        b = F(1e-6)
    return b


def _split(x):
    x = np.asarray(x, np.complex64)
    return np.ascontiguousarray(x.real), np.ascontiguousarray(x.imag)


def _symbol_chain(cfg, xr, xi, mistake):
    B, n = xr.shape
    fs, cls = F(cfg["fs"]), cfg["insp_class"]
    bnor = bnor_of(cfg)
    T = F(1.0) / bnor
    lo = (cls == INSP["psk"] and cfg["costas_order"] == 0) or (cls == INSP["ask"] and not cfg["ask_use_pll"])
    if lo:                                                       # manual offset: x * conj(lo)
        ph = ncqo_phases(B, n, PI_F * (F(2.0) * F(cfg["offset"]) / fs))
        s, c = sincos(ph)
        xr, xi = mix_conj(xr, xi, c, s)
    if cfg["agc_enabled"]:                                       # gain stage
        xr, xi = agc(xr, xi, AgcDesign(T, 1.0), mistake)
        xr, xi = F(2.0) * xr, F(2.0) * xi
    else:
        g = F(2.0) * db_to_mag(F(cfg["agc_gain_db"]))
        xr, xi = g * xr, g * xi
    if cls == INSP["psk"] and cfg["costas_order"] > 0:
        b, a = butter_lp(2, np.clip(F(2.0) * bnor, F(1e-3), F(0.95)))
        ca, cb = costas_design(F(2.0) * F(cfg["loop_bw"]) / fs)
        xr, xi = costas(xr, xi, int(cfg["costas_order"]), ca, cb, b, a, mistake)
    elif cls == INSP["fsk"]:
        dr, di = discriminator(xr, xi)
        if cfg["fsk_quad_demod"]:
            xr, xi = atan2(di, dr) * F(1.0 / math.pi), np.zeros_like(dr)
        else:
            rs, rc = sincos(F(cfg["fsk_phase"]))
            xr, xi = dr * rc - di * rs, dr * rs + di * rc
    elif cls == INSP["ask"]:
        if cfg["ask_use_pll"]:
            xr, xi = pll(xr, xi, *pll_design(F(2.0) * F(cfg["loop_bw"]) / fs), mistake=mistake)
        ch = cfg["ask_channel"]
        xr = cabs(xr, xi) if ch == 0 else (xr if ch == 1 else xi)
        xi = np.zeros_like(xr)
    if cfg["mf_type"] == 1:
        xr, xi = fir(xr, xi, taps_rrc(mf_span(T), T, cfg["mf_rolloff"]), mistake)
    if cfg["clock_type"] == 1:
        sr, si, emit = gardner(xr, xi, bnor, cfg["clock_gain"], mistake)
    else:
        sr, si, emit = sampler(xr, xi, bnor, cfg["clock_phase"])
    syms = [(sr[b][emit[b]] + 1j * si[b][emit[b]]).astype(np.complex64) for b in range(B)]
    if cfg["eq_type"] == 1:                                      # the CMA runs whether or not symbols are emitted
        syms = cma(syms, cfg["eq_rate"], cfg["eq_locked"], mistake)
    if not cfg["clock_running"]:
        return [np.zeros(0, np.complex64) for _ in range(B)]
    return [(F(0.75) * s.real + 1j * (F(0.75) * s.imag)).astype(np.complex64) for s in syms]


def _audio_chain(cfg, xr, xi, mistake):
    B, n = xr.shape
    fs = F(cfg["fs"])
    if cfg["agc_enabled"]:
        tau = F(cfg["agc_ts"]) * fs
        xr, xi = agc(xr, xi, AgcDesign(max(tau, F(2.0)), 1.0), mistake)
    fsd = float(fs)
    dc_alpha = F(1.0 - math.exp(-1.0 / (0.05 * fsd)))
    sq_alpha = F(1.0 - math.exp(-1.0 / (0.01 * fsd)))
    p = xr * xr + xi * xi
    sq = np.empty((B, n), np.float32)
    lev = np.zeros(B, np.float32)
    for t in range(n):                                           # squelch level, a one-pole average of the power
        lev = lev + sq_alpha * (p[:, t] - lev)
        sq[:, t] = lev
    dm = cfg["audio_demod"]
    if dm == AUDIO["am"]:
        v = cabs(xr, xi)
        out = np.empty((B, n), np.float32)
        dc = np.zeros(B, np.float32)
        for t in range(n):
            dc = dc + dc_alpha * (v[:, t] - dc)
            out[:, t] = v[:, t] - dc
        v = out
    elif dm == AUDIO["fm"]:
        dr, di = discriminator(xr, xi)
        v = atan2(di, dr) * F(1.0 / math.pi)
    elif dm in (AUDIO["usb"], AUDIO["lsb"]):
        fo = F(cfg["offset"]) if dm == AUDIO["usb"] else -F(cfg["offset"])
        s, c = sincos(ncqo_phases(B, n, PI_F * (F(2.0) * fo / fs)))
        v = xr * c - xi * s
    else:
        v = np.zeros((B, n), np.float32)
    if cfg["audio_squelch"]:
        v = np.where(sq > F(cfg["audio_squelch_level"]), v, F(0.0)).astype(np.float32)
    b, a = butter_lp(4, np.clip(F(2.0) * F(cfg["audio_cutoff"]) / fs, F(1e-4), F(0.95)))
    f = Iir(b, a, B)
    o = np.empty((B, n), np.float32)
    zero = np.zeros(B, np.float32)
    for t in range(n):
        o[:, t] = f.feed(np.stack([v[:, t], zero]))[0]
    # resampler: phase and step in binary64, the same instants for every lane
    step = float(cfg["audio_sample_rate"]) / fsd
    idx, al = [], []
    ph = 0.0
    for t in range(n):
        ph += step
        if ph >= 1.0:
            ph -= 1.0
            a_ = F(ph / step)
            if a_ > F(1.0) and mistake != "rs_no_clamp":
                a_ = F(1.0)
            idx.append(t)
            al.append(a_)
    idx, al = np.array(idx, np.int64), np.array(al, np.float32)
    prev = np.concatenate([np.zeros((B, 1), np.float32), o[:, :-1]], axis=1)
    vol = F(cfg["audio_volume"])
    r = vol * ((F(1.0) - al) * o[:, idx] + al * prev[:, idx])
    return [(r[b] + 0j).astype(np.complex64) for b in range(B)]


def run(cfg, x, mistake=None):
    """cfg: dict of the inspector configuration (the sdb / oracle field names); x: [B, n] complex64 channel samples
    -> list of (soft complex64, hard uint8) per lane"""
    assert mistake in (None,) + MISTAKES
    x = np.atleast_2d(np.asarray(x, np.complex64))
    cls = cfg["insp_class"]
    if cls == INSP["raw"]:
        soft = [x[b].copy() for b in range(len(x))]
    elif cls == INSP["audio"]:
        soft = _audio_chain(cfg, *_split(x), mistake)
    else:
        soft = _symbol_chain(cfg, *_split(x), mistake)
    mode = 1 if cls == INSP["ask"] else 0
    return [(s, decide(s, mode, int(cfg["bits_per_symbol"]), mistake)) for s in soft]
