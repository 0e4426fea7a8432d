"""Exact binary32 statement of the inspector's SNR meter, oracle/SPEC_SN.md (SN.1 - SN.4) and the SPEC Y.7 step it
runs.  TEST INFRASTRUCTURE ONLY.

Written from the SPEC text alone, independently of oracle/ and of the CUDA kernels: numpy binary32 element-wise
operations in SPEC's order, the Y.7 gradient sum in bin order, SPEC M's atan2, |x| and exp from chain_stmt.

`mistake` plants one deliberate error, so that the tests can show the comparison would catch it:
    "ask_clamp"         ask values at or above 1 counted in the last bin instead of dropped
    "step_on_empty"     a feed without symbols still runs a Y.7 step
    "bin_scaled"        the bin written as floor((v - min) L / (max - min))
    "keep_h_on_change"  a re-plan with another inspector configuration keeps h
"""
import numpy as np

from chain_stmt import PI_F, atan2, cabs, exp10

F = np.float32
MISTAKES = ("ask_clamp", "step_on_empty", "bin_scaled", "keep_h_on_change")
CLASSES = {"psk": 0, "fsk": 1, "ask": 2}
LIMIT = 1 << 31


def bins(x, mode, L, mistake=None):
    """SN.1: the bin of every symbol of x (complex64), -1 where it is not counted.  mode 0 argument, 1 modulus."""
    x = np.asarray(x, np.complex64)
    re, im = x.real.astype(F), x.imag.astype(F)
    if mode == 0:
        v, mn, h = atan2(im, re), -PI_F, F(PI_F - (-PI_F))
    else:
        v, mn, h = cabs(re, im), F(0.0), F(F(1.0) - F(0.0))
    fL = F(L)
    with np.errstate(invalid="ignore", over="ignore"):
        s = np.floor((v - mn) * fL / h) if mistake == "bin_scaled" else np.floor((v - mn) / h * fL)
        s = s.astype(F)
        out = np.full(len(x), -1, np.int64)
        ok = ~np.isnan(s)
        if mode == 0 or mistake == "ask_clamp":
            out[ok] = np.minimum(s[ok], fL - 1).astype(np.int64)
        else:
            keep = ok & (s < fL)
            out[keep] = s[keep].astype(np.int64)
    return out


def y7_step(h, sigma, alpha, K):
    """SPEC Y.7 on the histogram h[L] -> (model H, new sigma, delta)"""
    L = len(h)
    hmax = max(int(h.max()), 1)
    Ht = (h.astype(F) / F(hmax)).astype(F)
    hx = F(F(1.0) / F(L))
    x = (np.arange(L).astype(F) * hx).astype(F)
    x = np.where(x >= F(0.5), x - F(1.0), x).astype(F)
    sigma, alpha = F(sigma), F(alpha)
    sigma2 = F(sigma * sigma)
    g = exp10((-x * x / sigma2) * F(0.4342944819032518))
    intlen = F(F(1.0) / F(K))
    start = F(F(0.5) * intlen)
    skips = [F(start + F(j) * intlen) for j in range(K)]
    i = np.arange(L)
    H = np.zeros(L, F)
    for skip in skips:
        t = F(F(1.0) - F(skip - np.floor(skip)))
        s = int(np.floor(F(F(L) * skip)))
        i1 = (L + i - s) % L
        i2 = (L + i1 - 1) % L
        H = (H + t * g[i1]).astype(F)
        H = (H + F(F(1.0) - t) * g[i2]).astype(F)
    m = H.max()
    if m > 0:
        H = (H / m).astype(F)
    tm = np.zeros(L, F)
    for skip in skips:
        d = (x - skip).astype(F)
        tm = (tm + d * d).astype(F)
    sigmainv = F(F(1.0) / sigma)
    sigma3inv = F(F(sigmainv * sigmainv) * sigmainv)
    T = (tm * ((H - Ht) / sigma3inv)).astype(F)
    delta = F(0.0)
    for v in T:                                  # in bin order
        delta = F(delta + v)
    delta = F(delta / F(L))
    return H, F(sigma + F(-alpha * delta)), delta


def comb_k(bps):
    """SN.2: K = 2^bps, bps 0 read as 1"""
    return 1 << (bps if bps else 1)


class Meter:
    """SN.3: the meter of one (chain, stream), switched on with (sigma, alpha)"""

    def __init__(self, cls, L, bps, sigma, alpha, mistake=None):
        self.mode = 1 if cls == "ask" else 0
        self.L, self.bps, self.K, self.alpha, self.mistake = L, bps, comb_k(bps), F(alpha), mistake
        self._fresh(F(sigma))

    def _fresh(self, sigma):
        self.h = np.zeros(self.L, np.int64)
        self.model = np.zeros(self.L, F)
        self.sigma, self.delta, self.steps, self.stepped = F(sigma), F(0.0), 0, 0

    @property
    def snr(self):
        """SN.5: 1 / (K sigma)"""
        return F(F(1.0) / F(F(self.K) * self.sigma))

    @property
    def counted(self):
        return int(self.h.sum())

    def feed(self, x):
        """SN.2: one feed's soft symbols"""
        if len(x) == 0 and self.mistake != "step_on_empty":
            self.stepped = 0
            return
        b = bins(x, self.mode, self.L, self.mistake)
        self.h += np.bincount(b[b >= 0], minlength=self.L)
        if (self.h >= LIMIT).any():
            self.h >>= 1
        self.model, self.sigma, self.delta = y7_step(self.h.astype(np.uint32), self.sigma, self.alpha, self.K)
        self.steps += 1
        self.stepped = 1

    def reset(self, sigma):
        """SN.3: sigma only, h kept"""
        self.sigma = F(sigma)

    def replan(self, same_cfg, bps, alpha):
        """SN.4 for a surviving inspector with the same class and L"""
        self.alpha = F(alpha)
        if same_cfg:
            return
        sigma = F(1.0 / 8.0) if bps != self.bps else self.sigma
        self.bps, self.K = bps, comb_k(bps)
        h = self.h
        self._fresh(sigma)
        if self.mistake == "keep_h_on_change":
            self.h = h
