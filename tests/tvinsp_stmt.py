"""Statement of SPEC TI.1-TI.3 (oracle/SPEC_TI.md), the Analog TV tab on an inspector, over the exact binary32
statement of SPEC TV (tv_stmt.TvStmt).  TEST INFRASTRUCTURE ONLY.

TI.1 in numpy binary32, one rounding per operation in the order written: k·|x| + dc with |x| = sqrt(re·re + im·im)
for ask, k·arg(x)/π + dc with SPEC M's atan2 (chain_stmt.atan2) for psk and fsk.  TI.3: the first frame a feed
completes, as the ring holds it at that moment, and its number.

`mistake` plants one deliberate error, so that the tests can show the comparison would catch it:
    "post_last"     the feed's last completed frame posted instead of its first
    "psk_modulus"   psk converted with the modulus
"""
import math

import numpy as np

import tv_stmt
from chain_stmt import atan2

F = np.float32
MISTAKES = ("post_last", "psk_modulus")
PI_F = F(math.pi)


def convert(cls, k, dc, x, mistake=None):
    """TI.1 of a feed's soft symbols"""
    x = np.ascontiguousarray(x, np.complex64)
    re, im = x.real.astype(F), x.imag.astype(F)
    if cls == "ask" or (cls == "psk" and mistake == "psk_modulus"):
        return F(k) * np.sqrt(re * re + im * im) + F(dc)
    return F(k) * atan2(im, re) / PI_F + F(dc)


class TabStmt:
    def __init__(self, cls, p, invert=False, dc=0.0, mistake=None):
        assert mistake is None or mistake in MISTAKES
        self.cls, self.mistake = cls, mistake
        self.tv = tv_stmt.TvStmt(p)
        self.k, self.dc = (-1.0 if invert else 1.0), dc
        self.posted = np.zeros((self.tv.H, self.tv.W), F)
        self.posted_no, self.completed = 0, 0

    def set_params(self, p, invert=False, dc=0.0):
        """TI.4: True when taken"""
        if not self.tv.set_params(p):
            return False
        self.k, self.dc = (-1.0 if invert else 1.0), dc
        return True

    def feed(self, x):
        self.completed = 0                                   # TI.2: a feed without symbols changes nothing else
        for v in convert(self.cls, self.k, self.dc, x, self.mistake):
            f0 = self.tv.frames
            self.tv.step(v)
            if self.tv.frames == f0:
                continue
            self.completed += 1
            if self.completed == 1 or self.mistake == "post_last":
                self.posted = self.tv.ring[(self.tv.frames - 1) % tv_stmt.RING].copy()
                self.posted_no = self.tv.frames

    def status_key(self):
        """as tvinsp_oracle.Status.key()"""
        b = lambda v: int(F(v).view(np.uint32))              # noqa: E731
        L, hs, g = self.tv.estimates()
        return (self.tv.frames, self.posted_no, self.completed, self.tv.W, self.tv.H, b(L), b(hs), b(g))
