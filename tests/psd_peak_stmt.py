"""Exact statement of the main PSD's peak detectors, oracle/SPEC_PK.md.  TEST INFRASTRUCTURE ONLY.

Written from the SPEC text alone, independently of the CUDA kernels.  PK has no sums: fmax and fmin return one of
their operands, so numpy binary32 element-wise operations give the same bits as any correct implementation.

    PK.1  per stream, frames numbered across feeds; group g holds frames g P ... g P + P - 1
    PK.2  max = fmax(... fmax(f0, f1) ..., fP-1), min the same with fmin, per bin; NaN operands ignored (maxNum /
          minNum), all-NaN gives NaN; the first frame of the group starts the value
    PK.3  the partial max, min and frame count carry across feeds
    PK.4  outputs [stream][group][N], linear, DC at 0 (the dB layout is applied by the caller, after the extremes)

`mistake` plants one deliberate error, so that the tests can show the comparison would catch it:
    "off_by_one"  groups of P + 1 frames
    "max"         np.maximum / np.minimum (NaN-propagating) instead of np.fmax / np.fmin
"""
import numpy as np

MISTAKES = ("off_by_one", "max")


class Carry:
    """The partial group of PK.3: per-stream running extremes and the frame count they hold."""
    __slots__ = ("mx", "mn", "count")

    def __init__(self):
        self.mx = self.mn = None
        self.count = 0


def group_peaks(psd, P, carry=None, mistake=None):
    """PK.1-PK.3 over one feed's per-frame PSD psd [S, F, N] float32 -> (max [S, groups, N], min [S, groups, N], carry).
    `carry` is the Carry of the previous feed (a new one when None); it is updated in place and returned."""
    assert mistake in (None,) + MISTAKES
    psd = np.asarray(psd, np.float32)
    S, F, N = psd.shape
    carry = Carry() if carry is None else carry
    size = P + 1 if mistake == "off_by_one" else P
    hi, lo = (np.maximum, np.minimum) if mistake == "max" else (np.fmax, np.fmin)
    maxes, mins = [], []
    for f in range(F):
        frame = psd[:, f]
        if carry.count == 0:
            carry.mx, carry.mn = frame.copy(), frame.copy()         # the first frame starts the value
        else:
            carry.mx, carry.mn = hi(carry.mx, frame), lo(carry.mn, frame)
        carry.count += 1
        if carry.count == size:
            maxes.append(carry.mx)
            mins.append(carry.mn)
            carry.mx = carry.mn = None
            carry.count = 0
    stack = lambda xs: np.stack(xs, axis=1).astype(np.float32) if xs else np.zeros((S, 0, N), np.float32)
    return stack(maxes), stack(mins), carry


def same(a, b):
    """bit-identical, except that any NaN equals any NaN (PK.2 says NaN, not which one)"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32)))
