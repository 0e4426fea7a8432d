"""SPEC FC.1 (oracle/SPEC_FC.md) stated in binary64: v[l] = |sum_n x[n] conj(x[n - l])| over the cyclic block, the
unnormalised autocorrelation the FAC tab computes, with a bound on what a binary32 SPEC transform may differ by, and
the margins of the decisions v feeds.  TEST INFRASTRUCTURE ONLY."""
import numpy as np

EPS32 = 2.0 ** -24


def v64(block):
    """|inverse(|F(x)|^2)|[l] for l < L / 2, unnormalised, in binary64"""
    x = np.asarray(block, np.complex128)
    X = np.fft.fft(x)
    return np.abs(np.fft.ifft(np.abs(X) ** 2) * len(x))[:len(x) // 2]


def bound(block):
    """|v32 - v64| <= bound: two binary32 transforms of log2 L stages each (plus the power and the magnitude) perturb
    A by at most a few ulps per stage of its largest value A[0] = L sum |x|^2"""
    x = np.asarray(block, np.complex128)
    L = len(x)
    a0 = L * np.sum(np.abs(x) ** 2)
    return 8.0 * np.log2(L) * EPS32 * a0


def decisions(v, lo, hi, b):
    """(pos, pos_margin): the first arg-max of v over [lo, hi) and how far every other value lies below it; the
    decision is fixed by v64 wherever the margin exceeds 2 b"""
    w = v[lo:hi]
    i = int(np.argmax(w))
    rest = np.delete(w, i)
    return lo + i, (w[i] - rest.max()) if rest.size else np.inf


def records(v, lo, hi):
    """the excluded-record set of one block fed alone: lags whose value exceeds every earlier one of the window, and
    each decision's margin (distance of v to the running maximum it is compared with)"""
    w = v[lo:hi]
    prev = np.maximum.accumulate(np.concatenate([[-np.inf], w]))[:-1]
    return w > prev, np.abs(w - prev)
