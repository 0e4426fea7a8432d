"""Float64 statement of the inspector spectrum sources and baud estimators, SPEC.md sections U and W.  TEST
INFRASTRUCTURE ONLY.

Written from the SPEC text alone, independently of oracle/ and of the CUDA kernels.  Everything is binary64 /
complex128 after the float32 channel samples are read.

    U.1  a feed of n_ch >= Ns + 1 channel samples c emits x[i] = c[n_ch - Ns + i], x[-1] = c[n_ch - Ns - 1]
    U.2  d = x[i] conj(x[i-1]), delta = x[i] - x[i-1]: psd x; cyclo d; fmspect angle(d) / pi (atan2(0, 0) = 0);
         timediff delta; abstimediff |delta|; exp_2 / exp_4 / exp_8 x^2, x^4, x^8
    U.3  s[k] = |FFT(w o p)[k]|^2 / Ns, w = Blackman-Harris(Ns) with the N - 1 denominator of SPEC W
    U.4  fac[l] = |IFFT_unnormalised(|FFT(x)|^2)[l]| / Ns, l < Ns / 2, no window
    U.5  baud-fac on a[l] = Re IFFT_unnormalised(P), P = |FFT(|delta|)|^2 with P[0] = 0: l0 = first l >= 1 with
         a[l] < 0, amax = max a[l0 .. Ns/2), l* = first l in [l0, Ns/2 - 1) with a[l] >= amax / 2, a[l] >= a[l-1],
         a[l] >= a[l+1]; valid iff amax > 0 and l* exists; fs / l*.
         baud-nonlinear: k* = lowest arg-max of the U.3 spectrum of |delta| over [8, Ns/2); valid iff s[k*] > 0;
         k* fs / Ns.

Besides value and validity every estimator returns a margin: the smallest distance, in the units of a[] or s[], by
which one of the comparisons that chose the answer holds.  A float32 implementation whose a[] or s[] lie within E of
the statement must give the same answer wherever the margin exceeds 2 E.

`mistake` plants one deliberate error, so that the tests can show the comparison would catch it:
    "window_n"   Blackman-Harris with the denominator N instead of N - 1
    "cyclo_conj" cyclo as conj(x[i]) x[i-1], which mirrors the spectrum
    "fm_no_pi"   fmspect without the 1 / pi
    "fac_mean"   baud-fac without the mean removal (P[0] kept)
    "kmin0"      baud-nonlinear searching from k = 0 instead of 8
"""
import math

import numpy as np

KINDS = ("psd", "cyclo", "fmspect", "timediff", "abstimediff", "exp_2", "exp_4", "exp_8", "fac")
SIZES = tuple(1 << k for k in range(6, 13))
KMIN = 8
MISTAKES = ("window_n", "cyclo_conj", "fm_no_pi", "fac_mean", "kmin0")
EPS = 2.0 ** -24                      # binary32 unit roundoff


def blackman_harris(N, mistake=None):
    den = N if mistake == "window_n" else N - 1
    x = 2.0 * math.pi * np.arange(N, dtype=np.float64) / den
    return 0.35875 - 0.48829 * np.cos(x) + 0.14128 * np.cos(2 * x) - 0.01168 * np.cos(3 * x)


def frame(chan, ns):
    """U.1 -> (x[0 .. ns), x[-1 .. ns-1)) in complex128, or None when nothing is emitted"""
    c = np.asarray(chan, np.complex64).astype(np.complex128)
    if len(c) < ns + 1:
        return None
    return c[len(c) - ns:], c[len(c) - ns - 1:len(c) - 1]


def pretransform(kind, x, p, mistake=None):
    """U.2 in complex128"""
    if kind in ("psd", "fac"):
        return x
    if kind == "cyclo":
        return np.conj(x) * p if mistake == "cyclo_conj" else x * np.conj(p)
    if kind == "fmspect":
        return np.angle(x * np.conj(p)) / (1.0 if mistake == "fm_no_pi" else math.pi) + 0j
    if kind == "timediff":
        return x - p
    if kind == "abstimediff":
        return np.abs(x - p) + 0j
    return x ** {"exp_2": 2, "exp_4": 4, "exp_8": 8}[kind]


def spectrum(kind, ns, chan, mistake=None):
    """U.3 / U.4 -> float64 array (ns values, ns / 2 for fac) or None"""
    f = frame(chan, ns)
    if f is None:
        return None
    q = pretransform(kind, *f, mistake=mistake)
    if kind == "fac":
        X = np.fft.fft(q)
        return np.abs(np.fft.ifft(np.abs(X) ** 2) * ns)[:ns // 2] / ns
    X = np.fft.fft(blackman_harris(ns, mistake) * q)
    return np.abs(X) ** 2 / ns


def baud_fac_acf(ns, chan, mistake=None):
    """a[l], l < ns / 2, of U.5 baud-fac"""
    x, p = frame(chan, ns)
    X = np.fft.fft(np.abs(x - p))
    P = np.abs(X) ** 2
    if mistake != "fac_mean":
        P[0] = 0.0
    return (np.fft.ifft(P) * ns).real[:ns // 2]


def baud_fac(ns, fs, chan, mistake=None):
    """-> (value or None, margin)"""
    if frame(chan, ns) is None:
        return None, math.inf
    a = baud_fac_acf(ns, chan, mistake)
    h = ns // 2
    neg = np.flatnonzero(a[1:] < 0)
    if len(neg) == 0:
        return None, float(np.min(a[1:]))
    l0 = int(neg[0]) + 1
    margin = min(float(np.min(a[1:l0])) if l0 > 1 else math.inf, -float(a[l0]))
    amax = float(np.max(a[l0:h]))
    if not amax > 0:
        return None, min(margin, -amax)
    margin = min(margin, amax)
    thr = 0.5 * amax
    for l in range(l0, h - 1):
        slack = (a[l] - thr, a[l] - a[l - 1], a[l] - a[l + 1])
        if min(slack) >= 0:
            return fs / l, min(margin, float(min(slack)))
        margin = min(margin, max(-float(v) for v in slack if v < 0))     # the condition fails by this much
    return None, margin


def baud_nonlinear(ns, fs, chan, mistake=None):
    """-> (value or None, margin)"""
    s = spectrum("abstimediff", ns, chan)
    if s is None:
        return None, math.inf
    lo = 0 if mistake == "kmin0" else KMIN
    v = s[lo:ns // 2]
    k = int(np.argmax(v))
    rest = np.delete(v, k)
    margin = float(v[k] - rest.max()) if len(rest) else math.inf
    if not v[k] > 0:
        return None, margin
    return (k + lo) * fs / ns, min(margin, float(v[k]))


# ---- bounds (SPEC T style) ------------------------------------------------------------------------------------------
# per-sample error of the float32 pre-transform, relative to the scale named in `_input_err`
_REL = {"psd": 2, "fac": 1, "cyclo": 6, "fmspect": 0, "timediff": 2, "abstimediff": 4, "exp_2": 6, "exp_4": 16,
        "exp_8": 40}
ATAN2_ABS = 2.4e-7                    # SPEC M.2


def _input_err(kind, x, p):
    """bound on |float32 pre-transform - exact| per sample (window rounding included)"""
    ax, ap = np.abs(x), np.abs(p)
    if kind in ("psd", "fac"):
        return _REL[kind] * EPS * ax
    if kind == "cyclo":
        return _REL[kind] * EPS * ax * ap
    if kind == "fmspect":
        return np.full(len(x), (ATAN2_ABS + 12 * EPS * math.pi) / math.pi + 2 * EPS)
    if kind in ("timediff", "abstimediff"):
        return _REL[kind] * EPS * (ax + ap)
    return _REL[kind] * EPS * ax ** {"exp_2": 2, "exp_4": 4, "exp_8": 8}[kind]


def _fft_err(ns, v_norm):
    """bound on the absolute error of one output of a binary32 radix-4 transform of a vector of 2-norm v_norm"""
    return 4.0 * EPS * (math.log2(ns) + 2) * v_norm


def spectrum_bound(kind, ns, chan):
    """per-bin bound on |float32 spectrum - statement|: 1e-5 relative + what a transform error E of X does to |X|^2"""
    x, p = frame(chan, ns)
    q = pretransform(kind, x, p)
    s = spectrum(kind, ns, chan)
    if kind == "fac":
        eX = _fft_err(ns, np.linalg.norm(q)) + np.sum(_input_err(kind, x, p))
        X = np.abs(np.fft.fft(q))
        dP = 2 * X * eX + eX ** 2 + 2 * EPS * X ** 2
        eA = np.sum(dP) + _fft_err(ns, np.linalg.norm(X ** 2))
        return 1e-5 * s + eA / ns
    w = blackman_harris(ns)
    E = _fft_err(ns, np.linalg.norm(w * q)) + np.sum(w * _input_err(kind, x, p))
    return 1e-5 * s + (2 * np.sqrt(s * ns) * E + E ** 2) / ns


def acf_bound(ns, chan):
    """bound on |float32 a[l] - statement| for baud-fac"""
    x, p = frame(chan, ns)
    q = np.abs(x - p)
    X = np.abs(np.fft.fft(q))
    eX = _fft_err(ns, np.linalg.norm(q)) + np.sum(_input_err("abstimediff", x, p))
    dP = 2 * X * eX + eX ** 2 + 2 * EPS * X ** 2
    dP[0] = 0.0
    P = X ** 2
    P[0] = 0.0
    return float(np.sum(dP) + _fft_err(ns, np.linalg.norm(P)))
