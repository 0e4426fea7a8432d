"""Float64 statement of the main PSD, SPEC.md sections W, P, Q, R and M.6.  TEST INFRASTRUCTURE ONLY.

Written from the SPEC text alone, independently of oracle/ and of the CUDA kernels, so that both can be held to the
mathematics rather than only to each other.  Everything is binary64 except what the SPEC fixes in binary32: the
converted samples (Q, exact in binary32) and the DC-removal estimate and subtraction (R).

    W    window taps of length L, x = 2 pi n / (L - 1): Hamming, Hann, flat-top, Blackman-Harris (not rounded here)
    P    psd[k] = |FFT(w o x)[k]|^2 / N per frame of N consecutive samples, DC at index 0
    Q    RAW_FLOAT32 as is; RAW_UNSIGNED8 (v - 128) / 128; RAW_SIGNED8 v / 128; RAW_SIGNED16 v / 32768;
         iq_reverse takes the pair as (Q, I)
    R    per block of n samples: y = x - c (binary32), then c <- c + alpha (m - c) (binary32), alpha =
         (float)(1 - exp(-n / (fs 0.1))), m the mean of the raw block summed in binary64 in runs of 256 samples
         (index order, the last run partial) and then over the run sums (index order), divided by n, rounded once
    M.6  PSDMessage layout: halves swapped, 10 log10(p + 1e-8)
"""
import math

import numpy as np

KINDS = ("none", "hamming", "hann", "flat_top", "blackmann_harris")

# SPEC W cosine-sum coefficients a_j of sum_j a_j cos(j x)
_COEF = {
    "none": (1.0,),
    "hamming": (0.54, -0.46),
    "hann": (0.5, -0.5),
    "flat_top": (1.0, -1.93, 1.29, -0.388, 0.028),
    "blackmann_harris": (0.35875, -0.48829, 0.14128, -0.01168),
}


def window(N, kind):
    """SPEC W taps in binary64 (symmetric form, denominator N - 1), not rounded."""
    if N > 1:
        x = 2.0 * math.pi * np.arange(N, dtype=np.float64) / (N - 1)
    else:
        x = np.zeros(N)
    w = np.zeros(N)
    for j, a in enumerate(_COEF[kind]):
        w += a * np.cos(j * x)
    return w


def convert(raw, fmt, iq_reverse=False):
    """SPEC Q: native samples -> complex64.  raw: [..., n] complex64 for "f32", [..., n, 2] integers otherwise."""
    if fmt == "f32":
        x = np.asarray(raw, np.complex64)
        re, im = x.real.astype(np.float64), x.imag.astype(np.float64)
    else:
        v = np.asarray(raw).astype(np.float64)
        if fmt == "u8":
            v = (v - 128.0) / 128.0
        elif fmt == "s8":
            v = v / 128.0
        elif fmt == "s16":
            v = v / 32768.0
        else:
            raise ValueError(fmt)
        re, im = v[..., 0], v[..., 1]
    if iq_reverse:
        re, im = im, re
    out = (re + 1j * im).astype(np.complex64)
    assert np.array_equal(out.real.astype(np.float64), re) and np.array_equal(out.imag.astype(np.float64), im)
    return out


def _seq_sum(v):
    """v[0] + v[1] + ... from 0.0, one binary64 rounding per addition, in index order."""
    return float(np.cumsum(np.concatenate([[0.0], np.asarray(v, np.float64)]))[-1])


def _block_sum(v):
    """SPEC R's two-level sum: sequential within runs of 256 (the last one partial), then over the run sums."""
    return _seq_sum([_seq_sum(v[i:i + 256]) for i in range(0, len(v), 256)])


def dc_remove(blocks, fs):
    """SPEC R over consecutive blocks (complex64 each, already converted by Q) -> corrected complex64 blocks."""
    c = np.zeros(2, np.float32)
    out = []
    for b in blocks:
        b = np.asarray(b, np.complex64)
        n = len(b)
        alpha = np.float32(1.0 - math.exp(-n / (fs * 0.1)))
        m = np.array([_block_sum(b.real) / n, _block_sum(b.imag) / n], np.float32)
        y = np.empty_like(b)
        y.real = b.real - c[0]
        y.imag = b.imag - c[1]
        out.append(y)
        c = (c + alpha * (m - c)).astype(np.float32)
    return out


def psd(x, N, kind):
    """SPEC P in complex128 over the consecutive N-sample frames of x -> [frames, N] float64."""
    x = np.asarray(x).astype(np.complex128)
    frames = len(x) // N
    X = np.fft.fft(x[:frames * N].reshape(frames, N) * window(N, kind), axis=1)
    return (X.real ** 2 + X.imag ** 2) / N


def shift_db(p):
    """SPEC M.6 on the last axis: bin k moves to (k + N/2) mod N, then 10 log10(p + 1e-8), in binary64."""
    p = np.asarray(p, np.float64)
    return 10.0 * np.log10(np.roll(p, p.shape[-1] // 2, axis=-1) + 1e-8)
