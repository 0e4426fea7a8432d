"""Float64 statement of the spectral tuner, SPEC.md section S.  TEST INFRASTRUCTURE ONLY.

Written from the SPEC text alone, independently of oracle/specttuner.c and of the CUDA kernels, so that both can be
held to the mathematics rather than only to each other.  Everything is binary64 except what the SPEC fixes in binary32:
the channel parameters (f0, bw, guard are SUFLOAT), the NCQO frequency of a `precise` channel and the NCQO phase
accumulator (SPEC N), which runs in float32 as the specified state does.

    S.1  window N, hop N/2, unnormalised forward transform of input samples [m N/2, m N/2 + N)
    S.2  geometry (center, size, width)
    S.3  weights k h, k = 1/N; h the brick wall [-halfw, halfw) convolved with the 7-tap Blackman-Harris spectrum,
         h = 1 for a channel spanning the whole band; bin +i -> slot i, bin -j -> slot size - j
    S.4  unnormalised size-point inverse transform; out[i] = w[i] cur[i] + w[i + size/2] prev[size/2 + i],
         w[i] = sin^2(pi i / size), prev = 0 before the first transform; `precise`: times conj(lo)
"""
import math

import numpy as np

TWO_PI = 2.0 * math.pi
# SPEC S.3 coefficients c_|m| of the periodic Blackman-Harris spectrum
BH_C = (0.35875, 0.48829 / 2.0, 0.14128 / 2.0, 0.01168 / 2.0)
PI_F = np.float32(math.pi)
TWO_PI_F = np.float32(TWO_PI)


def geometry(N, f0, bw, guard):
    """SPEC S.2 in binary64 from the float32 parameters -> (center, size, width)."""
    f0, bw, guard = float(np.float32(f0)), float(np.float32(bw)), float(np.float32(guard))
    center = int(2 * math.floor(f0 / (4.0 * math.pi) * N + 0.5)) % N
    m = math.ceil(guard * bw / TWO_PI * N - 1e-3)
    m = min(max(m, 4), N)
    size = 1
    while size < m:
        size <<= 1
    width = min(max(math.ceil(m / guard - 1e-3), 2), size)
    return center, size, width


def weights(N, halfw):
    """k h for the signed bins b = -halfw .. halfw - 1 (SPEC S.3), float64."""
    b = np.arange(-halfw, halfw)
    if 2 * halfw >= N:                                    # the channel spans the whole band
        return np.full(2 * halfw, 1.0 / N)
    h = np.zeros(2 * halfw)
    for m in range(-3, 4):
        q = b - m
        h += BH_C[abs(m)] * ((q >= -halfw) & (q < halfw))
    return h / N


def lo_omega(N, f0, center, size):
    """float32 NCQO angular frequency of a `precise` channel (SPEC S.4, N): the residual f0 - 2 pi center / N,
    wrapped into (-pi, pi], scaled by the decimation N / size to radians per channel sample."""
    resid = float(np.float32(f0)) - TWO_PI * center / N
    resid = math.pi - ((math.pi - resid) % TWO_PI)          # (-pi, pi]
    fnor = np.float32(resid * (N / size) / math.pi)
    return np.float32(PI_F * fnor)


def lo_phases(omega, n):
    """The NCQO phase at each of n reads: phi_0 = 0, phi <- wrap(phi + omega) in float32 (SPEC N)."""
    phi = np.empty(n, np.float32)
    p = np.float32(0.0)
    for i in range(n):
        phi[i] = p
        p = np.float32(p + omega)
        if p >= TWO_PI_F:
            p = np.float32(p - TWO_PI_F)
        elif p < 0:
            p = np.float32(p + TWO_PI_F)
    return phi


def spectra(x, N):
    """S.1: the unnormalised forward transforms of the windows [m N/2, m N/2 + N) of x -> [hops, N] complex128
    (trailing samples that do not complete a window are not transformed)."""
    x = np.asarray(x).astype(np.complex128)
    if len(x) < N:
        return np.zeros((0, N), np.complex128)
    hops = (len(x) - N) // (N // 2) + 1
    frames = np.lib.stride_tricks.as_strided(x, shape=(hops, N), strides=(x.strides[0] * (N // 2), x.strides[0]))
    return np.fft.fft(frames, axis=1)


def channel(x, N, f0, bw, guard=1.0, precise=False, X=None):
    """Channel-rate samples of one channel over the input x, complex128.  X: spectra(x, N), when already at hand."""
    center, size, width = geometry(N, f0, bw, guard)
    halfw, hs = width // 2, size // 2
    X = spectra(x, N) if X is None else X
    hops = X.shape[0]
    kh = weights(N, halfw)
    slots = np.zeros((hops, size), np.complex128)
    up = np.arange(halfw)                                                     # bin +i -> slot i
    slots[:, up] = X[:, (center + up) % N] * kh[halfw + up]
    dn = np.arange(1, halfw + 1)                                              # bin -j -> slot size - j
    slots[:, size - dn] = X[:, (center - dn) % N] * kh[halfw - dn]
    cur = np.fft.ifft(slots, axis=1) * size                                   # S.4, unnormalised
    w = np.sin(np.pi * np.arange(size) / size) ** 2
    prev = np.zeros((hops, hs), np.complex128)
    prev[1:] = cur[:-1, hs:]
    out = (w[:hs] * cur[:, :hs] + w[hs:] * prev).reshape(-1)
    if precise:
        phi = lo_phases(lo_omega(N, f0, center, size), len(out)).astype(np.float64)
        out = out * (np.cos(phi) - 1j * np.sin(phi))
    return out


# ------------------------------------------------------------------------------------------------------------------
# channel sets and inputs shared by the CPU and GPU channeliser tests
# ------------------------------------------------------------------------------------------------------------------
def f32(v):
    return float(np.float32(v))


def edge_channels(N):
    """The geometry edges of SPEC S.2 / S.3 at window N, as channel parameter dicts (float32-representable)."""
    b = TWO_PI / N                                          # one bin
    c0 = 2 * (N // 8)                                       # an even bin away from the edges
    bw_dc = f32(max(TWO_PI * 0.02, 12 * b))                 # wide enough to reach across DC at N = 64
    return [
        dict(f0=f32(TWO_PI * 0.125), bw=f32(TWO_PI * 0.03), guard=1.0),
        dict(f0=0.0, bw=f32(TWO_PI * 0.05), guard=1.0),                        # centred on DC
        dict(f0=f32(TWO_PI - 0.4 * b), bw=f32(TWO_PI * 0.02), guard=1.0),     # centre wraps to bin 0
        dict(f0=f32(TWO_PI - max(0.004 * N, 2.6) * b), bw=bw_dc, guard=1.0),  # straddles DC from above
        dict(f0=f32(max(0.003 * N, 1.7) * b), bw=bw_dc, guard=1.0),           # straddles DC from below
        dict(f0=f32(TWO_PI * 0.25), bw=f32(TWO_PI), guard=1.0),               # full band: h = 1, size = N
        dict(f0=f32(TWO_PI * 0.3), bw=f32(b), guard=8.0),                     # minimum width 2
        dict(f0=f32(TWO_PI * 0.7003), bw=f32(TWO_PI * 0.011), guard=1.5),
        dict(f0=f32(TWO_PI * 0.61), bw=f32(TWO_PI * 0.017), guard=1.3),
        dict(f0=f32(TWO_PI * 0.131), bw=f32(TWO_PI * 0.02), guard=1.0),       # shares bins with the first
        dict(f0=f32((c0 + 0.6) * b), bw=f32(TWO_PI * 0.01), guard=2.0, precise=True),   # residual > 0
        dict(f0=f32((c0 + 1.4) * b), bw=f32(TWO_PI * 0.01), guard=2.0, precise=True),   # residual < 0
        dict(f0=f32(TWO_PI - 0.6 * b), bw=f32(TWO_PI * 0.01), guard=1.0, precise=True), # wrapped centre
    ]


def signal(n, chans, seed, noise=0.05):
    """complex64 noise plus one tone near each channel's f0 (so that every channel carries a signal well above the
    float32 floor) and one in no channel."""
    rng = np.random.default_rng(seed)
    x = noise * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    t = np.arange(n)
    for i, c in enumerate(chans):
        f = c["f0"] / TWO_PI + (0.05 + 0.02 * i) * c["bw"] / TWO_PI
        x += (0.2 + 0.02 * i) * np.exp(2j * np.pi * f * t)
    x += 0.3 * np.exp(2j * np.pi * 0.45 * t)
    return x.astype(np.complex64)
