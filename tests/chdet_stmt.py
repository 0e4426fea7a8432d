"""Exact statement of the channel detector, SPEC.md section K.  TEST INFRASTRUCTURE ONLY.

Written from the SPEC text alone, independently of oracle/ and of the CUDA kernels.  SPEC K is order-independent
(an order statistic and maxima, no sums), so the statement is exact: numpy binary32 element-wise operations give
the same bits as any correct implementation.

    K.1  per frame, in order: avg <- avg + alpha (psd - avg); the first frame ever initialises avg
    K.2  per feed: N0_inst = the (N/4)-th smallest avg (0-based); N0 <- N0 + gamma (N0_inst - N0), the first update
         N0 = N0_inst; T = N0 snr.  A feed without frames changes nothing.
    K.3  maximal runs [a, b) of avg > T in ascending frequency j = (k + N/2) mod N, clipped at both band edges
    K.4  the first 8192 runs only; runs narrower than min_bins dropped; the total kept before the 256 cap;
         S0 = max avg over the run, snr = S0 / N0; frequencies in binary64

`mistake` plants one deliberate error, so that the tests can show the comparison would catch it:
    "rank"     the (N/4 - 1)-th smallest value as the noise floor
    "ge"       avg >= T instead of avg > T
    "no_shift" runs in bin order k instead of frequency order j
    "wrap"     a run touching the top edge merged with one touching the bottom edge
    "no_cap"   every run examined, not only the first 8192
"""
import numpy as np

MAXRAW = 8192
CAP = 256
MISTAKES = ("rank", "ge", "no_shift", "wrap", "no_cap")


class Channel:
    __slots__ = ("bin_lo", "bin_hi", "S0", "N0", "snr")

    def __init__(self, a, b, s0, n0, snr):
        self.bin_lo, self.bin_hi, self.S0, self.N0, self.snr = int(a), int(b), np.float32(s0), np.float32(n0), \
            np.float32(snr)

    def key(self):
        """bins and the bit patterns of S0, N0, snr"""
        return (self.bin_lo, self.bin_hi, int(self.S0.view(np.uint32)), int(self.N0.view(np.uint32)),
                int(self.snr.view(np.uint32)))


def runs(mask):
    """maximal runs [a, b) of True in a 1-D bool array, no wrap-around"""
    d = np.diff(np.concatenate(([False], mask, [False])).astype(np.int8))
    return np.flatnonzero(d == 1), np.flatnonzero(d == -1)


def frequencies(a, b, N, samp_rate, center):
    """K.4 in binary64: (f_lo, f_hi, fc, bw) of bins [a, b)"""
    f_lo = center + (a - N / 2) * samp_rate / N
    f_hi = center + (b - N / 2) * samp_rate / N
    return f_lo, f_hi, (f_lo + f_hi) / 2, f_hi - f_lo


class Detector:
    def __init__(self, N, alpha, gamma, snr, min_bins, mistake=None):
        assert N >= 16 and N & (N - 1) == 0 and mistake in (None,) + MISTAKES
        self.N, self.min_bins, self.mistake = N, max(1, int(min_bins)), mistake
        self.alpha, self.gamma, self.snr = np.float32(alpha), np.float32(gamma), np.float32(snr)
        self.avg = None
        self.n0 = None
        self.channels, self.total = [], 0

    def feed(self, frames):
        """frames: [f, N] float32 linear PSD frames, DC at index 0 -> (channels up to the cap, total)"""
        frames = np.asarray(frames, np.float32).reshape(-1, self.N)
        if len(frames) == 0:
            return self.channels, self.total
        for p in frames:                                            # K.1
            self.avg = p.copy() if self.avg is None else self.avg + self.alpha * (p - self.avg)
        N = self.N
        rank = N // 4 - (1 if self.mistake == "rank" else 0)        # K.2
        inst = np.sort(self.avg)[rank]
        self.n0 = inst if self.n0 is None else np.float32(self.n0 + self.gamma * (inst - self.n0))
        thr = np.float32(self.n0 * self.snr)
        v = self.avg if self.mistake == "no_shift" else np.roll(self.avg, N // 2)     # v[j] = avg[(j + N/2) mod N]
        a, b = runs(v >= thr if self.mistake == "ge" else v > thr)  # K.3
        if self.mistake == "wrap" and len(a) > 1 and a[0] == 0 and b[-1] == N:
            a, b = np.append(a[1:-1], a[-1]), np.append(b[1:-1], b[0] + N)
            v = np.concatenate([v, v])
        if self.mistake != "no_cap":                                # K.4
            a, b = a[:MAXRAW], b[:MAXRAW]
        keep = (b - a) >= self.min_bins
        a, b = a[keep], b[keep]
        self.total = len(a)
        with np.errstate(divide="ignore"):
            self.channels = []
            for lo, hi in zip(a[:CAP], b[:CAP]):
                s0 = v[lo:hi].max()
                self.channels.append(Channel(lo, hi, s0, self.n0, np.float32(s0) / np.float32(self.n0)))
        return self.channels, self.total


# ---- scenes: multi-feed PSD sequences at the edges of K ------------------------------------------------------------
def _carriers(p, N, spans, level):
    for k0, k1 in spans:
        k = np.arange(k0, k1) % N
        p[..., k] += level


def scenes(N, streams=1, seed=0):
    """[(name, dict(alpha, gamma, snr, min_bins), [feed [streams, frames, N] float32, ...])] for one size N.
    Every stream gets its own noise; the structure (carriers, ties, patterns) is the same."""
    rng = np.random.default_rng(seed * 7919 + N)
    noise = lambda f: rng.exponential(1.0, (streams, f, N)).astype(np.float32)
    w = max(2, N // 32)
    out = []

    def carrier_feeds(frames):
        fs = []
        for f in frames:
            p = noise(f)
            _carriers(p, N, [(N // 8, N // 8 + max(1, N // 64)), (5 * N // 8, 5 * N // 8 + max(3, N // 16))], 20.0)
            fs.append(p)
        return fs

    for alpha in (0.0, 0.25, 1.0):
        for gamma in (0.0, 0.25, 1.0):
            out.append(("noise_carriers_a%g_g%g" % (alpha, gamma),
                        dict(alpha=alpha, gamma=gamma, snr=4.0, min_bins=max(1, N // 512)), carrier_feeds([1, 4, 2])))
    out.append(("zero_frame_feed", dict(alpha=0.25, gamma=0.5, snr=4.0, min_bins=1), carrier_feeds([2, 0, 3])))

    # carriers touching both band edges (around k = N/2) and one straddling DC (k = 0)
    fs = []
    for f in (2, 1):
        p = noise(f)
        _carriers(p, N, [(N // 2 - w, N // 2 + w), (N - w, N + w)], 40.0)
        fs.append(p)
    out.append(("edges_dc", dict(alpha=1.0, gamma=1.0, snr=6.0, min_bins=1), fs))

    # isolated one-bin runs every fourth bin
    fs = []
    for f in (1, 3):
        p = noise(f)
        p[..., 1::4] += 50.0
        fs.append(p)
    out.append(("one_bin_runs", dict(alpha=0.0, gamma=0.0, snr=100.0, min_bins=1), fs))

    # ties: a constant spectrum (every bin equals T at snr 1; one band-wide run below snr 1), and a quartile inside
    # a block of more than N/4 equal bins
    const = [np.full((streams, f, N), 2.5, np.float32) for f in (1, 2)]
    out.append(("constant_snr1", dict(alpha=0.25, gamma=0.25, snr=1.0, min_bins=1), const))
    out.append(("constant_snr_half", dict(alpha=0.25, gamma=0.25, snr=0.5, min_bins=1), const))
    fs = []
    for f in (1, 2):
        p = noise(f) + 3.0
        idx = rng.permutation(N)
        p[..., idx[:N // 8]] = 0.25
        p[..., idx[N // 8:N // 2]] = 1.0
        fs.append(p)
    out.append(("tied_quartile", dict(alpha=1.0, gamma=0.25, snr=2.0, min_bins=1), fs))

    # zeros: N0 = 0, T = 0; with carriers over the zero floor snr = S0 / 0 = inf
    out.append(("all_zero", dict(alpha=0.25, gamma=0.25, snr=4.0, min_bins=1),
                [np.zeros((streams, f, N), np.float32) for f in (1, 2)]))
    fs = []
    for f in (1, 2):
        p = np.zeros((streams, f, N), np.float32)
        _carriers(p, N, [(N // 8, N // 8 + w), (3 * N // 4, 3 * N // 4 + 1)], 5.0)
        fs.append(p)
    out.append(("zero_floor", dict(alpha=0.25, gamma=1.0, snr=4.0, min_bins=1), fs))

    out.append(("snr_below_1", dict(alpha=0.25, gamma=0.25, snr=0.5, min_bins=1), [noise(f) for f in (2, 1)]))

    if N >= 1024:
        # runs of two bins every three, every tenth one cut to a single bin: > 256 kept, the cut ones dropped
        pat = np.zeros(N, bool)
        pat[0::3] = True
        pat[1::3] = True
        pat[1::30] = False
        fs = []
        for f in (1, 2):
            p = noise(f) * 0.1
            p[..., np.roll(pat, N // 2)] += 30.0
            fs.append(p)
        out.append(("many_channels", dict(alpha=0.5, gamma=0.5, snr=4.0, min_bins=2), fs))
    if N >= 1 << 15:
        # alternating bins: N/2 one-bin runs, more than the 8192 examined; those past the cap would pass min_bins
        fs = []
        for f in (1, 1):
            p = noise(f) * 0.1
            p[..., 0::2] += 1000.0
            fs.append(p)
        out.append(("alternating", dict(alpha=1.0, gamma=1.0, snr=100.0, min_bins=1), fs))
    return out
