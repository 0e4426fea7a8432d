"""SPEC FC.2 - FC.4 (oracle/SPEC_FC.md) stated in numpy binary32, from the SPEC text alone: the statistics of a feed's
blocks over the lag window, the excluded-record rule, the tiled power sum, the averaging and the per-feed status.
TEST INFRASTRUCTURE ONLY.  Every operation is one float32 rounding in the SPEC's order (numpy never contracts)."""
import numpy as np

F = np.float32
TILE = 1024


class FacStmt:
    def __init__(self, L, alpha=1.0, lags=None, sigma=5.0):
        lo, hi = lags if lags is not None else (0, 0)
        if lo == 0 and hi == 0:
            hi = L // 2
        assert 0 <= lo < hi <= L // 2
        self.L, self.lo, self.hi, self.alpha, self.sigma = L, lo, hi, F(alpha), float(sigma)
        self.max, self.min = F(-np.inf), F(np.inf)
        self.fac = np.zeros(L // 2, np.float32)

    def feed_v(self, vs, tiles=TILE, reset_local_per_block=False, record_in_power=False, max_before=False,
               max_outside=False):
        """FC.2 - FC.4 over the v arrays of one feed's completed blocks.  The keyword arguments plant the mistakes the
        statement test must catch; all False is the SPEC."""
        with np.errstate(invalid="ignore", divide="ignore"):     # an all-zero block divides 0 by 0, as the tab does
            return self._feed_v(vs, tiles, reset_local_per_block, record_in_power, max_before, max_outside)

    def _feed_v(self, vs, tiles, reset_local_per_block, record_in_power, max_before, max_outside):
        local, pos, power, count = F(-np.inf), 0, F(0), 0
        for v in vs:
            v = np.asarray(v, np.float32)
            if reset_local_per_block:
                local = F(-np.inf)
            w = v[self.lo:self.hi]
            # FC.2 records: a value above every earlier value of the feed's window (NaN never is one)
            prev = np.fmax.accumulate(np.concatenate([[local], w]))[:-1]
            rec = w > prev
            if w.size and np.any(rec):
                top = np.nanmax(w[rec])
                local, pos = F(top), self.lo + int(np.flatnonzero(rec)[-1])
            sq = np.where(rec & (not record_in_power), F(0), w * w).astype(np.float32)
            count += int(w.size - (0 if record_in_power else rec.sum()))
            # tiles of 1024 lags from lo, each summed by the fixed tree s[i] += s[i + h], h = 512 .. 1; tile sums in order
            for t0 in range(0, w.size, tiles):
                s = np.zeros(tiles, np.float32)
                part = sq[t0:t0 + tiles]
                s[:part.size] = part
                h = tiles // 2
                while h:
                    s[:h] = s[:h] + s[h:2 * h]
                    h //= 2
                power = F(power + s[0])
            old_max = self.max
            src = v if max_outside else w
            if src.size and not np.all(np.isnan(src)):
                self.max = F(np.fmax(self.max, np.nanmax(src)))
                self.min = F(np.fmin(self.min, np.nanmin(src)))
            m = old_max if max_before else self.max
            # FC.3
            t = (v / m).astype(np.float32)
            self.fac = (self.fac + self.alpha * (t - self.fac)).astype(np.float32)
        sigmas, marker = F(0), 0
        if len(vs) and not np.isinf(local) and count > 0:
            sigmas = F(local / np.sqrt(F(power / F(count))))
            marker = int(float(sigmas) > self.sigma)
        return dict(blocks=len(vs), peak_lag=pos if len(vs) else 0, max=self.max, min=self.min, sigmas=sigmas,
                    marker=marker)


def key(st):
    b = lambda x: int(np.float32(x).view(np.uint32))     # noqa: E731
    return (st["blocks"], st["peak_lag"], b(st["max"]), b(st["min"]), b(st["sigmas"]), st["marker"])
