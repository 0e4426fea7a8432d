"""Statement of SPEC US (oracle/SPEC_US.md): the emissions of one scheduled channel, feed by feed, with the history
kept the way the engine keeps it (a ring of Ns + 1 samples indexed by t mod (Ns + 1), written only with the samples a
later frame of this interval can still need).  Each frame goes through `frame_fn`, in practice the oracle's
sdo_spectsrc_frame / sdo_estimate_baud, which take the last Ns + 1 samples of what they are given.

`reference` is the whole-stream form of US.3 / US.4: the emission at t_j is frame_fn over c[0 .. t_j - 1]."""
import numpy as np

# planted mistakes, each rejected by a named case of tests/test_spectsched_stmt.py
MISTAKES = ("frame_ends_early", "emits_before_ns1", "history_not_carried")


def schedule(feeds, ns, interval, frame_fn, mistake=None, state=None):
    """feeds: the channel samples of each feed (1-D complex64).  Returns ([[(t_j, frame_fn(frame)), ...] per feed],
    state); pass the state back in to continue (a re-plan that carries the history)."""
    ns1, I = ns + 1, int(interval)
    ring, t, v = state if state is not None else (np.zeros(ns1, np.complex64), 0, 0)
    ring = ring.copy()
    out = []
    for f in feeds:
        f = np.asarray(f, np.complex64)
        T0, T1 = t, t + len(f)
        lo = 0 if mistake == "emits_before_ns1" else v + ns1      # US.3 / US.5: t_j - Ns - 1 >= v
        first = (T0 // I + 1) * I
        if first < lo:
            first += -(-(lo - first) // I) * I
        em = []
        for tj in range(first, T1 + 1, I):
            m = np.arange(tj - ns1, tj, dtype=np.int64) - (1 if mistake == "frame_ends_early" else 0)
            inside = m >= T0
            frame = np.where(inside, f[np.clip(m - T0, 0, max(len(f) - 1, 0))], ring[m % ns1])
            em.append((tj, frame_fn(frame.astype(np.complex64))))
        nxt = (T1 // I + 1) * I                                    # samples a later frame can still need
        a = min(T1, max(T0, nxt - ns1))
        m = np.arange(a, T1, dtype=np.int64)
        ring[m % ns1] = f[m - T0]
        if a > T0:
            v = a
        if mistake == "history_not_carried":
            ring[:] = 0
        t = T1
        out.append(em)
    return out, (ring, t, v)


def reference(c, ns, interval, frame_fn):
    """[(t_j, frame_fn(c[:t_j]))] for every t_j = j I <= len(c) with t_j >= Ns + 1"""
    I = int(interval)
    first = max(I, -(-(ns + 1) // I) * I)
    return [(tj, frame_fn(c[:tj])) for tj in range(first, len(c) + 1, I)]


def same(a, b):
    """emission lists equal bit for bit (values compared as their binary32 patterns; None = nothing / invalid)"""
    if len(a) != len(b):
        return False
    for (ta, ra), (tb, rb) in zip(a, b):
        if ta != tb or len(ra) != len(rb):
            return False
        for x, y in zip(ra, rb):
            if (x is None) != (y is None):
                return False
            if x is not None and not np.array_equal(np.atleast_1d(np.float32(x)).view(np.uint32),
                                                    np.atleast_1d(np.float32(y)).view(np.uint32)):
                return False
    return True
