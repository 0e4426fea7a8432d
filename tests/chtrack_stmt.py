"""Exact statement of channel tracking across detector updates, oracle/SPEC_KT.md.  TEST INFRASTRUCTURE ONLY.

Written from the SPEC text alone, independently of oracle/ and of the CUDA kernels.  The only arithmetic is the
binary32 smoothing of KT.4, one rounding per operation, so the statement is exact.

    KT.1  one update per detector update (feeds without frames change nothing)
    KT.2  input: the K.4 list, ascending frequency, detection d = [a_d, b_d) with peak S0_d
    KT.3  detections in order; candidates: unmatched tracks with overlap min(b_d, b_t) - max(a_d, a_t) > 0; the
          largest overlap wins, ties by the smaller a_t, then the smaller id
    KT.4  matched: [a, b) <- [a_d, b_d); S0 <- S0 + beta (S0_d - S0); age += 1, present += 1, misses = 0
    KT.5  unmatched: age += 1, misses += 1; removed when misses > hold; every removal before any insertion
    KT.6  unmatched detections open tracks (id = next_id++, from 1) in ascending frequency while fewer than 256 are
          live; the rest count in `dropped`
    KT.7  output: every live track in ascending (a, id); snr = S0 / N0

`mistake` plants one deliberate error, so that the tests can show the comparison would catch it:
    "first_overlap"     the first candidate in (a, id) order instead of the largest overlap
    "insert_first"      insertions before removals (the tracks about to be removed still take room)
    "misses_ge"         removal at misses >= hold instead of misses > hold
    "smooth_unmatched"  an unmatched track smoothed towards 0 as if detected at S0_d = 0
"""
import numpy as np

CAP = 256
MISTAKES = ("first_overlap", "insert_first", "misses_ge", "smooth_unmatched")


class Track:
    __slots__ = ("a", "b", "S0", "id", "age", "present", "misses")

    def __init__(self, a, b, s0, id_):
        self.a, self.b, self.S0, self.id = int(a), int(b), np.float32(s0), int(id_)
        self.age, self.present, self.misses = 1, 1, 0

    def key(self):
        """range, the bit pattern of S0, id and counters"""
        return (self.a, self.b, int(np.float32(self.S0).view(np.uint32)), self.id, self.age, self.present,
                self.misses)


class Tracker:
    def __init__(self, beta, hold, mistake=None):
        assert 0 < beta <= 1 and 0 <= hold <= 65535 and mistake in (None,) + MISTAKES
        self.beta, self.hold, self.mistake = np.float32(beta), int(hold), mistake
        self.tracks, self.next_id, self.dropped = [], 1, 0

    def update(self, dets):
        """dets: [(a, b, S0)] in ascending frequency (the K.4 list of one update) -> live tracks, ascending (a, id)"""
        old = self.tracks                                   # ascending (a, id)
        matched = [False] * len(old)
        new_dets = []
        for a_d, b_d, s0_d in dets:                         # KT.3
            best, best_key = None, None
            for i, t in enumerate(old):
                ov = min(b_d, t.b) - max(a_d, t.a)
                if matched[i] or ov <= 0:
                    continue
                k = (-ov, t.a, t.id)
                if best is None or k < best_key:
                    best, best_key = i, k
                    if self.mistake == "first_overlap":
                        break
            if best is None:
                new_dets.append((a_d, b_d, s0_d))
                continue
            t = old[best]                                   # KT.4
            matched[best] = True
            t.a, t.b = int(a_d), int(b_d)
            t.S0 = np.float32(t.S0 + np.float32(self.beta * np.float32(np.float32(s0_d) - t.S0)))
            t.age += 1
            t.present += 1
            t.misses = 0
        kept = []
        for i, t in enumerate(old):                         # KT.5
            if matched[i]:
                kept.append(t)
                continue
            t.age += 1
            t.misses += 1
            if self.mistake == "smooth_unmatched":
                t.S0 = np.float32(t.S0 + np.float32(self.beta * np.float32(np.float32(0) - t.S0)))
            gone = t.misses >= self.hold if self.mistake == "misses_ge" else t.misses > self.hold
            if not gone:
                kept.append(t)
        room = CAP - (len(old) if self.mistake == "insert_first" else len(kept))
        for a_d, b_d, s0_d in new_dets:                     # KT.6
            if room <= 0:
                self.dropped += 1
                continue
            kept.append(Track(a_d, b_d, s0_d, self.next_id))
            self.next_id += 1
            room -= 1
        self.tracks = sorted(kept, key=lambda t: (t.a, t.id))   # KT.7
        return self.tracks


def snr(track, n0):
    """KT.7: S0 / N0 in binary32"""
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.float32(np.float32(track.S0) / np.float32(n0))


# ---- scenes: sequences of K.4 lists at the edges of KT ---------------------------------------------------------------
def _d(a, b, s0):
    return (int(a), int(b), np.float32(s0))


def list_scenes():
    """[(name, [K.4 list per update])].  Each list is [(a, b, S0)] in ascending frequency with disjoint runs."""
    out = []
    # carriers that appear, vanish for 1, 2 and 9 updates, and return
    seq = []
    for u in range(24):
        lst = [_d(100, 120, 10.0 + u)]
        if u not in (3,) and u not in (6, 7) and not 10 <= u < 19:
            lst.append(_d(300, 310, 50.0 - u))
        if u % 5 != 2:
            lst.append(_d(500 + (u % 3), 520 + (u % 4), 3.0 + 0.125 * u))
        seq.append(sorted(lst))
    out.append(("appear_vanish_return", seq))
    # a run that splits in two, and two runs that merge (the right one overlapping more)
    out.append(("split", [[_d(100, 200, 8.0)], [_d(100, 200, 9.0)], [_d(100, 140, 7.0), _d(150, 200, 12.0)],
                          [_d(100, 140, 7.5), _d(150, 200, 11.0)], [_d(90, 210, 6.0)]]))
    out.append(("merge", [[_d(100, 130, 5.0), _d(140, 200, 9.0)], [_d(100, 130, 5.5), _d(140, 200, 8.0)],
                          [_d(100, 200, 20.0)], [_d(100, 200, 21.0)], [_d(100, 130, 4.0), _d(140, 200, 7.0)]]))
    # overlap ties: one detection covers two tracks by the same amount (smaller a wins), and two tracks with the same
    # a and the same overlap (a newer track moved onto the start of an older one in hold; the smaller id wins)
    out.append(("tie_a", [[_d(100, 110, 4.0), _d(120, 130, 6.0)], [_d(105, 125, 8.0)], [_d(105, 125, 9.0)],
                          [_d(100, 110, 2.0), _d(120, 130, 3.0)]]))
    out.append(("tie_id", [[_d(201, 220, 4.0)], [_d(180, 200, 1.0)], [_d(185, 205, 5.0)], [_d(201, 205, 6.0)],
                           [_d(201, 205, 7.0)], [], [_d(201, 205, 8.0)]]))
    # cap: 256 tracks live, then 256 others (dropped while the first are in hold), then the first return
    first = [_d(8 * i, 8 * i + 3, 10.0 + i) for i in range(CAP)]
    second = [_d(8 * i + 4, 8 * i + 7, 100.0 + i) for i in range(CAP)]
    half = [_d(8 * i + 4, 8 * i + 7, 50.0 + i) for i in range(0, CAP, 2)]
    out.append(("cap_dropped", [first, second, second, first, half, [], second, first]))
    # empty updates and an empty start
    out.append(("empty_updates", [[], [_d(10, 20, 3.0)], [], [], [_d(12, 22, 4.0)], [], [], [], [], [_d(10, 20, 1.0)]]))
    return out


def drive(lists, beta, hold, mistake=None):
    """Tracks every list of a scene; returns [(keys of the live tracks, dropped, next_id)] per update."""
    t = Tracker(beta, hold, mistake)
    out = []
    for lst in lists:
        t.update(lst)
        out.append(([x.key() for x in t.tracks], t.dropped, t.next_id))
    return out
