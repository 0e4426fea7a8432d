"""ctypes binding of the CPU oracle's channel tracker (sdo_chtrack_*, oracle/chtrack.c, SPEC_KT.md), built by
oracle/chtrack.mk as oracle/_build/libsdchtrack.so.  TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib

CAP = 256
LIB_PATH = os.path.join(oracle_lib.ORACLE_DIR, "_build", "libsdchtrack.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        subprocess.run(["make", "-C", oracle_lib.ORACLE_DIR, "-f", "chtrack.mk"], check=True, capture_output=True)
        _lib = C.CDLL(LIB_PATH)
    return _lib


class OTrack(C.Structure):
    _fields_ = [("a", C.c_uint), ("b", C.c_uint), ("s0", C.c_float), ("id", C.c_uint), ("age", C.c_uint),
                ("present", C.c_uint), ("misses", C.c_uint)]


class OChTrack(C.Structure):
    _fields_ = [("beta", C.c_float), ("hold", C.c_uint), ("count", C.c_uint), ("next_id", C.c_uint),
                ("dropped", C.c_ulonglong), ("tr", OTrack * CAP)]


class Tracker:
    def __init__(self, beta, hold):
        self.L = lib()
        self.t = OChTrack()
        self.L.sdo_chtrack_init(C.byref(self.t), C.c_float(beta), C.c_uint(hold))

    def update(self, dets):
        """dets: [(a, b, S0)] in ascending frequency (a K.4 list)"""
        arr = (oracle_lib.OChannel * max(1, len(dets)))()
        for i, (a, b, s0) in enumerate(dets):
            arr[i].bin_lo, arr[i].bin_hi, arr[i].s0 = int(a), int(b), float(np.float32(s0))
        self.L.sdo_chtrack_update(C.byref(self.t), arr, C.c_uint(len(dets)))
        return self.keys()

    def keys(self):
        """(a, b, bits of S0, id, age, present, misses) of every live track, ascending (a, id)"""
        return [(r.a, r.b, int(np.float32(r.s0).view(np.uint32)), r.id, r.age, r.present, r.misses)
                for r in self.t.tr[:self.t.count]]

    @property
    def dropped(self):
        return self.t.dropped

    @property
    def next_id(self):
        return self.t.next_id
