"""ctypes binding of the source-decimation oracle (oracle/decimate.c, SPEC L in oracle/SPEC_L.md), built by
oracle/decimate.mk as oracle/_build/libsddecim.so over the parity oracle.  TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib

LIB_PATH = os.path.join(oracle_lib.ORACLE_DIR, "_build", "libsddecim.so")
FORMATS = {"f32": 0, "u8": 1, "s8": 2, "s16": 3}
_lib = None


class DecimateState(C.Structure):
    """sdo_decimate"""
    _fields_ = [("D", C.c_uint), ("n", C.c_uint), ("h", C.POINTER(C.c_float)), ("hist", C.c_void_p),
                ("phase", C.c_uint)]


def lib():
    global _lib
    if _lib is None:
        oracle_lib.lib()                       # the parity oracle the decimator links against, built first
        subprocess.run(["make", "-C", oracle_lib.ORACLE_DIR, "-f", "decimate.mk"], check=True, capture_output=True)
        L = C.CDLL(LIB_PATH)
        L.sdo_decimate_init.argtypes = [C.c_void_p, C.c_uint]
        L.sdo_decimate_free.argtypes = [C.c_void_p]
        L.sdo_decimate_reset.argtypes = [C.c_void_p]
        L.sdo_decimate_feed.restype = C.c_size_t
        L.sdo_decimate_feed.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_size_t, C.c_void_p]
        _lib = L
    return _lib


class Decimator:
    """SPEC L source decimator.  feed() takes complex64 (f32) or interleaved I,Q integer arrays (u8 / s8 / s16) and
    returns the complex64 outputs of that feed."""

    def __init__(self, D, fmt="f32"):
        self.L = lib()
        self.D, self.fmt = D, FORMATS[fmt] if isinstance(fmt, str) else int(fmt)
        self.s = DecimateState()
        if self.L.sdo_decimate_init(C.byref(self.s), D):
            raise ValueError("decimation out of range: %d" % D)

    @property
    def taps(self):
        return np.ctypeslib.as_array(self.s.h, shape=(self.s.n,)).copy()

    def feed(self, x):
        x = np.ascontiguousarray(x)
        m = len(x) if self.fmt == 0 else len(x) // 2
        y = np.empty(m // self.D + 1, np.complex64)
        k = self.L.sdo_decimate_feed(C.byref(self.s), x.ctypes.data_as(C.c_void_p), self.fmt, m,
                                     y.ctypes.data_as(C.c_void_p))
        return y[:k]

    def reset(self):
        self.L.sdo_decimate_reset(C.byref(self.s))

    def close(self):
        if self.s.h:
            self.L.sdo_decimate_free(C.byref(self.s))

    __del__ = close
