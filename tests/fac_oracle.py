"""ctypes binding of the CPU oracle's FAC tab (sdo_fac_*, oracle/fac.c, SPEC_FC.md), built by oracle/fac.mk as
oracle/_build/libsdfac.so.  TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib

LIB_PATH = os.path.join(oracle_lib.ORACLE_DIR, "_build", "libsdfac.so")
_lib = None


class Status(C.Structure):
    _fields_ = [("blocks", C.c_uint), ("peak_lag", C.c_uint), ("max", C.c_float), ("min", C.c_float),
                ("sigmas", C.c_float), ("marker", C.c_int)]

    def key(self):
        """(blocks, peak_lag, bits of max, min, sigmas, marker)"""
        b = lambda x: int(np.float32(x).view(np.uint32))     # noqa: E731
        return (self.blocks, self.peak_lag, b(self.max), b(self.min), b(self.sigmas), self.marker)


class Acc(C.Structure):
    _fields_ = [("blocks", C.c_uint), ("pos", C.c_uint), ("count", C.c_uint), ("local", C.c_float),
                ("power", C.c_float)]


class _Plan(C.Structure):
    _fields_ = [("raw", C.c_char * 256)]      # sdo_spec_plan: opaque here, sized generously


class OFac(C.Structure):
    _fields_ = [("L", C.c_uint), ("lo", C.c_uint), ("hi", C.c_uint), ("alpha", C.c_float), ("sigma", C.c_double),
                ("p", C.c_uint), ("max", C.c_float), ("min", C.c_float), ("blk", C.c_void_p),
                ("fac", C.POINTER(C.c_float)), ("v", C.POINTER(C.c_float)), ("plan", _Plan)]


def lib():
    global _lib
    if _lib is None:
        subprocess.run(["make", "-C", oracle_lib.ORACLE_DIR, "-f", "fac.mk"], check=True, capture_output=True)
        _lib = C.CDLL(LIB_PATH)
        _lib.sdo_fac_init.argtypes = [C.c_void_p, C.c_uint, C.c_float, C.c_uint, C.c_uint, C.c_double]
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


class Fac:
    """One FAC chain of the oracle (sdo_fac)."""

    def __init__(self, L, alpha=1.0, lags=None, sigma=5.0):
        self.L_ = lib()
        self.f = OFac()
        lo, hi = lags if lags is not None else (0, 0)
        if self.L_.sdo_fac_init(C.byref(self.f), L, alpha, lo, hi, sigma):
            raise ValueError("sdo_fac_init refused L=%d lags=%s" % (L, lags))

    def __del__(self):
        if getattr(self, "f", None) is not None and self.f.blk:
            self.L_.sdo_fac_free(C.byref(self.f))

    @property
    def L(self):
        return self.f.L

    def feed(self, x):
        x = np.ascontiguousarray(x, np.complex64)
        st = Status()
        self.L_.sdo_fac_feed(C.byref(self.f), _ptr(x), C.c_uint(len(x)), C.byref(st))
        return st

    def magnitude(self, block, twice=False):
        block = np.ascontiguousarray(block, np.complex64)
        assert len(block) == self.f.L
        v = np.empty(self.f.L // 2, np.float32)
        self.L_.sdo_fac_magnitude(C.byref(self.f), _ptr(block), _ptr(v), C.c_int(1 if twice else 0))
        return v

    def update_feed(self, vs):
        """FC.2 - FC.4 on given v arrays, one per block, as one feed"""
        a = Acc()
        self.L_.sdo_fac_acc_init(C.byref(a))
        for v in vs:
            v = np.ascontiguousarray(v, np.float32)
            self.L_.sdo_fac_update(C.byref(self.f), C.byref(a), _ptr(v))
        st = Status()
        self.L_.sdo_fac_finish(C.byref(self.f), C.byref(a), C.byref(st))
        return st

    @property
    def fac(self):
        return np.ctypeslib.as_array(self.f.fac, shape=(self.f.L // 2,)).copy()

    @property
    def p(self):
        return self.f.p
