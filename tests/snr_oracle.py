"""ctypes binding of the CPU oracle's SNR meter (sdo_snrm_*, oracle/snr.c, SPEC_SN.md), built by oracle/snr.mk as
oracle/_build/libsdsnr.so.  TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib

LIB_PATH = os.path.join(oracle_lib.ORACLE_DIR, "_build", "libsdsnr.so")
_lib = None


class Status(C.Structure):
    _fields_ = [("counted", C.c_ulonglong), ("steps", C.c_uint), ("stepped", C.c_uint), ("sigma", C.c_float),
                ("snr", C.c_float), ("delta", C.c_float)]

    def key(self):
        """(counted, steps, stepped, bits of sigma, snr, delta)"""
        b = lambda x: int(np.float32(x).view(np.uint32))     # noqa: E731
        return (self.counted, self.steps, self.stepped, b(self.sigma), b(self.snr), b(self.delta))


class _Est(C.Structure):
    _fields_ = [("sigma", C.c_float), ("alpha", C.c_float), ("hx", C.c_float), ("delta", C.c_float),
                ("bps", C.c_uint), ("intervals", C.c_uint), ("length", C.c_uint),
                ("gaussian", C.c_void_p), ("hi", C.c_void_p), ("htilde", C.c_void_p)]


class OMeter(C.Structure):
    _fields_ = [("L", C.c_uint), ("K", C.c_uint), ("bps", C.c_uint), ("mode", C.c_int),
                ("h", C.POINTER(C.c_uint)), ("model", C.POINTER(C.c_float)), ("est", _Est), ("st", Status)]


def lib():
    global _lib
    if _lib is None:
        subprocess.run(["make", "-C", oracle_lib.ORACLE_DIR, "-f", "snr.mk"], check=True, capture_output=True)
        _lib = C.CDLL(LIB_PATH)
        _lib.sdo_snrm_init.argtypes = [C.c_void_p, C.c_int, C.c_uint, C.c_uint, C.c_float, C.c_float]
        _lib.sdo_snrm_bin.argtypes = [C.c_int, C.c_uint, oracle_lib.Cpx]
        _lib.sdo_snrm_bin.restype = C.c_uint
        _lib.sdo_snrm_feed.argtypes = [C.c_void_p, C.c_void_p, C.c_uint]
        _lib.sdo_snrm_reset.argtypes = [C.c_void_p, C.c_float]
        _lib.sdo_snrm_replan.argtypes = [C.c_void_p, C.c_int, C.c_uint, C.c_float]
    return _lib


CLASSES = {"psk": 0, "fsk": 1, "ask": 2}


def bin_of(mode, L, x):
    """SN.1 of one symbol: its bin, or -1 when it is not counted"""
    b = lib().sdo_snrm_bin(mode, L, oracle_lib.Cpx(float(np.float32(x.real)), float(np.float32(x.imag))))
    return -1 if b == L else int(b)


class Meter:
    """One meter of the oracle (sdo_snrm)"""

    def __init__(self, cls, L, bps, sigma, alpha):
        self.L_ = lib()
        self.m = OMeter()
        if self.L_.sdo_snrm_init(C.byref(self.m), CLASSES[cls], L, bps, sigma, alpha):
            raise ValueError("sdo_snrm_init refused %s L=%d" % (cls, L))

    def __del__(self):
        if getattr(self, "m", None) is not None and self.m.h:
            self.L_.sdo_snrm_free(C.byref(self.m))

    def feed(self, x):
        x = np.ascontiguousarray(x, np.complex64)
        self.L_.sdo_snrm_feed(C.byref(self.m), x.ctypes.data_as(C.c_void_p), C.c_uint(len(x)))

    def reset(self, sigma):
        self.L_.sdo_snrm_reset(C.byref(self.m), sigma)

    def replan(self, same_cfg, bps, alpha):
        self.L_.sdo_snrm_replan(C.byref(self.m), int(same_cfg), bps, alpha)

    @property
    def h(self):
        return np.ctypeslib.as_array(self.m.h, shape=(self.m.L,)).copy()

    def seed(self, h):
        """set h (the 2^31 halving is reached from a histogram near the limit)"""
        np.ctypeslib.as_array(self.m.h, shape=(self.m.L,))[:] = h

    @property
    def model(self):
        return np.ctypeslib.as_array(self.m.model, shape=(self.m.L,)).copy()

    @property
    def status(self):
        s = self.m.st
        return Status(s.counted, s.steps, s.stepped, s.sigma, s.snr, s.delta)
