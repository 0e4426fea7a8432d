"""ctypes binding of the power-inspector oracle (oracle/power.c, SPEC PW in oracle/SPEC_PW.md), built by
oracle/power.mk as oracle/_build/libsdpower.so.  TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib

LIB_PATH = os.path.join(oracle_lib.ORACLE_DIR, "_build", "libsdpower.so")
_lib = None


class PowerState(C.Structure):
    """sdo_power"""
    _fields_ = [("M", C.c_uint64), ("acc", C.c_double), ("c", C.c_double), ("n", C.c_uint64)]


def lib():
    global _lib
    if _lib is None:
        subprocess.run(["make", "-C", oracle_lib.ORACLE_DIR, "-f", "power.mk"], check=True, capture_output=True)
        L = C.CDLL(LIB_PATH)
        L.sdo_power_init.argtypes = [C.c_void_p, C.c_uint64]
        L.sdo_power_feed.restype = C.c_size_t
        L.sdo_power_feed.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
        _lib = L
    return _lib


class Power:
    """SPEC PW integrator of one channel: feed() takes complex64 channel samples and returns the float32 means that
    feed completed; the partial group carries to the next feed."""

    def __init__(self, M):
        self.L = lib()
        self.s = PowerState()
        self.L.sdo_power_init(C.byref(self.s), M)

    def feed(self, x):
        x = np.ascontiguousarray(x, dtype=np.complex64)
        out = np.empty(len(x), np.float32)
        k = self.L.sdo_power_feed(C.byref(self.s), x.ctypes.data_as(C.c_void_p), len(x),
                                  out.ctypes.data_as(C.c_void_p))
        return out[:k]


def gui_raw_mode(x, max_samples, state=None):
    """The RMS tab's raw-mode integration, transcribed line by line (Default/RMSInspector/RMSInspector.cpp:538-560
    samplesMessage and :327-338 checkMaxSamples): qreal is a Python float (binary64); SU_C_REAL(x * SU_C_CONJ(x))
    with std::complex<float> is re re - im (-im), two rounded float32 products and one rounded float32 sum.
    state = [kahanAcc, kahanC, count] carries across calls.  -> the float32 means pushed."""
    if state is None:
        state = [0.0, 0.0, 0]
    x = np.asarray(x, np.complex64)
    re, im = x.real.astype(np.float32), x.imag.astype(np.float32)
    inputs = (re * re + im * im).astype(np.float32).tolist()
    acc, c, count = state
    out = []
    for inp in inputs:
        y = inp - c
        t = acc + y
        c = (t - acc) - y
        acc = t
        count += 1
        if count >= max_samples:                       # checkMaxSamples
            if count > 0:
                out.append(acc / float(count))
            c = acc = 0.0
            count = 0
    state[:] = [acc, c, count]
    return np.array(out, np.float32)
