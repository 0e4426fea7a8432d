"""ctypes binding of the CPU oracle's Analog TV tab (sdo_tvinsp_*, oracle/tvinsp.c, SPEC_TI.md), built by
oracle/tvinsp.mk as oracle/_build/libsdtvinsp.so.  TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib

LIB_PATH = os.path.join(oracle_lib.ORACLE_DIR, "_build", "libsdtvinsp.so")
_lib = None
CLASSES = {"psk": 0, "fsk": 1, "ask": 2}


class Status(C.Structure):
    """sdo_tvinsp_status (the layout of sdb_tv_status)"""
    _fields_ = [("frames", C.c_uint64), ("posted_no", C.c_uint64), ("completed", C.c_uint32), ("width", C.c_uint32),
                ("height", C.c_uint32), ("line_len", C.c_float), ("hsync_len", C.c_float), ("agc_gain", C.c_float)]

    def key(self):
        """(frames, posted_no, completed, width, height, bits of line_len, hsync_len, agc_gain)"""
        b = lambda x: int(np.float32(x).view(np.uint32))     # noqa: E731
        return (self.frames, self.posted_no, self.completed, self.width, self.height, b(self.line_len),
                b(self.hsync_len), b(self.agc_gain))


class _Tab(C.Structure):
    _fields_ = [("tv", C.c_void_p), ("mode", C.c_int), ("k", C.c_float), ("dc", C.c_float),
                ("posted", C.POINTER(C.c_float)), ("st", Status)]


def lib():
    global _lib
    if _lib is None:
        subprocess.run(["make", "-C", oracle_lib.ORACLE_DIR, "-f", "tvinsp.mk"], check=True, capture_output=True)
        _lib = C.CDLL(LIB_PATH)
        _lib.sdo_tvinsp_init.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_float]
        _lib.sdo_tvinsp_free.argtypes = [C.c_void_p]
        _lib.sdo_tvinsp_set_params.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_float]
        _lib.sdo_tvinsp_feed.argtypes = [C.c_void_p, C.c_void_p, C.c_uint]
    return _lib


def params(p):
    """a parameter block (oracle_lib.TvParams, sigdigger_b200.TvParams or a dict of its fields) as oracle_lib.TvParams"""
    q = oracle_lib.TvParams()
    for name, _ in oracle_lib.TvParams._fields_:
        setattr(q, name, p[name] if isinstance(p, dict) else getattr(p, name))
    return q


class Tab:
    """One Analog TV tab of the oracle (sdo_tvinsp)"""

    def __init__(self, cls, p, invert=False, dc=0.0):
        self.L_ = lib()
        self.t = _Tab()
        if self.L_.sdo_tvinsp_init(C.byref(self.t), CLASSES[cls], C.byref(params(p)), int(invert), dc):
            raise ValueError("sdo_tvinsp_init refused %s" % cls)

    def __del__(self):
        if getattr(self, "t", None) is not None and self.t.tv:
            self.L_.sdo_tvinsp_free(C.byref(self.t))

    def set_params(self, p, invert=False, dc=0.0):
        """True when taken (TI.4)"""
        return self.L_.sdo_tvinsp_set_params(C.byref(self.t), C.byref(params(p)), int(invert), dc) == 0

    def feed(self, x):
        x = np.ascontiguousarray(x, np.complex64)
        self.L_.sdo_tvinsp_feed(C.byref(self.t), x.ctypes.data_as(C.c_void_p), C.c_uint(len(x)))

    @property
    def posted(self):
        s = self.t.st
        return np.ctypeslib.as_array(self.t.posted, shape=(s.height, s.width)).copy()

    @property
    def status(self):
        s = self.t.st
        return Status(s.frames, s.posted_no, s.completed, s.width, s.height, s.line_len, s.hsync_len, s.agc_gain)
