"""Builds tests/shim/reference_tu.cpp (the reference's calling code, Qt removed) against the shim headers and
libraries; shared by the CPU and GPU shim tests."""
import ctypes as C
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_lib = None
_build_dir = None


def build_dir():
    """A private directory, removed at exit, for the shared objects the tests compile: the repository tree they run
    from may be read-only."""
    global _build_dir
    if _build_dir is None:
        _build_dir = tempfile.TemporaryDirectory(prefix="sdb-shim-tests-")
    return _build_dir.name


def reference_tu():
    global _lib
    if _lib is None:
        import sigdigger_b200
        sigdigger_b200.load_library()          # fails loudly if the native library was not built
        so = os.path.join(build_dir(), "libreftu.so")
        libdir = os.path.join(ROOT, "sigdigger_b200")
        subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "tests", "shim", "reference_tu.cpp"), "-o", so, "-L", libdir, "-lsuscan",
                        "-lsigutils", "-Wl,-rpath," + libdir, "-lpthread"], check=True)
        L = C.CDLL(so)
        L.tu_analyzer_session.restype = C.c_long
        L.tu_analyzer_session.argtypes = [C.c_void_p, C.c_size_t, C.c_uint, C.c_uint, C.c_size_t, C.c_double, C.c_double,
                                          C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
        L.tu_gardner_task.restype = C.c_long
        L.tu_gardner_task.argtypes = [C.c_void_p, C.c_size_t, C.c_float, C.c_float, C.c_void_p, C.c_size_t]
        L.tu_costas_task.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_float, C.c_float, C.c_int, C.c_int]
        L.tu_pll_task.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_float, C.c_int]
        L.tu_agc_task.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_float]
        L.tu_xlate_task.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_float, C.c_float, C.c_int]
        L.tu_lpf_task.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_float]
        L.tu_mq_samples.restype = C.c_long
        L.tu_mq_samples.argtypes = [C.c_void_p, C.c_ulong, C.c_uint, C.c_void_p, C.c_void_p]
        L.tu_status_message.argtypes = [C.c_int, C.c_char_p, C.c_char_p, C.c_size_t]
        L.tu_tv_worker.restype = C.c_long
        L.tu_tv_worker.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                   C.c_void_p]
        _lib = L
    return _lib


def oracle_loop(oracle, feed, x):
    import numpy as np
    ref = np.empty_like(x)
    v = x.view(np.float32).reshape(-1, 2)
    for i in range(len(x)):
        r = feed(oracle.Cpx(float(v[i, 0]), float(v[i, 1])))
        ref[i] = np.float32(r.re) + 1j * np.float32(r.im)
    return ref


def oracle_costas(oracle, x, kind, arm_bw, loop_bw):
    L = oracle.lib()
    c = oracle.Costas()
    assert L.sdo_costas_init(C.byref(c), kind, 0.0, arm_bw, 3, loop_bw) == 0
    return oracle_loop(oracle, lambda v: L.sdo_costas_feed(C.byref(c), v), x)


def oracle_pll(oracle, x, bw):
    L = oracle.lib()
    p = oracle.Pll()
    L.sdo_pll_init(C.byref(p), 0.0, bw)
    return oracle_loop(oracle, lambda v: L.sdo_pll_track(C.byref(p), v), x)


def oracle_agc(oracle, x, tau):
    L = oracle.lib()
    ap = oracle.AgcParams()
    L.sdo_agc_params_from_tau(C.byref(ap), tau, 2.0)
    ap.delay_line_size, ap.mag_history_size = 20, 20
    a = oracle.Agc()
    assert L.sdo_agc_init(C.byref(a), C.byref(ap)) == 0
    return oracle_loop(oracle, lambda v: L.sdo_agc_feed(C.byref(a), v), x)


def oracle_xlate(oracle, x, rel_freq, phase):
    import numpy as np
    L = oracle.lib()
    o = oracle.Ncqo()
    L.sdo_ncqo_init(C.byref(o), -rel_freq)
    L.sdo_ncqo_set_phase(C.byref(o), -phase)
    y = np.empty_like(x)
    L.sdo_carrier_xlate(oracle.ptr(x), oracle.ptr(y), len(x), C.byref(o))
    return y


def oracle_gardner_frequency(oracle, x, gain, bnor):
    """Gardner detector fed with x[n] conj(x[n-1]) (prev = 0 at the start), Tasks/WaveSampler.cpp:188-196; the
    product in binary32 steps, as the C++ operator computes it"""
    import numpy as np
    L = oracle.lib()
    cd = oracle.Clock()
    L.sdo_clock_init(C.byref(cd), gain, bnor)
    f = np.float32
    v = x.view(np.float32).reshape(-1, 2)
    pr, pi = f(0), f(0)
    ref = []
    o = oracle.Cpx(0, 0)
    for i in range(len(x)):
        a, b = f(v[i, 0]), f(v[i, 1])
        re = f(f(a * pr) + f(b * pi))
        im = f(f(b * pr) - f(a * pi))
        pr, pi = a, b
        if L.sdo_clock_feed(C.byref(cd), oracle.Cpx(float(re), float(im)), C.byref(o)):
            ref.append(np.float32(o.re) + 1j * np.float32(o.im))
    return np.array(ref, np.complex64)
