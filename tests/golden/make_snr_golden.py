"""Writes tests/golden/ref_snr.npz: the sigma / SNR trajectory of Misc/SNREstimator.cpp, compiled from the reference
into oracle/_ref/libsdref.so (`make -C oracle ref`), driven as the inspector's SNR meter drives it with the GUI's
toggle values (sigma 1, alpha 1 / K) over the histograms of the oracle meter (oracle/snr.c) on seeded noisy PSK
symbols.  TEST INFRASTRUCTURE ONLY: run by hand where the reference is built; tests/test_snr_ref.py reads the file."""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import snr_oracle  # noqa: E402

CASES = ((1, 256), (2, 256), (3, 400))
FEEDS = 24


def symbols(bps, seed):
    """FEEDS feeds of noisy 2^bps-PSK soft symbols, 500 to 1500 per feed"""
    rng = np.random.default_rng(seed)
    K = 1 << bps
    out = []
    for _ in range(FEEDS):
        n = int(rng.integers(500, 1500))
        k = rng.integers(0, K, n)
        x = np.exp(1j * 2 * np.pi * (k + 0.5) / K) + 0.2 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
        out.append(x.astype(np.complex64))
    return out


def meter_histories(bps, L, seed):
    m = snr_oracle.Meter("psk", L, bps, 1.0, 1.0 / (1 << bps))
    hs = []
    for x in symbols(bps, seed):
        m.feed(x)
        hs.append(m.h)
    return np.array(hs, np.uint32)


def main():
    lib = C.CDLL(os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle", "_ref", "libsdref.so"))
    lib.ref_snr_estimator.argtypes = [C.c_uint, C.c_float, C.c_float, C.c_void_p, C.c_uint, C.c_uint, C.c_void_p,
                                      C.c_void_p, C.c_void_p]
    out = {}
    for bps, L in CASES:
        hs = np.ascontiguousarray(meter_histories(bps, L, 40 + bps))
        sig, snr, model = np.zeros(FEEDS, np.float32), np.zeros(FEEDS, np.float32), np.zeros(L, np.float32)
        assert lib.ref_snr_estimator(bps, C.c_float(1.0 / (1 << bps)), C.c_float(1.0), hs.ctypes.data, L, FEEDS,
                                     sig.ctypes.data, snr.ctypes.data, model.ctypes.data) == L
        out["hist_%d_%d" % (bps, L)] = hs
        out["ref_%d_%d" % (bps, L)] = np.concatenate([sig, snr, model])
    np.savez_compressed(os.path.join(HERE, "ref_snr.npz"), **out)


if __name__ == "__main__":
    main()
