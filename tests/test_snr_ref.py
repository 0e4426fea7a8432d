"""The oracle's SNR meter (oracle/snr.c) against Misc/SNREstimator.cpp compiled from the reference, driven with the
GUI's toggle values (sigma 1, alpha 1 / K): the same sigma and SNR trajectory over the meter's histograms, to the
bound tests/test_ref.py holds the Y.7 restatement to (libm's exp against SPEC M's)."""
import os
import sys

import numpy as np
import pytest

import snr_oracle

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_snr_golden as G  # noqa: E402

REF = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_snr.npz")


@pytest.mark.parametrize("bps,L", G.CASES)
def test_meter_tracks_the_compiled_estimator(bps, L):
    ref = np.load(REF)
    hist, r = ref["hist_%d_%d" % (bps, L)], ref["ref_%d_%d" % (bps, L)]
    sig, snr, model = r[:G.FEEDS], r[G.FEEDS:2 * G.FEEDS], r[2 * G.FEEDS:]
    m = snr_oracle.Meter("psk", L, bps, 1.0, 1.0 / (1 << bps))
    for f, x in enumerate(G.symbols(bps, 40 + bps)):
        m.feed(x)
        assert np.array_equal(m.h, hist[f]), f                 # the histories the reference was fed
        st = m.status
        assert abs(st.sigma - sig[f]) <= 1e-4 * abs(sig[f]), (bps, f, st.sigma, sig[f])
        assert abs(st.snr - snr[f]) <= 1e-4 * abs(snr[f]), (bps, f, st.snr, snr[f])
    assert np.abs(m.model - model).max() < 1e-4
