"""Registers and local memory of the SNR meter's kernel (k_snr, snr_kernels.cu), read from the built library.

k_snr holds the histogram and the Y.7 work arrays in shared memory and the bin arithmetic in registers; a spill would
put those operands in local memory, so an edit that makes ptxas spill fails here."""
from test_kernel_resources import usage  # noqa: F401  (the module fixture: cuobjdump -res-usage of the library)


def test_snr_kernel_does_not_spill(usage):  # noqa: F811
    found = {n: r for n, r in usage.items() if n.startswith("k_snr(")}
    assert len(found) == 1, "expected one k_snr in the library, found %s" % sorted(found)
    (name, r), = found.items()
    assert r["local"] == 0 and r["stack"] == 0, "%s spills: %d B local, %d B stack" % (name, r["local"], r["stack"])
    assert r["reg"] <= 255, "%s: %d registers" % (name, r["reg"])
