"""Registers and local memory of the Analog TV tab's kernel (k_tv_insp, tv_kernels.cu), read from the built library.

k_tv_insp keeps the processor's state and constants in lane 0's registers (92 registers when written) and the comb
delay line and the row being drawn in shared memory; a spill would put the per-sample recurrence's operands in local
memory, so an edit that makes ptxas spill, or grow past 128 registers (at least 16 one-warp CTAs per SM), fails here."""
from test_kernel_resources import usage  # noqa: F401  (the module fixture: cuobjdump -res-usage of the library)


def test_tv_insp_kernel_does_not_spill(usage):  # noqa: F811
    found = {n: r for n, r in usage.items() if n.startswith("k_tv_insp(")}
    assert len(found) == 1, "expected one k_tv_insp in the library, found %s" % sorted(found)
    (name, r), = found.items()
    assert r["local"] == 0 and r["stack"] == 0, "%s spills: %d B local, %d B stack" % (name, r["local"], r["stack"])
    assert r["reg"] <= 128, "%s: %d registers" % (name, r["reg"])
