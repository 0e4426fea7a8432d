"""Registers and local memory of the FAC tab's kernels (fac_kernels.cu), read from the built library.

The transform kernels hold a 4096-point unit in shared memory and run the SPEC F.2 stages with four butterflies per
thread in registers; the statistics kernels keep a tile's scan in registers.  A spill would put those operands in local
memory, so an edit that makes ptxas spill fails here."""
from test_kernel_resources import usage  # noqa: F401  (the module fixture: cuobjdump -res-usage of the library)

NAMES = ["k_fac_plan(", "k_fac_small(", "void k_fac_cols<(int)0>(", "void k_fac_cols<(int)1>(",
         "void k_fac_rows<(int)0>(", "void k_fac_rows<(int)1>(", "k_fac_tilemax(", "k_fac_prefix(", "k_fac_tilepow(",
         "k_fac_fixup(", "k_fac_average(", "k_fac_tail("]


def test_fac_kernels_do_not_spill(usage):  # noqa: F811
    for prefix in NAMES:
        found = {n: r for n, r in usage.items() if n.startswith(prefix)}
        assert len(found) == 1, "expected one %s in the library, found %s" % (prefix, sorted(found))
        (name, r), = found.items()
        assert r["local"] == 0 and r["stack"] == 0, "%s spills: %d B local, %d B stack" % (name, r["local"], r["stack"])
        assert r["reg"] <= 255, "%s: %d registers" % (name, r["reg"])
