"""Registers and local memory of the channel tracker, k_chtrack, read from the built library.

One warp per stream keeps the ranges of its up to 256 tracks in registers (8 per lane) while it matches the
detections one by one.  A spill would put that inner loop's operands in local memory, so an edit that makes ptxas
spill fails here."""
import pytest

from test_kernel_resources import usage  # noqa: F401  (the module fixture: cuobjdump -res-usage of the library)


def test_chtrack_does_not_spill(usage):  # noqa: F811
    found = {n: r for n, r in usage.items() if n.startswith("k_chtrack(")}
    assert len(found) == 1, "expected one k_chtrack in the library, found %s" % sorted(found)
    (name, r), = found.items()
    assert r["local"] == 0 and r["stack"] == 0, "%s spills: %d B local, %d B stack" % (name, r["local"], r["stack"])
    assert r["reg"] <= 64, "%s: %d registers" % (name, r["reg"])
