"""Registers and stack of the inspector kernel's class instances, read from the built library.

k_inspectors has one instance per inspector class (psk, fsk, ask, audio, raw), each launched over the CTAs of its own
class.  Every instance is compiled for 2 CTAs of 384 threads per SM: 65536 / (384 x 2) = 80 registers per thread.
ptxas keeps the psk, fsk, ask and audio instances within that bound with a 40-byte stack frame of spilled values
(the parent's single kernel spilled 132 B and reloaded 320 B); the raw instance does not spill.  The allowance below
is that frame: an edit that makes an instance spill more, or asks for more registers than 2 CTAs per SM allow, fails
here rather than as a slower benchmark.
"""
import pytest

from test_kernel_resources import REGS_PER_SM, usage  # noqa: F401  (usage is a fixture)

THREADS = 384
CTAS = 2
# instance (SDB_INSP_* class) -> largest stack frame in bytes
STACK_ALLOWANCE = {0: 40, 1: 40, 2: 40, 3: 40, 4: 0}


@pytest.mark.parametrize("cls", sorted(STACK_ALLOWANCE))
def test_inspector_instance_fits_two_ctas(usage, cls):  # noqa: F811
    prefix = "void k_inspectors<(int)%d>(" % cls
    found = {n: r for n, r in usage.items() if n.startswith(prefix)}
    assert len(found) == 1, "expected one instance %s in the library, found %s" % (prefix, sorted(found))
    (name, r), = found.items()
    limit = REGS_PER_SM // (THREADS * CTAS) // 8 * 8
    assert r["reg"] <= limit, "%s: %d registers, more than the %d that %d CTAs per SM allow" % (name, r["reg"], limit, CTAS)
    assert r["local"] == 0, "%s: %d B of local memory" % (name, r["local"])
    assert r["stack"] <= STACK_ALLOWANCE[cls], "%s spills: %d B stack, allowance %d B" % (
        name, r["stack"], STACK_ALLOWANCE[cls])


def test_no_other_inspector_kernel(usage):  # noqa: F811
    names = sorted(n for n in usage if "k_inspectors" in n)
    assert len(names) == len(STACK_ALLOWANCE), names
