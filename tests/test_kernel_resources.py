"""Registers and local memory of the 65536-point transform kernels, read from the built library.

k_fft65536 and k_chan_ifft16 are latency-bound between barriers, and the CTAs per SM that their registers allow
set their speed.  Both are compiled for 4 CTAs of 256 threads per SM (3 for the 4096-point inverse transform,
whose shared memory allows no more): 65536 / (256 x 4) = 64 registers per thread, 80 at 3 CTAs.  An edit that
makes ptxas spill to meet that bound, or a bound loosened so that one CTA fewer fits, fails here rather than as
a slower benchmark.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "sigdigger_b200", "libsigdigger_b200.so")
REGS_PER_SM = 65536
THREADS = 256

# kernel (demangled prefix of the instance) -> CTAs per SM it is compiled for
KERNELS = {
    "k_fft65536(": 4,
    "void k_chan_ifft16<(int)512>(": 4,
    "void k_chan_ifft16<(int)1024>(": 4,
    "void k_chan_ifft16<(int)2048>(": 4,
    "void k_chan_ifft16<(int)4096>(": 3,
}


def _tool(name):
    path = shutil.which(name)
    if path:
        return path
    for d in (os.path.dirname(shutil.which("nvcc") or ""), os.path.join(os.environ.get("CUDA_HOME", ""), "bin")):
        if d and os.path.exists(os.path.join(d, name)):
            return os.path.join(d, name)
    pytest.fail("%s not found: it ships with nvcc, which the build needs" % name)


@pytest.fixture(scope="module")
def usage():
    if not os.path.exists(LIB):
        pytest.fail("%s is not built: run __graft_entry__.build() first" % LIB)
    out = subprocess.run([_tool("cuobjdump"), "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    names = re.findall(r"^\s*Function (\S+):$", out, re.M)
    demangled = subprocess.run([_tool("cu++filt")], input="\n".join(names), capture_output=True, text=True,
                               check=True).stdout.splitlines()
    res = {}
    for mangled, name in zip(names, demangled):
        m = re.search(r"Function %s:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)" % re.escape(mangled), out)
        res[name] = dict(reg=int(m.group(1)), stack=int(m.group(2)), local=int(m.group(3)))
    return res


@pytest.mark.parametrize("kernel", sorted(KERNELS))
def test_transform_kernel_fits_its_occupancy(usage, kernel):
    found = {n: r for n, r in usage.items() if n.startswith(kernel)}
    assert len(found) == 1, "expected one instance of %s in the library, found %s" % (kernel, sorted(found))
    (name, r), = found.items()
    ctas = KERNELS[kernel]
    limit = REGS_PER_SM // (THREADS * ctas) // 8 * 8     # registers are allocated per thread in steps of 8
    assert r["reg"] <= limit, "%s: %d registers, more than the %d that %d CTAs per SM allow" % (name, r["reg"], limit, ctas)
    assert r["local"] == 0 and r["stack"] == 0, "%s spills: %d B local, %d B stack" % (name, r["local"], r["stack"])
