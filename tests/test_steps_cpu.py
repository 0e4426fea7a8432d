"""CPU: the select-form / compile-time variants of the per-sample steps that the inspector kernel's recurrence warps
run (clock_step_sel, costas_step_t<K, A>, agc_level_sel, the select form of SPEC M.2's atan2) are bit-identical to the
statement forms of sigdigger_b200/csrc/sdb_chain_steps.h, which the sigutils shim calls per sample and
tests/test_shim_cpu.py holds to the oracle.  tests/shim/steps_equiv.cu is compiled by nvcc for the HOST (the step
functions are __host__ __device__) and run here; no GPU involved."""
import os
import shutil
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc to compile the host-side check")
def test_select_forms_equal_statement_forms(tmp_path):
    src = os.path.join(HERE, "shim", "steps_equiv.cu")
    out = str(tmp_path / "steps_equiv")                   # the repository tree may be read-only
    r = subprocess.run(["nvcc", "-O2", "-fmad=false", "-Xcompiler", "-ffp-contract=off",
                        "-I" + os.path.join(HERE, "..", "include"), "-o", out, src], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    r = subprocess.run([out], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "mismatches 0" in r.stdout, r.stdout[-2000:]
