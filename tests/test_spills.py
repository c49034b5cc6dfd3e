"""The narrow phase's loop keeps its state in registers in both builds of the step kernel (ptxas -v, sm_90a; needs nvcc only)."""
import os
import shutil

import pytest

import spill_report


@pytest.mark.skipif(shutil.which(os.environ.get("NVCC", "nvcc")) is None, reason="needs nvcc")
def test_mpr_batch_does_not_spill():
    """rg_mpr_batch runs once per MPR iteration of every pair in flight: a spill there is paid on every trip, and under the
    13-warp build's 128-register cap it goes to local memory that the L1 beside 231 KB of shared memory cannot hold"""
    rep = spill_report.report()
    assert "rg_step_kernel<13>" in rep
    for kernel, r in rep.items():
        stack, st, ld = r["functions"]["rg_mpr_batch"]
        assert (st, ld) == (0, 0), "%s: rg_mpr_batch spills %d B stores / %d B loads" % (kernel, st, ld)
