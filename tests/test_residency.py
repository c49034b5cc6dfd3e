"""Shared-memory residency of the step kernel on an H100, from the CPU emulation build's layout (the same rg_make_layout)."""
import residency


def test_locked_fits_thirteen_environments_per_sm():
    """dactyl/locked's 8192-environment launch takes 5 rounds of 132 x 13 only if 13 scratch areas fit next to the staged model"""
    assert residency.budget("dactyl_locked", (0, 0, 0))["warps_per_cta"] == 13


def test_bench_configs_keep_their_residency():
    """environments per SM of the other bench configs at their capacities: none below what the previous layout fitted"""
    before = {"dactyl_full_perpendicular": 1, "rearrange_blocks5": 8, "rearrange_blocks5_tcp": 8, "rearrange_solver_arm": 13,
              "rearrange_ycb8": 5, "rearrange_ycb8_tcp": 5}
    for asset, warps in before.items():
        assert residency.budget(asset, residency.CAPS[asset])["warps_per_cta"] >= warps, asset
