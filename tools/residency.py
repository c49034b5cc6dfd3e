"""Shared-memory budget of the step kernel on an H100 for every asset at the capacities bench.py runs it with: the per-environment
scratch (4 * RgLayout.total, rg_make_layout), the per-CTA fixed part and the environments per SM that fit (rg_batch_size in
rg_engine.cu).  Host-side only: the layout comes from the CPU emulation build, which compiles the same rg_make_layout.

Development tool: python tools/residency.py"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))

OPTIN = 232448          # H100: cudaDevAttrMaxSharedMemoryPerBlockOptin
STATIC = 128            # rg_step_kernel's static shared memory (nvcc -Xptxas -v)
MODEL_VIEW = 1024       # RG_MODEL_DEV_BYTES
MAX_WARPS = 13          # RG_MAX_WARPS
# (contacts, rows, dofs per contact) as bench.py's CONFIGS pass them (0 = engine default 32 / 64 / 16)
CAPS = {"dactyl_locked": (0, 0, 0), "dactyl_full_perpendicular": (96, 288, 32), "rearrange_blocks5": (64, 128, 16),
        "rearrange_blocks5_tcp": (64, 160, 16), "rearrange_solver_arm": (0, 0, 0), "rearrange_ycb8": (64, 128, 16),
        "rearrange_ycb8_tcp": (64, 160, 16)}


def budget(asset, caps):
    import pyemu
    from robogym_b200 import modelblob

    blob = open(os.path.join(ROOT, "robogym_b200", "assets", asset + ".rgm"), "rb").read()
    m = modelblob.unpack(blob)
    e = pyemu.EmuBatch(blob, {k: m[k] for k in modelblob.DIMS}, 1, *caps)
    scratch = 4 * pyemu.lib().rge_scratch_floats(e.h)
    fixed = MODEL_VIEW + ((pyemu.lib().rge_small_bytes(e.h) + 127) & ~127) + 64
    warps = min((OPTIN - STATIC - fixed) // scratch, MAX_WARPS)
    return dict(asset=asset, caps=caps, scratch_bytes_per_env=scratch, fixed_bytes=fixed, warps_per_cta=warps,
                bytes_to_next_warp=(warps + 1) * scratch + fixed - (OPTIN - STATIC) if warps < MAX_WARPS else None)


def main():
    assets = sorted(f[:-4] for f in os.listdir(os.path.join(ROOT, "robogym_b200", "assets")) if f.endswith(".rgm"))
    for a in assets:
        print(json.dumps(budget(a, CAPS.get(a, (0, 0, 0)))))


if __name__ == "__main__":
    main()
