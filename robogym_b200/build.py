"""Build librobogym_b200.so in-tree for sm_90a (H100): `python -m robogym_b200.build [--force]`."""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "librobogym_b200.so")
DEPS = [os.path.join(SRC, f) for f in ("rg_engine.cu", "rg_cta.cu", "rg_arm.cu", "rg_groups.cu", "rg_kernel.inl", "rg_defs.h", "rg_dyn.inl", "rg_col.inl", "rg_sol.inl", "rg_step.inl", "rg_place.inl", "rg_goal.inl", "rg_obs.inl", "rg_arm.inl", "rg_groups.inl", "rg_host.h", "rg_derived_fields.h")]
DEPS += [os.path.join(HERE, "..", "include", f) for f in ("rg_model_fields.h", "robogym_b200.h")]


# the one-warp kernel (rg_engine.cu, with the C ABI), the one-environment-per-CTA kernel (rg_cta.cu) and the object groups'
# kernel (rg_groups.cu), linked into one library
SOURCES = ("rg_engine.cu", "rg_cta.cu", "rg_groups.cu")


def nvcc_cmd(extra=(), sources=("rg_engine.cu",), objects=()):
    nvcc = os.environ.get("NVCC", "nvcc")
    # -prec-div/-prec-sqrt=false: 2-ulp division / square root without the slow-path calls (measured +6 %, parity unchanged)
    return [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-prec-div=false", "-prec-sqrt=false", "-ftz=true",
            "-Xcompiler", "-fPIC", "-shared", *extra, "-o", OUT, *[os.path.join(SRC, s) for s in sources], *objects]


def arm_object(extra=()):
    """rg_arm.cu -> an object file in a temporary directory: the arm controller's kernels keep subnormals and round every
    operation as torch's float32 kernels do (no -ftz, IEEE division and square root, no FMA contraction)"""
    import tempfile

    obj = os.path.join(tempfile.mkdtemp(prefix="rg_arm_"), "rg_arm.o")
    subprocess.check_call([os.environ.get("NVCC", "nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
                           "-ftz=false", "-prec-div=true", "-prec-sqrt=true", "-fmad=false", "-Xcompiler", "-fPIC", *extra, "-c", "-o", obj,
                           os.path.join(SRC, "rg_arm.cu")])
    return obj


def _fresh():
    return os.path.exists(OUT) and all(os.path.getmtime(d) <= os.path.getmtime(OUT) for d in DEPS)


def build(force=False, verbose=False):
    if not force and _fresh():
        return OUT
    # several ranks of one job may get here together (torchrun): one compiles, the others wait and then find it fresh
    import fcntl

    with open(OUT + ".lock", "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if force or not _fresh():
                extra = ("-Xptxas", "-v") if verbose else ()
                obj = arm_object(extra)
                cmd = nvcc_cmd(extra, SOURCES, (obj,))
                tmp = OUT + ".tmp.%d" % os.getpid()
                cmd[cmd.index("-o") + 1] = tmp
                try:
                    subprocess.check_call(cmd)
                finally:
                    shutil.rmtree(os.path.dirname(obj), ignore_errors=True)
                os.replace(tmp, OUT)          # readers never see a half-written library
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)
    return OUT


def build_profile(level=1):
    """Same engine with per-stage clock64 counters in the RG_DBG dump (profiling only); level 2 breaks the Newton solve
    down instead of the collision stage."""
    out = os.path.join(HERE, "librobogym_b200_prof%s.so" % ("" if level == 1 else str(level)))
    obj = arm_object()
    cmd = nvcc_cmd(("-DRG_PROFILE=%d" % level,), SOURCES, (obj,))
    cmd[cmd.index("-o") + 1] = out
    subprocess.check_call(cmd)
    shutil.rmtree(os.path.dirname(obj), ignore_errors=True)
    return out


def build_variant(tag, defines):
    """Experimental build with extra -D flags (A/B measurements): librobogym_b200_<tag>.so."""
    out = os.path.join(HERE, "librobogym_b200_%s.so" % tag)
    flags = []
    for d in defines:                      # "-..." entries are raw nvcc flags ("+" stands for a space), the rest are -D macros
        flags += d.split() if d.startswith("-") else ["-D" + d]
    obj = arm_object()
    cmd = nvcc_cmd(tuple(flags), SOURCES, (obj,))
    cmd[cmd.index("-o") + 1] = out
    subprocess.check_call(cmd)
    shutil.rmtree(os.path.dirname(obj), ignore_errors=True)
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
    if "--profile" in sys.argv:
        print(build_profile())
        print(build_profile(2))
    for a in sys.argv[1:]:
        if a.startswith("--variant="):   # --variant=skew1:RG_SKEW=1
            tag, _, defs = a[len("--variant="):].partition(":")
            print(build_variant(tag, [d for d in defs.replace("+", " ").split(",") if d]))
