"""Registers, stack frame and spills of the step kernel's builds, function by function: `ptxas -v` on sm_90a with the flags of
robogym_b200/build.py.  The kernel is instantiated per warp count (rg_step_kernel<12>: 168 registers, <13>: 128), and a
function that fits in one build may spill in the other; the narrow phase's loop (rg_mpr_batch) must spill in neither.
Compiles to a temporary directory (about 30 s on one core); needs nvcc, no GPU.

Development tool: python tools/spill_report.py"""
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _name(mangled):
    """rg_step_kernel<13> / rg_mpr_batch from the Itanium-mangled names ptxas prints"""
    m = re.match(r"_Z(\d+)", mangled)
    if not m:
        return mangled
    name = mangled[m.end():m.end() + int(m.group(1))]
    t = re.match(r"ILi(\d+)EE", mangled[m.end() + int(m.group(1)):])
    return "%s<%s>" % (name, t.group(1)) if t else name


def parse(text):
    """{kernel: {"registers": n, "functions": {function: (stack bytes, spill store bytes, spill load bytes)}}} for every
    rg_step_kernel instantiation in a `ptxas -v` report; the kernel's own frame is listed under its own name"""
    out, kernel, func = {}, None, None
    for line in text.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            kernel = _name(m.group(1)) if m.group(1).startswith("_Z14rg_step_kernel") else None
            if kernel:
                out[kernel] = {"registers": None, "functions": {}}
            continue
        if kernel is None:
            continue
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            func = _name(m.group(1))
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and func:
            out[kernel]["functions"][func] = tuple(int(x) for x in m.groups())
            func = None
            continue
        m = re.search(r"Used (\d+) registers", line)
        if m:
            out[kernel]["registers"] = int(m.group(1))
    return out


def report():
    from robogym_b200 import build

    with tempfile.TemporaryDirectory() as d:
        cmd = build.nvcc_cmd(("-Xptxas", "-v", "-cubin"))
        cmd[cmd.index("-o") + 1] = os.path.join(d, "rg_engine.cubin")
        r = subprocess.run(cmd, cwd=d, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + r.stderr)
    return parse(r.stdout + r.stderr)


def main():
    rep = report()
    kernels = sorted(rep)
    print("%-24s" % "function" + "".join("%28s" % ("%s, %d regs" % (k, rep[k]["registers"])) for k in kernels))
    print("%-24s" % "" + "".join("%28s" % "stack / spill st / spill ld" for _ in kernels))
    funcs = sorted(set().union(*(rep[k]["functions"] for k in kernels)), key=lambda f: (not f.startswith("rg_step_kernel"), f))
    for f in funcs:
        cells = [rep[k]["functions"].get(f) for k in kernels]
        print("%-24s" % f + "".join("%28s" % ("%d / %d / %d" % c if c else "-") for c in cells))


if __name__ == "__main__":
    main()
