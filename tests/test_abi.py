"""The C ABI of include/robogym_b200.h: the library exports every function it declares, and the Python binding
(robogym_b200.engine) declares the same functions, struct layouts and constants (no compute calls, no GPU)."""
import ctypes
import os
import re
import subprocess

import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
# the header's structs and their ctypes mirrors in robogym_b200.engine
MIRRORS = {"rg_goal_in": "GoalIn", "rg_goal_out": "GoalOut", "rg_obs_in": "ObsIn", "rg_obs_out": "ObsOut"}


def header():
    """include/robogym_b200.h without its comments"""
    return re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "robogym_b200.h")).read(), flags=re.S)


def declared_functions():
    """{name: (return type, [parameter declarations])} of every function the header declares"""
    out = {}
    for ret, name, params in re.findall(r"^[ \t]*((?:const[ \t]+)?\w+[ \t]*\**)[ \t]*\b(rg_\w+)[ \t]*\(([^()]*)\)[ \t]*;", header(), re.M):
        params = [" ".join(p.split()) for p in params.split(",")]
        out[name] = (ret.strip(), [] if params == ["void"] else params)
    return out


def ctype_matches(decl, ct):
    """whether the ctypes type `ct` passes the C type of `decl` (a return type, or a parameter's type and name): a pointer or
    array as c_void_p or POINTER(...), a const char* as c_char_p, void as None and a scalar as its own ctypes type"""
    if re.fullmatch(r"(const )?char ?\* ?\w*", decl):
        return ct is ctypes.c_char_p
    if "*" in decl or "[" in decl:
        return ct is ctypes.c_void_p or (isinstance(ct, type) and issubclass(ct, ctypes._Pointer))
    scalar = {"void": None, "int": ctypes.c_int, "size_t": ctypes.c_size_t, "double": ctypes.c_double, "uint32_t": ctypes.c_uint32}
    return ct is scalar[decl.split()[0]]


def test_header_declares_the_boundary():
    fns = declared_functions()
    for f in ("rg_model_load", "rg_batch_create", "rg_batch_bind", "rg_step", "rg_forward", "rg_reset", "rg_last_error"):
        assert f in fns


def test_signature_table_matches_the_header():
    """engine.SIGNATURES covers exactly the functions the header declares, each with its arity and, for the return value and
    every parameter, a ctypes type of the declared kind."""
    from robogym_b200 import engine

    decl = declared_functions()
    assert sorted(engine.SIGNATURES) == sorted(decl)
    for name, (ret, params) in decl.items():
        restype, argtypes = engine.SIGNATURES[name]
        assert len(argtypes) == len(params), f"{name}: {len(argtypes)} argtypes for {len(params)} parameters"
        assert ctype_matches(ret, restype), f"{name}: restype {restype} for {ret}"
        for i, (p, ct) in enumerate(zip(params, argtypes)):
            assert ctype_matches(p, ct), f"{name}: argument {i} ({p}) declared as {ct}"


def test_struct_mirrors_and_constants_match_the_header(tmp_path):
    """A C program built from the header by the host compiler prints sizeof of every mirrored struct, offsetof and sizeof of
    each field the ctypes mirrors declare, every rg_field enumerator and RG_MAX_CONTACTS; ctypes and engine's constants
    must give the same numbers."""
    from robogym_b200 import engine

    lines, expect = [], {}
    for cname, pyname in MIRRORS.items():
        mirror = getattr(engine, pyname)
        lines.append(f'printf("sizeof {cname} %zu\\n", sizeof({cname}));')
        expect[f"sizeof {cname}"] = ctypes.sizeof(mirror)
        for f, _ in mirror._fields_:
            lines.append(f'printf("offsetof {cname}.{f} %zu\\n", offsetof({cname}, {f}));')
            lines.append(f'printf("sizeof {cname}.{f} %zu\\n", sizeof((({cname}*)0)->{f}));')
            expect[f"offsetof {cname}.{f}"], expect[f"sizeof {cname}.{f}"] = getattr(mirror, f).offset, getattr(mirror, f).size
    fields = re.findall(r"\b(RG_FIELD_\w+)\s*=", header())
    for e in fields + ["RG_MAX_CONTACTS"]:
        lines.append(f'printf("{e} %d\\n", (int){e});')
    expect.update({e: getattr(engine, e[len("RG_FIELD_"):]) for e in fields})
    expect["RG_MAX_CONTACTS"] = engine.MAX_CONTACTS
    src, exe = tmp_path / "abi_layout.c", tmp_path / "abi_layout"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "robogym_b200.h"\nint main(void) {\n' + "\n".join(lines) + "\nreturn 0;\n}\n")
    subprocess.run([os.environ.get("CC", "cc"), "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout
    got = {k: int(v) for k, v in (line.rsplit(" ", 1) for line in out.splitlines())}
    assert got == expect


def test_library_exports_every_declared_symbol():
    from robogym_b200 import build

    path = build.build()
    lib = ctypes.CDLL(path)
    for f in declared_functions():
        assert hasattr(lib, f), f"{f} declared in robogym_b200.h but not exported"
    lib.rg_last_error.restype = ctypes.c_char_p
    assert lib.rg_last_error() is not None


def test_name_tables_travel_in_the_blob(locked_blob, locked_names):
    """rg_model_name2id is served from the RGNAMES1 section of the blob: the Python packer and the C++ host loader
    (shared with the CUDA engine; reached here through the emulation build) agree with the names sidecar."""
    import pyemu
    from robogym_b200 import modelblob

    names = modelblob.unpack_names(locked_blob)
    assert names["joint"] == locked_names["joint"] and names["site"] == locked_names["site"]
    m = modelblob.unpack(locked_blob)
    e = pyemu.EmuBatch(locked_blob, {k: m[k] for k in modelblob.DIMS}, 1)
    L = pyemu.lib()
    for typ in ("body", "joint", "geom", "site", "actuator", "tendon"):
        for i, n in enumerate(locked_names[typ]):
            if n is not None:
                assert L.rge_name2id(e.h, typ.encode(), n.encode()) == locked_names[typ].index(n)
    assert L.rge_name2id(e.h, b"joint", b"no such joint") == -1
    assert L.rge_name2id(e.h, b"no such type", b"x") == -1


def test_unsupported_features_are_refused(locked_blob):
    """What the compiler can describe but the engine does not simulate must not load (ADVICE r1: such models used to step
    with silently wrong physics).  Elliptic cones, welds, joint couplings and mocap bodies are simulated since round 2; a
    connect constraint, a weld between bodies with more than RG_TJ = 8 dofs between them, or an actuator driven by mujoco-py's
    cascaded-PI controller (actuator_user[0] = 1; its law is not in the reference tree) is still refused."""
    import numpy as np

    import pyemu
    from robogym_b200 import modelblob

    names = modelblob.unpack_names(locked_blob)

    def add_eq(m, typ, b1, b2):
        m["neq"] = 1
        m["eq_type"], m["eq_obj1id"], m["eq_obj2id"], m["eq_active"] = (np.array([v], np.int32) for v in (typ, b1, b2, 1))
        m["eq_data"] = np.array([0, 0, 0, 1, 0, 0, 0.0])
        m["eq_solref"], m["eq_solimp"] = np.array([0.02, 1.0]), np.array([0.9, 0.95, 0.001, 0.5, 2.0])

    tip = names["body"].index("robot0:ffdistal")
    for edit, ok in ((lambda m: add_eq(m, 0, 0, tip), False),                                  # connect
                     (lambda m: add_eq(m, 1, 0, tip), True),                                   # weld world <-> fingertip: 6 dofs
                     (lambda m: add_eq(m, 1, names["body"].index("robot0:thdistal"), tip), False),    # thumb tip <-> fingertip: 11 dofs
                     (lambda m: m["actuator_user0"].__setitem__(0, 1.0), True)):                        # mujoco-py's cascaded-PI controller
        m = modelblob.unpack(locked_blob)
        edit(m)
        blob = modelblob.pack(m, names)
        if ok:
            pyemu.EmuBatch(blob, {k: m[k] for k in modelblob.DIMS}, 1)
        else:
            with pytest.raises(RuntimeError):
                pyemu.EmuBatch(blob, {k: m[k] for k in modelblob.DIMS}, 1)


@pytest.mark.gpu
def test_new_entry_points_on_the_device(locked_blob, locked_names):
    """rg_model_name2id / rg_model_set_field_async / rg_batch_create_ex / RG_FIELD_BODY_XVEL through ctypes on a GPU."""
    import numpy as np
    import torch

    from robogym_b200 import build, engine

    build.build()
    model = engine.DeviceModel(locked_blob, 0)
    assert model.name2id("joint", "robot0:WRJ1") == locked_names["joint"].index("robot0:WRJ1")
    assert model.name2id("site", "cube:center") == locked_names["site"].index("cube:center")
    with pytest.raises(ValueError):
        model.name2id("geom", "nope")
    sim = engine.BatchedSim(model, 4, 10, outputs=("site_xpos", "body_xpos", "body_xvel", "ncon", "warn", "contact"), contact_capacity=100, row_capacity=128)
    assert (sim.contact_capacity, sim.row_capacity) == (100, 128) and sim.contact.shape == (4, 100, 4)
    g0 = model.host["opt_gravity"].copy()
    # stream-ordered parameter edit: the step queued BEFORE the edit falls with gravity, the one after it does not
    sim.step()
    z1 = sim.body_xpos[:, locked_names["body"].index("target:middle"), 2].clone()
    v1 = sim.body_xvel[:, locked_names["body"].index("target:middle"), 5].clone()
    model.set_field("opt_gravity", [0.0, 0.0, 0.0])
    sim.step()
    torch.cuda.synchronize()
    v2 = sim.body_xvel[:, locked_names["body"].index("target:middle"), 5]
    # free-falling target cube: v_z = -g t after the first env-step (0.08 s), unchanged by the second (gravity off)
    assert torch.allclose(v1, torch.full_like(v1, g0[2] * 0.08), rtol=2e-3)
    assert torch.allclose(v2, v1, atol=1e-4)
    # linear velocity output equals the finite difference of the body position
    z2 = sim.body_xpos[:, locked_names["body"].index("target:middle"), 2]
    assert torch.allclose((z2 - z1) / 0.08, v2, rtol=5e-3)
    model.set_field("opt_gravity", g0)


def test_product_path_fails_loudly_without_gpu(locked_blob):
    """No CPU fallback: on a box without CUDA the engine raises instead of routing elsewhere."""
    import torch

    from robogym_b200 import engine

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(engine.EngineError):
        engine.DeviceModel(locked_blob, 0)


def test_scratch_budget_keeps_ten_environments_per_sm(locked_blob):
    """dactyl/locked must keep fitting 10 environments per SM: 227 KB opt-in shared memory minus the static part, the
    staged model arrays and the device model view, divided by 10 (rg_batch_size in rg_engine.cu).  Uses the CPU
    emulation build's layout, which is the same rg_make_layout()."""
    import pyemu
    from robogym_b200 import modelblob

    m = modelblob.unpack(locked_blob)
    e = pyemu.EmuBatch(locked_blob, {k: m[k] for k in modelblob.DIMS}, 1)
    scratch = 4 * pyemu.lib().rge_scratch_floats(e.h)
    small = pyemu.lib().rge_small_bytes(e.h)
    fixed = 768 + ((small + 127) & ~127) + 64 + 256            # model view (<= 768 B) + staged arrays + slack + static shared (128 B today)
    assert (232448 - fixed) // scratch >= 10, (scratch, small)


def test_world_shift_of_per_environment_rows():
    """BatchedSim.set_param keeps the engine's fp32 world shift for rows that live in world coordinates (host-side helper,
    device-agnostic: the index and the origin are created on the rows' device)."""
    import numpy as np
    import torch

    from robogym_b200.engine import world_shift_rows

    m = dict(body_parentid=np.array([0, 0, 1, 0]), geom_bodyid=np.array([0, 1, 2]), site_bodyid=np.array([1, 1]))
    v = torch.zeros(2, 12, dtype=torch.float64)
    world_shift_rows(torch, v, "body_pos", m, [1.0, 2.0, 3.0])
    assert v[1].view(4, 3).tolist() == [[0, 0, 0], [-1, -2, -3], [0, 0, 0], [-1, -2, -3]]      # world body itself stays
    v = torch.ones(2, 9, dtype=torch.float32)
    world_shift_rows(torch, v, "geom_pos", m, [1.0, 2.0, 3.0])
    assert v[0].view(3, 3).tolist() == [[0, -1, -2], [1, 1, 1], [1, 1, 1]]
    v = torch.ones(2, 6)
    assert torch.equal(world_shift_rows(torch, v, "site_pos", m, [1.0, 2.0, 3.0]), torch.ones(2, 6))   # nothing on the world body
