"""CPU tests of the drop-in boundary: the C-ABI library loads without a GPU, exports every symbol include/bepucuda.h declares, its type
registry agrees with the oracle's, and there is no CPU fallback."""
import ctypes as C
import os
import re

import pytest

import bepuphysics2_b200 as bp
from bepuphysics2_b200 import native
from oracle import binding as ob
from tests import planner

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol(libs):
    cuda, _ = bp.load_libraries()
    header = open(os.path.join(ROOT, "include", "bepucuda.h")).read()
    declared = sorted(set(re.findall(r"\b(bepucuda_[a-z_0-9]+)\s*\(", header)))
    assert declared, "no declarations parsed"
    for name in declared:
        assert hasattr(cuda, name), "libbepucuda.so does not export %s" % name
    assert sorted(native.C_ABI_SYMBOLS) == declared


def test_type_registry_matches_oracle_and_reference_sizes(libs):
    # (bodies, prestep floats, impulse floats) from the reference's struct definitions (SURVEY.md §8a table)
    expected = {0: (1, 11, 4), 1: (1, 15, 5), 2: (1, 19, 6), 3: (1, 23, 7), 4: (2, 14, 4), 5: (2, 18, 5), 6: (2, 22, 6), 7: (2, 26, 7),
                8: (1, 18, 6), 9: (1, 25, 9), 10: (1, 32, 12), 15: (2, 21, 6), 16: (2, 28, 9), 17: (2, 35, 12),
                22: (2, 8, 3), 25: (2, 9, 1), 26: (2, 14, 1), 27: (2, 12, 1), 29: (2, 9, 3), 30: (2, 5, 3), 46: (2, 14, 4), 47: (2, 14, 5),
                23: (2, 8, 2), 24: (2, 8, 1), 28: (2, 9, 1), 31: (2, 9, 6), 32: (4, 3, 1), 33: (2, 12, 1), 34: (2, 10, 1), 35: (2, 3, 1), 36: (3, 3, 1),
                37: (2, 14, 2), 38: (2, 15, 1), 39: (2, 12, 1), 40: (2, 13, 1), 41: (2, 6, 1), 42: (1, 9, 3), 43: (1, 5, 3), 44: (1, 11, 3), 45: (1, 8, 3),
                52: (2, 8, 3), 53: (2, 11, 3), 54: (2, 6, 1), 55: (2, 4, 1)}
    assert sorted(t for t in range(64) if bp.type_info(t) is not None) == sorted(expected), "every registered type has a pinned layout"
    for type_id in range(64):
        ours, theirs = bp.type_info(type_id), ob.type_info(type_id)
        assert ours == theirs, "type %d: device registry %s vs oracle %s" % (type_id, ours, theirs)
        if type_id in expected:
            assert ours == expected[type_id]


def test_unsupported_type_is_reported(libs):
    cuda, _ = bp.load_libraries()
    assert cuda.bepucuda_type_info(63, None, None, None) == native.ERR_UNSUPPORTED_TYPE


def test_error_codes_match_the_header():
    header = open(os.path.join(ROOT, "include", "bepucuda.h")).read()
    defined = {name: int(value) for name, value in re.findall(r"#define BEPUCUDA_ERR_([A-Z_]+) \((-?\d+)\)", header)}
    assert len(defined) == 7
    assert defined == {name[4:]: getattr(native, name) for name in dir(native) if name.startswith("ERR_")}


def test_contact_count_matches_the_type_registry(libs):
    """native.contact_count (the feature-id layout of bepucuda_set_contact_features / bepucuda_update_contacts) and bp.type_info against the
    reference's layouts (tests/golden/type_layouts.json): one contact per depth row and one penetration impulse per contact, 0 for joints and ids
    without a type, and the bodies and row counts of every type."""
    for type_id in range(64):
        info, n = bp.type_info(type_id), native.contact_count(type_id)
        assert n == planner.contacts(type_id), type_id
        if type_id not in planner.TYPE_LAYOUTS:
            assert info is None, type_id
            continue
        ref = planner.TYPE_LAYOUTS[type_id]
        assert info == (ref["bodies"], len(ref["prestep_rows"]), len(ref["impulse_rows"])), type_id
        assert len(planner.penetration_rows(type_id)) == n, type_id


def test_no_cpu_fallback_without_a_device(libs):
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    sim = bp.Simulation()
    with pytest.raises(bp.BepuCudaError) as e:
        bp.CudaTimestepper(sim)
    assert e.value.code == native.ERR_NO_DEVICE


def test_product_sources_never_reference_the_oracle():
    pkg = os.path.join(ROOT, "bepuphysics2_b200")
    for dirpath, _, files in os.walk(pkg):
        if "build" in dirpath:
            continue
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp", ".inc")):
                text = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in text.lower() or f == "__init__.py" and "oracle" not in text.lower(), "%s mentions the oracle" % os.path.join(dirpath, f)


def test_only_the_checkers_load_the_oracle():
    """Outside tests/ (which includes the diagnostic scripts of tests/tools) only bench.py (cpu_baseline / --impl reference legs) and
    __graft_entry__.py (build() compiles it, smoke() checks against it) may touch oracle/."""
    allowed = {"bench.py", "__graft_entry__.py"}
    for dirpath, dirnames, files in os.walk(ROOT):
        rel = os.path.relpath(dirpath, ROOT)
        dirnames[:] = [d for d in dirnames if not d.startswith(".") and d not in ("gpurun_out", "baseline", "build", "__pycache__")]
        if rel == "." :
            dirnames[:] = [d for d in dirnames if d not in ("tests", "oracle")]
        for f in files:
            if f.endswith(".py") and not (rel == "." and f in allowed):
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b|oracle[/\\.]binding|libbepu_oracle", text, flags=re.M), "%s uses the oracle" % os.path.join(rel, f)


def test_public_header_is_plain_c(tmp_path):
    """include/bepucuda.h is the drop-in boundary: it has to compile as C99 (what a P/Invoke / cgo / ctypes binding generator consumes) and as
    C++11, with no CUDA or torch types in any signature."""
    import subprocess

    header = open(os.path.join(ROOT, "include", "bepucuda.h")).read()
    code = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    code = re.sub(r"bepucuda|BEPUCUDA|void\* cuda_stream", "", code)  # the one stream handle crosses as an opaque void*
    for forbidden in ("cuda", "torch", "at::", "std::", "#include <cuda"):
        assert forbidden not in code, "%r appears in the public header's code" % forbidden
    c = tmp_path / "use.c"
    c.write_text('#include "bepucuda.h"\nint main(void) { bepucuda_config cfg; bepucuda_timings t; (void)cfg; (void)t; return bepucuda_type_info(0, 0, 0, 0) == 0; }\n')
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"), str(c)], check=True)
    cpp = tmp_path / "use.cpp"
    cpp.write_text('#include "bepucuda.h"\nint main() { return 0; }\n')
    subprocess.run(["g++", "-std=c++11", "-Wall", "-Werror", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"), str(cpp)], check=True)


def test_csharp_binding_declares_every_entry_point():
    """integration/csharp/BepuCuda.cs (the P/Invoke stub INTEGRATION.md hands to a bepuphysics2 maintainer; not compilable here) must not drift from
    the header: one [DllImport] per exported function, same argument count."""
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "bepucuda.h")).read(), flags=re.S)
    cs = open(os.path.join(ROOT, "integration", "csharp", "BepuCuda.cs")).read()
    declared = {m.group(1): m.group(2) for m in re.finditer(r"\b(bepucuda_[a-z_0-9]+)\s*\(([^;{]*?)\)\s*;", header)}
    bound = {m.group(1): m.group(2) for m in re.finditer(r"extern\s+\w+\s+(bepucuda_[a-z_0-9]+)\s*\(([^)]*)\)", cs)}
    assert sorted(declared) == sorted(bound)
    count = lambda args: 0 if args.strip() in ("", "void") else args.count(",") + 1
    for name in declared:
        assert count(declared[name]) == count(bound[name]), "%s: %d C parameters vs %d in the C# binding" % (name, count(declared[name]), count(bound[name]))


def test_csharp_timestepper_follows_the_reference_scheduler_rule_and_checks_the_callbacks():
    """integration/csharp/CudaTimestepper.cs evaluates the velocity-iteration scheduler host-side: a result below 1 means VelocityIterationCount
    (Solver_Solve.cs:L743-751), never Math.Max(1, n); and it takes the behavioural integrator properties from the simulation's callbacks."""
    cs = open(os.path.join(ROOT, "integration", "csharp", "CudaTimestepper.cs")).read()
    assert "Math.Max(1, solver.VelocityIterationScheduler" not in cs
    assert re.search(r"scheduled\s*<\s*1\s*\?\s*solver\.VelocityIterationCount\s*:\s*scheduled", cs)
    for prop in ("AngularIntegrationMode", "AllowSubstepsForUnconstrainedBodies", "IntegrateVelocityForKinematics"):
        assert "callbacks." + prop in cs and "live." + prop in cs
    # the Python host mirror applies the same rule
    import bepuphysics2_b200 as bp

    sim = bp.Simulation(substeps=4, velocity_iterations=3)
    sim.set_solve_description(4, 3, velocity_iteration_scheduler=lambda i: [2, 0, -1, 5][i])
    assert sim.velocity_iterations == [2, 3, 3, 5]


def test_library_binary_matches_its_stamp(libs):
    """The stamp next to libbepucuda.so records a digest of the sources AND the sha256 of the binary built from them; the loader refuses a binary
    that does not match (a stale or foreign .so next to a fresh stamp)."""
    import shutil
    import tempfile

    from bepuphysics2_b200 import _build

    assert _build.binary_matches_stamp() is True
    with tempfile.TemporaryDirectory() as d:
        lib = os.path.join(d, "libbepucuda.so")
        shutil.copy(_build.LIB_CUDA, lib)
        shutil.copy(_build.LIB_CUDA + ".stamp", lib + ".stamp")
        assert _build.binary_matches_stamp(lib) is True
        with open(lib, "ab") as f:
            f.write(b"\0")
        assert _build.binary_matches_stamp(lib) is False
        os.remove(lib + ".stamp")
        assert _build.binary_matches_stamp(lib) is None
