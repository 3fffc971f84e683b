"""Code size and budget of the integrated contact-only WarmStart kernel, read from the built libbepucuda.so (cuobjdump).

The WarmStart launches whose poses and world inertias the incremental update integrated (kLaunchBodiesIntegrated: every WarmStart of substeps > 0
of a 100 k-body pile) run integrated_constraint_stage_kernel, which has no pose integration. The head stages of that pile run all eight convex
contact types side by side on each SM, so the SM fetches the code of all of them, and the project has measured instruction supply as a limit on
those stages before. Before this instantiation existed those launches ran the integrating kernel: 11 504 SASS instructions in the fast build (96
registers, 48 B stack), 14 536 in the strict one. This test holds the integrated kernel, in both builds, to a budget set from the build that
introduced it (fast 4 512, strict 5 320 instructions, CUDA 12.9, sm_90a) plus about 10 %, to less than half the integrating one, and to the
contact-only WarmStart register and residency budget without spills."""
import os
import re
import shutil
import subprocess

import pytest

from tests.kernel_resources import LIB, MAX_STACK_BYTES, MIN_WARPS_PER_SM, REGISTER_BUDGET, resident_warps, resource_usage

KERNEL = re.compile(r"_ZN\d+(bepu_fast|bepu_strict)\d+(constraint_stage_kernel|integrated_constraint_stage_kernel)ILi1ELi\d+ELb0ELb1EE")
BUDGET = {"bepu_fast": 5000, "bepu_strict": 5850}


def warm_start_kernels():
    """(flavour, integrated) -> (mangled name, resource usage) of the contact-only WarmStart kernels without kExt."""
    found = {}
    for name, res in resource_usage().items():
        m = KERNEL.match(name)
        if m:
            found[(m.group(1), m.group(2).startswith("integrated"))] = (name, res)
    return found


@pytest.fixture(scope="module")
def sass_sizes():
    """(flavour, integrated) -> SASS instruction count."""
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump is not available")
    kernels = warm_start_kernels()
    out = subprocess.run([tool, "-sass", "-fun", ",".join(name for name, _ in kernels.values()), LIB], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL,
                         text=True, check=True).stdout
    counts, current = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            current = m.group(1)
            counts.setdefault(current, 0)
        elif current and re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+\S", line):
            counts[current] += 1
    return {key: counts[name] for key, (name, _) in kernels.items() if name in counts}


def test_both_contact_only_warm_start_instantiations_exist_in_both_flavours():
    assert set(warm_start_kernels()) == {(f, i) for f in ("bepu_fast", "bepu_strict") for i in (False, True)}


def test_the_integrated_warm_start_stays_within_its_instruction_budget(sass_sizes):
    for flavour, limit in BUDGET.items():
        assert sass_sizes[(flavour, True)] <= limit, (flavour, sass_sizes)
        assert 2 * sass_sizes[(flavour, True)] < sass_sizes[(flavour, False)], (flavour, sass_sizes)


def test_the_integrated_warm_start_keeps_the_contact_only_register_budget_without_spills():
    for (flavour, integrated), (name, res) in warm_start_kernels().items():
        if integrated:
            assert res["REG"] <= REGISTER_BUDGET and res["LOCAL"] == 0 and res["STACK"] <= MAX_STACK_BYTES, (name, res)
            assert resident_warps(res["REG"], res["SHARED"]) >= MIN_WARPS_PER_SM, (name, res)
