"""Register and shared-memory budget of the contact-only stage kernels, read from the built libbepucuda.so (cuobjdump --dump-resource-usage).

The contact-only WarmStart / Solve instantiations (kContacts, launched for batches whose every bundle is a contact) exist to be resident at 20 warps
per SM or more (WarmStart 20 at 96 registers, Solve 24 at 80), so that the next stage's CTAs find free slots while a head batch still runs. A
source change that pushes them past their budget, or makes them spill, silently takes that away; this test catches it without a GPU."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "bepuphysics2_b200", "libbepucuda.so")

# H100 (sm_90) per-SM limits
REGS_PER_SM = 65536
REG_ALLOC_UNIT = 256  # registers are allocated per warp in units of 256
SMEM_PER_SM = 228 * 1024
SMEM_RESERVED_PER_CTA = 1024
MAX_WARPS_PER_SM = 64
CTA_WARPS = 2  # kStageBlockThreads = 64

REGISTER_BUDGET = 96  # WarmStartFirst / WarmStart
MIN_WARPS_PER_SM = 20
SOLVE_REGISTER_BUDGET = 80
SOLVE_MIN_WARPS_PER_SM = 24
# The WarmStart kernels pass argument structs to the out-of-line angular-momentum integrators on the stack (48 B); any larger frame is spill.
MAX_STACK_BYTES = 48

CONTACT_KERNEL = re.compile(r"_ZN\d+(bepu_fast|bepu_strict)23constraint_stage_kernelILi(\d)ELi(\d+)ELb([01])ELb1EE")


def resource_usage():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(LIB):
        pytest.skip("libbepucuda.so has not been built")
    if not os.path.exists(tool):
        pytest.skip("cuobjdump is not available")
    out = subprocess.run([tool, "--dump-resource-usage", LIB], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=True).stdout
    kernels = {}
    name = None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        if name and "REG:" in line:
            kernels[name] = {k: int(v) for k, v in re.findall(r"(REG|STACK|SHARED|LOCAL):(\d+)", line)}
            name = None
    return kernels


def resident_warps(regs, shared):
    per_warp = -(-regs * 32 // REG_ALLOC_UNIT) * REG_ALLOC_UNIT
    ctas_by_regs = REGS_PER_SM // (per_warp * CTA_WARPS)
    ctas_by_smem = SMEM_PER_SM // (shared + SMEM_RESERVED_PER_CTA)
    return min(min(ctas_by_regs, ctas_by_smem) * CTA_WARPS, MAX_WARPS_PER_SM)


def contact_kernels():
    kernels = resource_usage()
    found = {}
    for name, res in kernels.items():
        m = CONTACT_KERNEL.match(name)
        if m:
            flavour, stage, minb, ext = m.groups()
            found[(flavour, int(stage), int(minb), ext == "1")] = res
    return found


def test_contact_only_stage_kernels_exist_for_both_flavours_and_all_three_stages():
    found = contact_kernels()
    for flavour in ("bepu_fast", "bepu_strict"):
        assert {stage for (f, stage, _, _) in found if f == flavour} == {0, 1, 2}, sorted(found)


def test_contact_only_stage_kernels_stay_within_the_register_budget_without_spills():
    found = contact_kernels()
    assert found
    for key, res in found.items():
        assert res["REG"] <= (SOLVE_REGISTER_BUDGET if key[1] == 2 else REGISTER_BUDGET), (key, res)
        assert res["LOCAL"] == 0 and res["STACK"] <= MAX_STACK_BYTES, (key, res)


def test_contact_only_stage_kernels_keep_at_least_20_warps_resident_per_sm():
    found = contact_kernels()
    assert found
    for key, res in found.items():
        assert resident_warps(res["REG"], res["SHARED"]) >= (SOLVE_MIN_WARPS_PER_SM if key[1] == 2 else MIN_WARPS_PER_SM), (key, res)


def test_resident_warp_arithmetic():
    assert resident_warps(96, 13328) == 20
    assert resident_warps(80, 13328) == 24
    assert resident_warps(113, 13328) == 16
    assert resident_warps(95, 13328) == 20
