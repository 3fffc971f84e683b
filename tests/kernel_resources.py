"""The stage kernels' registers, stack and shared memory, read from the built libbepucuda.so (cuobjdump --dump-resource-usage), the warps per SM
they leave resident on an H100, and the budgets the tests hold them to."""
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
