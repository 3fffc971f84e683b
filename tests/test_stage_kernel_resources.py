"""Register and shared-memory budget of the contact-only stage kernels, read from the built libbepucuda.so (cuobjdump --dump-resource-usage).

The contact-only WarmStart / Solve instantiations (kContacts, launched for batches whose every bundle is a contact) exist to be resident at 20 warps
per SM or more (WarmStart 20 at 96 registers, Solve 24 at 80), so that the next stage's CTAs find free slots while a head batch still runs. A
source change that pushes them past their budget, or makes them spill, silently takes that away; this test catches it without a GPU."""
import re

from tests.kernel_resources import MAX_STACK_BYTES, MIN_WARPS_PER_SM, REGISTER_BUDGET, SOLVE_MIN_WARPS_PER_SM, SOLVE_REGISTER_BUDGET, resident_warps, resource_usage

CONTACT_KERNEL = re.compile(r"_ZN\d+(bepu_fast|bepu_strict)23constraint_stage_kernelILi(\d)ELi(\d+)ELb([01])ELb1EE")


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
