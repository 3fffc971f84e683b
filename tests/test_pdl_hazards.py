"""The programmatic-dependent-launch rule of DESIGN §3 held to the shipped kernels, not to a model of them.

A stage kernel's prologue runs before its grid-dependency wait, while its predecessor still runs, and may load only what that predecessor does not
write. libbepucuda_hazard.so (-DBEPU_HAZARD, built next to the shipped library) delays every post-wait access of every PDL kernel, so that the
next grid's prologue loads all land before any store of its predecessor, and can plant one wrong-side load per context (a canary). On the CPU:
the one trigger function, the variant's build, and that the GPU configurations reach every launch flag and instantiation. On the GPU
(tests/tools/pdl_hazards.py in a child process with BEPUCUDA_VARIANT=hazard): the residency that makes the delay meaningful, every configuration
bit for bit against the oracle with the delay on, and every canary caught."""
import json
import os
import re
import subprocess
import sys

import pytest

from bepuphysics2_b200 import _build, sharding
from tests import planner
from tests.tools import pdl_hazards as hz

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bepuphysics2_b200", "csrc")
CUOBJDUMP = os.path.join(os.path.dirname(_build.NVCC), "cuobjdump")
BARRIER = -1  # kernel id of a rank barrier in the launch lists below


# ---- CPU ----------------------------------------------------------------------------------------------------------------------------------------
def test_every_pdl_trigger_goes_through_the_one_function():
    """griddepcontrol appears once in csrc/, in pdl_wait_then_trigger, and each of the three PDL kernels (the stage kernels' constraint_stage_body,
    the incremental update's integrate_body_pose, the rank barrier) reaches it: a new PDL kernel cannot escape the hazard build's delay."""
    hits = []
    for name in sorted(os.listdir(CSRC)):
        path = os.path.join(CSRC, name)
        if os.path.isfile(path):
            with open(path) as f:
                for n, line in enumerate(f, 1):
                    if "griddepcontrol." in line and not line.lstrip().startswith("//"):
                        hits.append((name, line.strip()))
    assert hits == [("bepu_device_types.h", 'asm volatile("griddepcontrol.wait;" ::: "memory");'),
                    ("bepu_device_types.h", 'asm volatile("griddepcontrol.launch_dependents;");')], hits
    with open(os.path.join(CSRC, "bepu_device_types.h")) as f:
        body = f.read().split("void pdl_wait_then_trigger(", 1)[1].split("\n}\n", 1)[0]
    assert "griddepcontrol.launch_dependents" in body
    for name, function in (("bepu_solver_kernels.cuh", "constraint_stage_body"), ("bepu_solver_kernels.cuh", "integrate_body_pose"),
                           ("bepu_layout_kernels.cu", "shard_barrier_kernel")):
        with open(os.path.join(CSRC, name)) as f:
            text = f.read()
        start = text.index(function + "(")
        assert "pdl_wait_then_trigger(" in text[start:text.index("\n}\n", start)], function


def _kernels(lib):
    """Mangled names of the kernels a library defines (their host stubs share the device names)."""
    out = subprocess.run(["nm", lib], check=True, stdout=subprocess.PIPE, text=True).stdout
    return sorted({line.split()[-1] for line in out.splitlines() if line.split()[1:2] in (["T"], ["W"], ["t"]) and re.search(r"_kernel[A-Z]", line.split()[-1]) and "__device_stub" not in line and "launch_" not in line})


def _sass(lib, functions):
    return subprocess.run([CUOBJDUMP, "-sass", "-fun", ",".join(functions), lib], check=True, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True).stdout


def test_hazard_variant_builds_for_sm_90a_with_both_flavours_and_the_shipped_library_has_none_of_it(libs):
    """The hazard variant of every kernel, both numerics flavours, for sm_90a, with the delay compiled into the stage kernels (the integrated
    WarmStart and the incremental update of each flavour are read) and the rank barrier; the shipped library has the same kernels and no timer read
    there. A variant build leaves the shipped library's paths alone."""
    shipped = (_build.BUILD, _build.LIB_CUDA)
    lib, _ = _build.build(variant="hazard", defines=_build.VARIANTS["hazard"])
    assert (_build.BUILD, _build.LIB_CUDA) == shipped and lib == os.path.join(os.path.dirname(_build.LIB_CUDA), "libbepucuda_hazard.so")
    kernels = _kernels(lib)
    assert kernels == _kernels(_build.LIB_CUDA)
    probes = [k for k in kernels if "shard_barrier_kernel" in k or "integrated_constraint_stage_kernel" in k or re.search(r"constraint_stage_kernelILi3ELi1E", k)]
    for ns in ("bepu_fast", "bepu_strict"):
        assert sum(ns in k for k in probes) == 2, (ns, probes)
    hazard, plain = _sass(lib, probes), _sass(_build.LIB_CUDA, probes)
    assert "arch = sm_90a" in hazard
    timed = {part.split(None, 1)[0] for part in hazard.split("Function : ")[1:] if "GLOBALTIMER" in part}
    assert timed == set(probes), sorted(set(probes) - timed)
    assert plain.count("Function : ") == len(probes) and "GLOBALTIMER" not in plain


def _launch_context(name):
    _, kw, kind, _ = hz.CONFIGS[name]
    integrator = kw.get("integrator")
    return kind == "terms", integrator.angular_integration_mode if integrator is not None else 0


def config_launches(name):
    """Per context of configuration `name` (one, or one per rank): rows stage, kernel, flags, warps of every launch the GPU run makes with PDL or
    that precedes one, in program order; the body count."""
    sim = hz.make_sim(name)
    ranks = hz.CONFIGS[name][3]
    ext, mode = _launch_context(name)
    if ranks:
        shards, _, _, _ = sharding.partition(sim, ranks)
        fallback = sharding.fallback_rank(sim, ranks)
        plans = [planner.plan(planner.shard_sources(shards[r]), sim.bundle_width, sim.fallback_batch_threshold, sim.batch_count, sim.body_count, True, r,
                              fallback) for r in range(ranks)]
    else:
        plans = [planner.plan(planner.sim_sources(sim), sim.bundle_width, sim.fallback_batch_threshold, sim.batch_count, sim.body_count)]
    out = []
    for p in plans:
        ops, _ = p.program(sim.velocity_iterations, len(sim.constrained_kinematics), True, bool(ranks), sim.body_count)
        ops = ops[(ops[:, 2] > 0) | (ops[:, 3] == planner.RANK_BARRIER)]
        kernel, flags = planner.resolve(ops, ext, mode, False).T
        rows = []
        for op, k, f in zip(ops, kernel, flags):
            stage = int(op[0])
            if int(op[3]) == planner.RANK_BARRIER:
                rows.append((stage, BARRIER, 0, 8))
            elif stage <= planner.INCREMENTAL:
                ctas = (int(op[2]) + 1) // 2 + ((sim.body_count + 63) // 64 if f & planner.BODIES_INTEGRATED and stage == planner.INCREMENTAL else 0)
                rows.append((stage, int(k), int(f), 2 * ctas))
            else:
                rows.append((stage, planner.KERNEL_FULL, int(f), 0))  # kinematic and final pose passes: launched without PDL
        out.append((rows, sim.body_count, bool(ranks), p))
    return out


def test_gpu_configurations_reach_every_launch_flag_and_instantiation(libs):
    """Across the configurations the GPU check runs, with their launch contexts: row prefetch, world loads on a Solve and on a WarmStart, owned
    loads, the bodies-integrated flag; the full, contact-only, integrated WarmStart, deep, kExt and sharded instantiations; the incremental update's
    body CTAs; a rank barrier. Without them the check would hold the rule only where it is easy."""
    seen = set()
    for name in hz.CONFIGS:
        for rows, _, sharded, _ in config_launches(name):
            for stage, kernel, flags, _ in rows:
                if kernel == BARRIER:
                    seen.add("rank barrier")
                    continue
                if stage > planner.INCREMENTAL:
                    continue
                seen |= {what for bit, what in ((planner.ROWS, "prefetch rows"), (planner.EARLY_OWNED, "early owned"), (planner.BODIES_INTEGRATED, "bodies integrated"))
                         if flags & bit}
                if flags & planner.EARLY_WORLD:
                    seen.add("early world on %s" % ("Solve" if stage == planner.SOLVE else "WarmStart"))
                if stage == planner.INCREMENTAL:
                    seen.add("incremental body CTAs" if flags & planner.BODIES_INTEGRATED else "incremental")
                    continue
                if sharded:
                    seen.add("sharded")
                elif kernel == planner.KERNEL_DEEP:
                    seen.add("deep")
                elif kernel == planner.KERNEL_CONTACTS:
                    seen.add("integrated WarmStart" if stage == planner.WS and flags & planner.BODIES_INTEGRATED else "contact-only")
                else:
                    seen.add("full")
                if flags & planner.EXT:
                    seen.add("kExt")
    want = {"prefetch rows", "early world on Solve", "early world on WarmStart", "early owned", "bodies integrated", "full", "contact-only",
            "integrated WarmStart", "deep", "kExt", "sharded", "incremental body CTAs", "rank barrier"}
    assert want <= seen, sorted(want - seen)


# Warps per SM each instantiation keeps resident (its __launch_bounds__): the full switch 16, the contact-only kernels 20 (their WarmStart budget;
# the Solve one keeps 24), the deep kernels 24; the rank barrier is one 256-thread CTA.
RESIDENT_WARPS = {planner.KERNEL_FULL: 16, planner.KERNEL_CONTACTS: 20, planner.KERNEL_DEEP: 24, BARRIER: 64}


def residency_failures(launches, sm_count):
    """Pairs of consecutive PDL launches that do not fit on the device together, as device fractions: every launch of a context and the one after
    it (all ranks of a configuration share the device, so their pairs add up). In a scene with deep batches, several waves long, only a dependent
    that loads body records before its wait is checked, and it needs only the start of its first wave (one CTA per SM) beside the predecessor's
    last wave: the deep kernels themselves load no body record before their wait."""
    worst = {}
    deep = any(k == planner.KERNEL_DEEP for rows, _, _, _ in launches for _, k, _, _ in rows)
    for rows, _, _, _ in launches:
        for i in range(1, len(rows)):
            (s0, k0, _, w0), (s1, k1, f1, w1) = rows[i - 1], rows[i]
            if (s1 > planner.INCREMENTAL and k1 != BARRIER) or (s0 > planner.INCREMENTAL and k0 != BARRIER):
                continue  # a launch without PDL on either side: no overlap
            c0, c1 = RESIDENT_WARPS[k0] * sm_count, RESIDENT_WARPS[k1] * sm_count
            if deep:
                if not f1 & (planner.EARLY_WORLD | planner.EARLY_OWNED | planner.BODIES_INTEGRATED):
                    continue  # the deep scene: only dependents that load body records before their wait
                # several waves deep: one dependent CTA per SM must start beside the predecessor's last wave
                need = (w0 % c0 or c0) / c0 + min(w1, 2 * sm_count) / c1
            else:
                need = w0 / c0 + w1 / c1
            worst[i] = worst.get(i, 0.0) + need
    return {i: f for i, f in worst.items() if f > 1.0}


@pytest.mark.gpu
def test_pdl_hazards_on_the_h100(libs):
    """With the delay on: every configuration's pair of consecutive PDL launches fits on the device together, every configuration in both execution
    modes equals the oracle bit for bit, and every canary makes its scene differ. Whether a canary also differed with plain timing is reported."""
    import torch

    sm_count = torch.cuda.get_device_properties(0).multi_processor_count
    for name in hz.CONFIGS:
        bad = residency_failures(config_launches(name), sm_count)
        assert not bad, "%s: launches that do not fit beside their predecessor on %d SMs: %s" % (name, sm_count, sorted(bad.items())[:5])
    assert os.path.exists(os.path.join(os.path.dirname(_build.LIB_CUDA), "libbepucuda_hazard.so")), "__graft_entry__.build() builds the hazard variant"
    env = dict(os.environ, BEPUCUDA_VARIANT="hazard")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.join(ROOT, "tests", "tools", "pdl_hazards.py"), "--check"]
    r = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    result = json.loads(r.stdout.strip().split("\n")[-1])
    print(json.dumps(result, indent=1))
    differing = {k: v["difference"] for k, v in result["scenes"].items() if v["difference"] is not None}
    assert not differing, differing
    missed = [k for k, v in result["canaries"].items() if not v["caught_with_delay"]]
    assert not missed, missed
    assert len(result["canaries"]) == sum(len(names) for _, names in hz.CANARIES.values())
