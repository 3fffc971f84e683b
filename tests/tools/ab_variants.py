"""A/B of the staged kernel experiments (DESIGN.md §9) against the shipped library.

    python tests/tools/ab_variants.py build [name ...]     # libbepucuda_<name>.so per variant (no GPU needed)
    python tests/tools/ab_variants.py run [name ...]       # on an H100: parity subset + bench per variant that has been built, one table

Variant libraries are large (about 33 MB each): build only what a session will measure and delete them afterwards
(`python tests/tools/ab_variants.py clean`). A variant that fails the parity subset is reported as such and not benchmarked."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
PKG = os.path.join(ROOT, "bepuphysics2_b200")
VARIANTS = {
    # name: extra -D flags, e.g. deep16 = -DBEPU_DEEP_MINB=16 (64 registers for deep batches).
}
PARITY = "box_stack or shape_pile or fallback or randomised or unconstrained or registered_host or deterministic"


def lib(name):
    return os.path.join(PKG, "libbepucuda_%s.so" % name)


def build(names):
    for name in names:
        print("building", name, VARIANTS[name], flush=True)
        subprocess.check_call([sys.executable, "-m", "bepuphysics2_b200._build", "--variant=" + name] + VARIANTS[name], cwd=ROOT)


def run(names):
    rows = []
    for name in [None] + [n for n in names if os.path.exists(lib(n))]:
        env = dict(os.environ)
        if name:
            env["BEPUCUDA_VARIANT"] = name
        label = name or "shipped"
        t = subprocess.run([sys.executable, "-m", "pytest", "tests", "-m", "gpu", "-x", "-q", "-k", PARITY], cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        verdict = t.stdout.strip().splitlines()[-1] if t.stdout.strip() else "no output"
        if t.returncode != 0:
            rows.append((label, "PARITY FAILED: " + verdict, None))
            print(t.stdout[-3000:], flush=True)
            continue
        b = subprocess.run([sys.executable, "bench.py", "--no-cpu-baseline", "--steps", "40", "--warmup", "5"], cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
        try:
            line = json.loads(b.stdout.strip().splitlines()[-1])
        except Exception:  # noqa: BLE001
            rows.append((label, verdict, "bench failed: " + b.stderr[-300:]))
            continue
        rows.append((label, verdict, "100 k: %.3f ms/step (e2e %.3f)   1 M: %.3f ms/step   stage profile %s" % (
            line["ms_per_step"], line["e2e"]["ms_per_step"], line.get("large_scene", {}).get("ms_per_step", float("nan")), line.get("stage_profile_ms"))))
    for label, verdict, bench in rows:
        print("%-14s | %s | %s" % (label, verdict, bench))


def main():
    cmd = sys.argv[1] if len(sys.argv) > 1 else ""
    names = sys.argv[2:] or list(VARIANTS)
    unknown = [n for n in names if n not in VARIANTS]
    if unknown or cmd not in ("build", "run", "clean"):
        sys.exit("usage: ab_variants.py build|run|clean [%s]" % " ".join(VARIANTS))
    if cmd == "build":
        build(names)
    elif cmd == "run":
        run(names)
    else:
        for n in names:
            for path in (lib(n), lib(n) + ".stamp"):
                if os.path.exists(path):
                    os.remove(path)


if __name__ == "__main__":
    main()
