"""Development diagnostic: per configuration of tests/test_fast_build_precision.py, each constraint type's lane error against the float64
evaluation of the same solve, for the strict and the fast GPU build, with the flips and ill-conditioned lanes (see compare_builds there).
Needs a GPU. Usage: python tests/tools/fast_error_stats.py [configuration ...]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from bepuphysics2_b200 import _build  # noqa: E402
from oracle import binding as ob  # noqa: E402
from tests import test_fast_build_precision as fp  # noqa: E402


def main(names):
    _build.build()
    ob.build()
    dll = fp.build_driver()
    for name in names or fp.CONFIGS:
        case = fp.Case(name)
        x64 = case.lanes(case.f64(dll))
        table = fp.compare_builds(case.lanes(case.gpu(strict=True)), case.lanes(case.gpu(strict=False)), x64)
        print(fp.format_table(name, table))
        for verdict in ("ok", "typical_ok"):
            for line in fp.failures(table, verdict):
                print("  %s check fails: %s" % ("issue" if verdict == "ok" else "typical-lane", line))
        print()


if __name__ == "__main__":
    main(sys.argv[1:])
