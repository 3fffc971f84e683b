"""Generates tests/golden/reference_frame_digests.json: the answers of tests/reference_frame.py (the reference's single-threaded frame restated on
the transpiled reference, oracle/_ref/libbepu_ref.so) on the scene matrix and the PredictBoundingBoxes cases of
tests/test_oracle_driver_pinned_to_reference.py, one SHA-256 each. Run from the repository root where the transpiled library is built
(oracle/ref_transpile/build_ref.py); the file is committed so that the oracle and the device are held to the restatement everywhere."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests import reference_frame as rf  # noqa: E402
from tests import test_oracle_driver_pinned_to_reference as t  # noqa: E402

if __name__ == "__main__":
    if rf.library() is None:
        raise SystemExit("the transpiled reference is not built (oracle/ref_transpile/build_ref.py)")
    out = {"solve": {name: t.digest(t.run_reference(name)) for name in sorted(t.CASES)},
           "bounds": {name: t.bounds_digest(*t.bounds_reference(name)) for name in sorted(t.BOUNDS_CASES)}}
    with open(t.DIGESTS, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print(t.DIGESTS)
