"""Pins the constraint data layouts to the reference. tests/golden/type_layouts.json is generated from the reference's C# sources by
tests/golden/make_type_layouts.py (ordered scalar rows of every PrestepData / AccumulatedImpulses struct and the body count of every registered
type processor: the layout the reference's own ConstraintDescriptionMappingTests round-trips). Checked here: the device and oracle registries
(all 44 types, nothing missing), the row order the joint kernels document and index, and the row order the contact scene generators write."""
import json
import os
import re

import numpy as np

import bepuphysics2_b200 as bp
from bepuphysics2_b200 import scenes
from oracle import binding as ob
from tests import planner

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = planner.TYPE_LAYOUTS


def _compact(rows):
    """['LocalOffsetA.X','LocalOffsetA.Y','LocalOffsetA.Z','SpringSettings.AngularFrequency'] -> ['LocalOffsetA xyz', 'AngularFrequency']"""
    out, i = [], 0
    strip = lambda s: re.sub(r"^(MaterialProperties\.)?(SpringSettings\.|ServoSettings\.|Settings\.)?", "", s)
    while i < len(rows):
        base, _, last = rows[i].rpartition(".")
        if last == "X" and base:
            comps, j = "", i
            while j < len(rows) and rows[j].rpartition(".")[0] == base and rows[j].rpartition(".")[2] in "XYZW":
                comps += rows[j].rpartition(".")[2].lower()
                j += 1
            out.append(strip(base) + " " + comps)
            i = j
        else:
            out.append(strip(rows[i]))
            i += 1
    return out


def test_registries_cover_exactly_the_reference_type_set(libs):
    supported = sorted(t for t in range(64) if bp.type_info(t) is not None)
    assert supported == sorted(FIXTURE), "device registry and the reference's registered type processors differ"
    for type_id, t in FIXTURE.items():
        want = (t["bodies"], len(t["prestep_rows"]), len(t["impulse_rows"]))
        assert bp.type_info(type_id) == want, "device registry, type %d (%s)" % (type_id, t["processor"])
        assert ob.type_info(type_id) == want, "oracle registry, type %d (%s)" % (type_id, t["processor"])


def test_joint_kernels_document_and_index_rows_in_reference_order():
    """Every joint struct in csrc/bepu_joints*.cuh carries a `// prestep: ... | impulses: ...` line listing the rows its code indexes; that list
    must be the reference struct's field order."""
    ids = {}
    text = ""
    for name in ("bepu_joints.cuh", "bepu_joints_more.cuh"):
        text += open(os.path.join(ROOT, "bepuphysics2_b200", "csrc", name)).read() + "\n"
    for m in re.finditer(r"X\((\d+), (\w+)\)", text):
        ids[m.group(2)] = int(m.group(1))
    seen = set()
    for m in re.finditer(r"// prestep: ([^|\n]+)\| impulses?: ([^\n]+)\n", text):
        prestep_doc, impulse_doc = [x.strip() for x in m.group(1).split(",")], m.group(2).strip()
        struct = re.compile(r"struct (\w+) \{\n\s+static constexpr int kBodies").search(text, m.end()).group(1)  # the constraint struct the comment heads
        t = FIXTURE[ids[struct]]
        assert prestep_doc == _compact(t["prestep_rows"]), "%s prestep rows: documented %s, reference %s" % (struct, prestep_doc, _compact(t["prestep_rows"]))
        rows = t["impulse_rows"]
        if impulse_doc == "1":
            assert len(rows) == 1
        elif re.fullmatch(r"[xyzw]+", impulse_doc):
            assert [r.lower() for r in rows] == list(impulse_doc)
        else:
            assert [x.strip() for x in impulse_doc.split(",")] == _compact(rows)
        seen.add(ids[struct])
    assert seen == {t for t in FIXTURE if t >= 22}, "joint types without a checked row list: %s" % sorted({t for t in FIXTURE if t >= 22} - seen)


def test_contact_prestep_generators_write_rows_in_reference_order():
    """scenes.convex_prestep / nonconvex_prestep (what every contact parity test and the bench feed to both the oracle and the device) against the
    reference field order, by writing recognisable values."""
    for n in (1, 2, 3, 4):
        offs = (np.arange(n * 3, dtype=np.float32).reshape(1, n, 3) + 100)
        depths = (np.arange(n, dtype=np.float32).reshape(1, n) + 200)
        normal, offset_b = np.array([[0.1, 0.2, 0.3]], dtype=np.float32), np.array([[7, 8, 9]], dtype=np.float32)
        for two_body, type_id in ((False, n - 1), (True, n + 3)):
            pre = scenes.convex_prestep(offs, depths, normal, offset_b if two_body else None, friction=0.5, spring_settings=(11.0, 12.0), max_recovery=13.0)[0]
            rows = FIXTURE[type_id]["prestep_rows"]
            assert len(rows) == pre.shape[0]
            got = dict(zip(rows, pre.tolist()))
            for i in range(n):
                assert [got["Contact%d.OffsetA.%s" % (i, c)] for c in "XYZ"] == offs[0, i].tolist()
                assert got["Contact%d.Depth" % i] == depths[0, i]
            assert np.allclose([got["Normal.%s" % c] for c in "XYZ"], normal[0])
            if two_body:
                assert [got["OffsetB.%s" % c] for c in "XYZ"] == [7, 8, 9]
            assert got["MaterialProperties.FrictionCoefficient"] == 0.5
            assert (got["MaterialProperties.SpringSettings.AngularFrequency"], got["MaterialProperties.SpringSettings.TwiceDampingRatio"]) == (11.0, 12.0)
            assert got["MaterialProperties.MaximumRecoveryVelocity"] == 13.0
    for n in (2, 3, 4):
        offs = (np.arange(n * 3, dtype=np.float32).reshape(1, n, 3) + 100)
        depths = (np.arange(n, dtype=np.float32).reshape(1, n) + 200)
        normals = (np.arange(n * 3, dtype=np.float32).reshape(1, n, 3) + 300)
        offset_b = np.array([[7, 8, 9]], dtype=np.float32)
        for two_body, type_id in ((False, 6 + n), (True, 13 + n)):
            pre = scenes.nonconvex_prestep(offs, depths, normals, offset_b if two_body else None, friction=0.5, spring_settings=(11.0, 12.0), max_recovery=13.0)[0]
            rows = FIXTURE[type_id]["prestep_rows"]
            assert len(rows) == pre.shape[0]
            got = dict(zip(rows, pre.tolist()))
            for i in range(n):
                assert [got["Contact%d.Offset.%s" % (i, c)] for c in "XYZ"] == offs[0, i].tolist()
                assert got["Contact%d.Depth" % i] == depths[0, i]
                assert [got["Contact%d.Normal.%s" % (i, c)] for c in "XYZ"] == normals[0, i].tolist()
            if two_body:
                assert [got["OffsetB.%s" % c] for c in "XYZ"] == [7, 8, 9]
            assert got["MaterialProperties.FrictionCoefficient"] == 0.5
            assert got["MaterialProperties.MaximumRecoveryVelocity"] == 13.0


def test_roofline_byte_model_uses_the_reference_access_filters():
    """The SURVEY.md §8d algorithmic bytes per evaluation behind `roofline.achieved`, as the compiled planner holds them (get_type_info of
    csrc/bepu_topology.cpp, built from csrc/bepu_type_table.h): per-type read / written float counts must be the sums over the access filters the
    reference declares for each type (fixture: parsed from the processor declarations and IBodyAccessFilter.cs), the bytes must follow from them
    and reproduce the worked examples of SURVEY.md §8d, and the incremental contact update must read every prestep row and write every depth."""
    with open(os.path.join(ROOT, "tests", "golden", "type_layouts.json")) as f:
        filters = json.load(f)["access_filters"]
    moved = lambda names: (sum(filters[f]["read"] for f in names), sum(filters[f]["write"] for f in names))  # read, written
    infos = {t: planner.type_info(t) for t in range(64)}
    assert {t for t, info in infos.items() if info} == set(FIXTURE), "the planner's types and the reference's registered type processors differ"
    for type_id, ref in FIXTURE.items():
        t = infos[type_id]
        bodies, prestep, impulses = ref["bodies"], len(ref["prestep_rows"]), len(ref["impulse_rows"])
        assert (t["bodies"], t["prestep_rows"], t["impulse_rows"]) == (bodies, prestep, impulses), type_id
        assert (t["solve_read"], t["solve_written"]) == moved(ref["solve_filters"]), "type %d: Solve filters %s" % (type_id, ref["solve_filters"])
        assert (t["warm_start_read"], t["warm_start_written"]) == moved(ref["warm_start_filters"]), "type %d: WarmStart filters %s" % (type_id, ref["warm_start_filters"])
        assert t["solve_bytes"] == 4 * (prestep + 2 * impulses + bodies + t["solve_read"] + t["solve_written"]), type_id
        assert t["warm_start_bytes"] == 4 * (prestep + impulses + bodies + t["warm_start_read"] + t["warm_start_written"]), type_id
        contacts = sum(1 for r in ref["prestep_rows"] if r.endswith(".Depth"))
        assert t["contacts"] == contacts, type_id
        assert t["incremental_bytes"] == (4 * (prestep + contacts + bodies + 6 * bodies) if contacts else 0), type_id
    # SURVEY.md §8d worked examples
    assert {k: infos[k]["solve_bytes"] for k in (7, 4, 3, 22, 47, 31, 25, 27, 30, 29)} == {7: 320, 4: 248, 3: 228, 22: 272, 47: 312, 31: 300, 25: 180, 27: 192, 30: 164, 29: 196}
