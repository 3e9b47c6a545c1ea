"""The inputs of tests/test_gpu_candidate_units.py (tests/cand_inputs.py) still reach the edges of the candidate lists' set emulation.

Each input runs through cand_inputs' model of CPython 3.12's setobject.c, which must first reproduce `list(set(...))` of the same tuples
exactly; then the model counts what the inputs reach and the floors below are asserted, so the generators cannot drift away from the
cases they are for: every resize threshold with the resize at lane 0, a middle lane and lane 31 of a 32-key chunk and with staged keys
pending after it, exactly 1228 and 1229 distinct keys, the linear probe window, the wrap at the table end, two or more perturb steps,
duplicates inside and across chunks, items with equal sides in six orientations, 16-bit and 32-bit keys; in the continuous domain tag
matches between distinct tuples (in the read-only probe and in lane 0's insertion), value-equal coordinates with other bits, equal tuples
from different codes, the fit test's 1e-6 boundary to the ulp, item sides 0, 5e-7, 1e-6 and 2e-6 apart, and coordinates past 2200.
"""
import collections
import math
import sys

import pytest

import cand_inputs as ci

pytestmark = pytest.mark.skipif(sys.version_info[:2] != (3, 12), reason="the candidate order is CPython 3.12's set order (DESIGN section 6)")


def _lane(l):
    return "lane0" if l == 0 else "lane31" if l == 31 else "mid"


def _run(cases, seq_of):
    st = ci.new_stats()
    out = []
    for k, c in enumerate(cases):
        seq, n = seq_of(c)
        order, over, _ = ci.run_device_order(seq, n, st)
        ref = ci.reference_order([t for _, t in seq])
        if over:
            assert len(ref) > ci.CAND_CAP and len(order) == ci.CAND_CAP + 1, "case %d" % k
        else:
            assert len(ref) <= ci.CAND_CAP and order == ref, "case %d: the model's order is not CPython's" % k
        out.append((seq, order, over, len(ref)))
    return st, out


@pytest.fixture(scope="module")
def discrete():
    cases = ci.discrete_cases()
    return cases, _run(cases, ci.case_sequence)


@pytest.fixture(scope="module")
def continuous():
    cases = ci.continuous_cases()
    return cases, _run(cases, ci.c_sequence)


def test_discrete_floors(discrete):
    cases, (st, runs) = discrete
    rs = collections.Counter((f, _lane(l)) for f, l, _ in st["resizes"])
    pend = collections.Counter((f, _lane(l)) for f, l, p in st["resizes"] if p > 0)
    print({k: v for k, v in st.items() if k != "resizes"}, dict(rs), dict(pend))
    for f in (5, 19, 77, 307):
        for lane in ("lane0", "mid", "lane31"):
            assert rs[(f, lane)] >= 1, "no resize at fill %d on %s" % (f, lane)
        assert pend[(f, "lane0")] >= 1 and pend[(f, "mid")] >= 1, "no resize at fill %d with staged keys pending" % f
    for bits in (4, 8):
        for kind in ("ems", "raw"):
            sel = [(r[2], r[3]) for c, r in zip(cases, runs) if c["kind"] == kind and ci.key_bits(c["cont"]) == bits]
            assert (False, ci.CAND_CAP) in sel, "%s, %d-bit keys: no list of exactly 1228 distinct keys" % (kind, 4 * bits)
            assert (True, ci.CAND_CAP + 1) in sel, "%s, %d-bit keys: no list of exactly 1229 distinct keys" % (kind, 4 * bits)
    assert any(n > ci.CAND_CAP + 1 and over for c, (_, _, over, n) in zip(cases, runs) if c["kind"] == "ems")
    assert st["window"] >= 1000 and st["wrap"] >= 1000 and st["perturb2"] >= 100 and st["perturb_max"] >= 4
    assert st["dup_in_chunk_lane0"] >= 100 and st["dup_in_chunk_lane31"] >= 100 and st["dup_across_chunks"] >= 1000
    r6 = collections.Counter()
    for c, (seq, _, _, _) in zip(cases, runs):
        a, b, z = c["item"]
        if c["R"] == 6 and seq:
            shape = "x=y=z" if a == b == z else "x=y" if a == b else "y=z" if b == z else "x=z" if a == z else "xyz"
            r6[shape] += 1
            r6["collapsed"] += len(set(ci.canon(c["item"], 6))) < 6
    print(dict(r6))
    for shape in ci.SHAPES:
        assert r6[shape] >= 5, "R = 6, %s: %d lists" % (shape, r6[shape])
    assert r6["collapsed"] >= 20
    conts = collections.Counter(c["cont"] for c, (seq, _, _, _) in zip(cases, runs) if seq)
    for side in (16, 17, 255):
        assert sum(v for k, v in conts.items() if k[0] == side) >= 20, "container of %d cells" % side


def _ulps_apart(t, u):
    return t != u and all(a == b or abs(a - b) <= 4 * math.ulp(max(abs(a), abs(b))) for a, b in zip(t, u))


def test_continuous_floors(continuous):
    cases, (st, runs) = continuous
    rs = collections.Counter((f, _lane(l)) for f, l, _ in st["resizes"])
    print({k: v for k, v in st.items() if k != "resizes"}, dict(rs))
    assert st["tag_probe"] >= 1 and st["tag_insert_same_chunk"] >= 1, "no tag match between distinct tuples"
    for f in (5, 19, 77, 307):
        assert rs[(f, "mid")] >= 1
    sel = [(over, n) for (_, _, over, n) in runs]
    assert (False, ci.CAND_CAP) in sel and (True, ci.CAND_CAP + 1) in sel
    zero_sign = near = equal_codes = past2200 = 0
    for seq, order, _, _ in runs:
        first = {}
        for r, t in seq:
            if t in first and first[t] != r:
                equal_codes += 1
                if ci.bits_of(t) != ci.bits_of(next(u for _, u in seq if u == t)):
                    zero_sign += 1
            first.setdefault(t, r)
        if len(order) < 300:
            near += sum(_ulps_apart(order[i], order[j]) for i in range(len(order)) for j in range(i))
        past2200 += any(v > 2200 for t in order for v in t)
    # value-equal tuples whose bits differ (0.0 / -0.0) collapse; tuples a few ulps apart (0.1 + 0.2 next to 0.3) stay distinct
    assert zero_sign >= 1 and near >= 10 and equal_codes >= 100 and past2200 >= 20, (zero_sign, near, equal_codes, past2200)
    edge_fit = edge_miss = 0
    apart = collections.Counter()
    for c in cases:
        for m in c["ems"]:
            for rot in range(c["R"]):
                sx = ci.rot_dims_c(c["item"], rot)[0]
                w = m[3] - m[0]
                lo, hi = math.nextafter(w, -math.inf) + 1e-6 >= sx, math.nextafter(w, math.inf) + 1e-6 >= sx
                if lo != hi:
                    edge_fit += w + 1e-6 >= sx
                    edge_miss += not (w + 1e-6 >= sx)
        if c["R"] == 6:
            a, b, z = c["item"]
            for d in (abs(a - b), abs(b - z), abs(a - z)):
                for name, v in (("0", 0.0), ("5e-7", 5e-7), ("2e-6", 2e-6)):
                    apart[name] += abs(d - v) < 1e-9
                if abs(d - 1e-6) < 1e-9:
                    apart["1e-6 kept" if not d < 1e-6 else "1e-6 skipped"] += 1
    print(edge_fit, edge_miss, dict(apart))
    assert edge_fit >= 5 and edge_miss >= 5, (edge_fit, edge_miss)
    for k in ("0", "5e-7", "2e-6", "1e-6 kept", "1e-6 skipped"):
        assert apart[k] >= 2, "item sides %s apart: %d" % (k, apart[k])
