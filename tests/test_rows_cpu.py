"""Action rows the leaf list never proposes (tests/rows_rule.py), replayed on the oracle against the records of the unmodified reference
(tests/golden/rows_*.npz, tests/golden/make_golden_rows.py): box corners and arbitrary points in every orientation LeafNode2Action can
express, the zero row, fractional / zero-sum / equal-side / out-of-range discrete rows, continuous extents that match no side or sit at
the 1e-6 match tolerance, positions at and just past the container walls.  Discrete and continuous float64 rows bit for bit; float32
continuous rows with identical discrete outcomes and coordinates within 1e-6 (as tests/test_f32_rows.py); error 2 on exactly the steps
where the reference raised.  The counts of what the records exercise are re-derived here and must reach rows_rule.MIN_COUNTS."""
import glob
import os

import numpy as np
import pytest

from rows_rule import MIN_COUNTS, RAISING, make_oracle, oracle_counts_step

G = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "rows_*.npz")))
TOL = 1e-6


def test_files_present():
    assert len(G) == 15


def _same(o, ref, f32, what):
    if not f32:
        assert np.array_equal(o, ref), "%s: observation differs at %s" % (what, np.argwhere(o != ref)[:4].tolist())
        return
    a, b = o.reshape(-1, 9), ref.reshape(-1, 9)
    assert np.array_equal(a[:, 6:9], b[:, 6:9]), "%s: valid / feasibility flags differ" % what
    assert np.abs(o - ref).max() <= TOL, "%s: coordinates differ by %g" % (what, np.abs(o - ref).max())


def replay(g, counts=None):
    """replay one record on the oracle; returns the oracle's step results"""
    orc = make_oracle(g)
    f32 = g["rows"].dtype == np.float32
    obs, k = g["obs"], 0
    nb, nl = int(g["nb"]), int(g["nl"])
    o = orc.reset()
    assert np.array_equal(o, obs[k]); k += 1
    for t in range(len(g["rows"])):
        row = g["rows"][t].astype(np.float64)
        lb = orc.n_lstsq
        res = orc.step(row)
        o2, r, d, info = res
        w = "%s step %d (%s)" % (g["name"], t, g["kind"][t])
        raised = bool(g["err"][t])
        assert (info.get("error") == 2) == raised, "%s: oracle error %s, reference raised %r" % (w, info.get("error"), str(g["err"][t]))
        assert info.get("error") in (None, 2), w
        assert d == bool(g["done"][t]), w
        if counts is not None:
            for kk, v in oracle_counts_step(orc, row, o, res, nb, nl, lb).items():
                counts[kk] += v
            counts["raised"] += int(raised)
        if not raised:
            _same(o2, obs[k], f32, w); k += 1
            assert info["counter"] == g["counter"][t], w
            assert (r == g["reward"][t]) if not f32 else abs(r - g["reward"][t]) <= 1e-6, "%s: reward %r, reference %r" % (w, r, g["reward"][t])
            if d:
                assert (info["ratio"] == g["ratio"][t]) if not f32 else abs(info["ratio"] - g["ratio"][t]) <= 1e-6, w
        o = orc.reset() if d else o2
        if d:
            assert np.array_equal(o, obs[k]), "%s: reset observation" % w
            k += 1
    assert k == len(obs)


@pytest.mark.parametrize("path", G, ids=[os.path.basename(p)[5:-4] for p in G])
def test_oracle_follows_the_reference_on_rows_of_its_own(path):
    replay(np.load(path))


def test_the_records_exercise_what_they_claim():
    tot = dict(failed_with_loads=0, offleaf_multi=0, lstsq=0, raised=0)
    raised_kinds = set()
    for p in G:
        g = np.load(p)
        c = dict(failed_with_loads=0, offleaf_multi=0, lstsq=0, raised=0)
        replay(g, c)
        for k, v in c.items():
            assert v == int(g["counts_" + k]), "%s: %s %d, the file says %d" % (p, k, v, int(g["counts_" + k]))
            tot[k] += v
        raised_kinds |= {str(k) for k, e in zip(g["kind"], g["err"]) if e}
    print("rows records:", tot, "raising kinds", sorted(raised_kinds))
    for k, v in MIN_COUNTS.items():
        assert tot[k] >= v, (k, tot[k], v)
    assert raised_kinds == set(RAISING)
