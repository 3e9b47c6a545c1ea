"""LNES='EVM' on the CPU: the model of tests/evm_oracle.py against records of the reference (tests/golden/make_golden_evm.py)."""
import hashlib
import os
import re

import numpy as np
import pytest

from evm_cases import EVM_CASES
from evm_oracle import EvmOracle, FLAG_CAND_OVERFLOW, zmap

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = np.load(os.path.join(HERE, "golden", "evm_golden.npz"))


def _rec(name):
    return {k.split("/", 1)[1]: GOLD[k] for k in GOLD.files if k.startswith(name + "/")}


def _zmap_at(rec, i):
    z = rec["zmap"][rec["zmap_off"][i]:rec["zmap_off"][i + 1]].tolist()
    out, p = {}, 1
    for _ in range(z[0]):
        k, n = z[p], z[p + 1:p + 5]
        p += 5
        lists = []
        for m in n:
            lists.append(z[p:p + m])
            p += m
        out[k] = tuple(lists)
    return out


def _replay(c, rec):
    """-> [(obs, ZMAP, flags)] of the model along the recorded rows"""
    m = EvmOracle(c["setting"], c["container"], c["nb"], c["nl"], stream=rec["stream"])
    o = m.reset()
    out = [(o, m.zmap(), m.flags)]
    for row in rec["rows"]:
        o, _, d, _ = m.step(row)
        if d:
            o = m.reset()
        out.append((o, m.zmap(), m.flags))
    return out


@pytest.mark.parametrize("name", sorted(EVM_CASES))
def test_model_matches_reference(name):
    """every observation before the capacity limit is the reference's, byte for byte; the ZMAP derived from the boxes is the reference's"""
    c, rec = EVM_CASES[name], _rec(name)
    ov = int(rec["overflow_step"])
    states = _replay(c, rec)
    assert len(states) == len(rec["digest"])
    for t, (o, Z, fl) in enumerate(states):
        assert [list(map(list, r)) for r in Z.values()] == [list(map(list, r)) for r in _zmap_at(rec, t).values()], (name, t)
        assert list(Z) == list(_zmap_at(rec, t)), (name, t)
        if t == ov:
            assert fl & FLAG_CAND_OVERFLOW, (name, t)
            break
        assert fl == 0, (name, t)
        leaves = o.reshape(-1, 9)[c["nb"]:c["nb"] + c["nl"], :5].astype(np.int16)
        assert np.array_equal(leaves, rec["leaves"][t]), (name, t)
        assert hashlib.sha1(np.ascontiguousarray(o, dtype=np.float64).tobytes()).digest() == rec["digest"][t].tobytes(), (name, t)


def test_records_reach_the_limit_and_leave_the_corners():
    """the records hold a stream crossing the per-level set limit, and EVM offers placements EV cannot (above z = 0, off the corners)"""
    assert any(int(_rec(n)["overflow_step"]) >= 0 for n in EVM_CASES)
    assert any(int(_rec(n)["overflow_step"]) < 0 for n in EVM_CASES if EVM_CASES[n]["setting"] == 2)
    rec = _rec("s1_10")
    lv = rec["leaves"].reshape(-1, 5)
    assert (lv[:, 2] > 0).any() and ((lv[:, 0] > 0) & (lv[:, 3] < 10)).any()


def test_zmap_derivation_rules():
    """start state, bottom and top upkeep, the W / L exclusions, sorted lists and key order"""
    assert zmap([], 10, 8, 6) == {0: ([0], [0], [10], [8])}
    Z = zmap([(0, 0, 0, 10, 3, 2), (2, 3, 0, 5, 8, 4), (1, 0, 2, 4, 3, 6)], 10, 8, 6)
    assert list(Z) == [0, 2, 4]
    assert Z[0] == ([0, 5], [0, 3], [0, 2, 10], [0, 3, 8])
    assert Z[2] == ([0, 4], [0, 3], [1, 10], [0, 3])
    assert Z[4] == ([2], [3], [5], [8])


def test_code_and_abi():
    import pct_b200._lib as L
    assert L.LNES_CODES["EVM"] == 5 and L.LNES_CODES["EV"] == 1
    h = open(os.path.join(ROOT, "include", "pct_b200.h")).read()
    assert re.search(r"PCT_LNES_EVM\s*=\s*5", h)
