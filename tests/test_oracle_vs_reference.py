"""CPU: lock-step of the C oracle against the unmodified Python reference (every observation including terminal ones, reward, done,
info), replayed from what the reference produced: tests/golden/reference_lockstep.npz, recorded by tests/golden/make_reference_lockstep.py."""
import json
import os
import sys

import numpy as np
import pytest

from harness import ITEM_SET, make_stream, policy_pick
from pct_oracle import OracleDiscrete

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from harness import CASES, CONT_CASES  # noqa: E402
from make_reference_lockstep import CASE_STEPS, CONT_CASE_STEPS, LOCKSTEP_STEPS, TIE_ENV, TIE_SEED, TIE_STEPS, info_text, obs_digest  # noqa: E402

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_lockstep.npz"))


@pytest.mark.parametrize("setting", [1, 2, 3])
def test_lockstep_with_reference(setting):
    ref = {k: G["lockstep_s%d_%s" % (setting, k)] for k in ("obs", "reward", "done", "info")}
    seed, env_id = 900 + setting, 3
    orc = OracleDiscrete(setting, stream=make_stream(seed, env_id, LOCKSTEP_STEPS + 64, setting))
    o = orc.reset()
    k = 0
    for t in range(LOCKSTEP_STEPS):
        assert obs_digest(o) == ref["obs"][k], t
        _, row = policy_pick(o, 80, 50, seed, env_id, t)
        o, r, d, i = orc.step(row)
        k += 1
        assert obs_digest(o) == ref["obs"][k], "observation after step %d (done=%s)" % (t, d)
        assert (r, d) == (ref["reward"][t], ref["done"][t]) and json.loads(info_text(i)) == json.loads(str(ref["info"][t]))
        if d:
            o = orc.reset()
            k += 1
    assert k == len(ref["obs"]) - 1


# ---- other configurations on fresh seeds (the committed full records of the same configurations are tests/golden/case_*.npz) ----
def _lockstep_record(orc, c, seed, env_id, steps):
    o = orc.reset()
    obs, rew, done, counter, ratio = [obs_digest(o)], [], [], [], []
    for t in range(steps):
        _, row = policy_pick(o, c["nb"], c["nl"], seed, env_id, t)
        o, r, d, info = orc.step(row)
        obs.append(obs_digest(o)); rew.append(r); done.append(d); counter.append(info["counter"]); ratio.append(info.get("ratio", -1.0))
        if d:
            o = orc.reset()
            obs.append(obs_digest(o))
    return dict(obs=np.array(obs), reward=np.array(rew), done=np.array(done), counter=np.array(counter), ratio=np.array(ratio))


def _equal_records(a, b):
    for k in ("obs", "reward", "done", "counter", "ratio"):
        assert np.array_equal(a[k], b[k]), k


@pytest.mark.parametrize("name", sorted(CASES))
def test_cases_lockstep_with_reference(name):
    """the recorder of tests/golden/make_golden_cases.py on the reference vs the same loop on the oracle, new seed"""
    from harness import case_stream
    c = dict(CASES[name], steps=CASE_STEPS)
    orc = OracleDiscrete(c["setting"], container_size=c["container"], internal_node_holder=c["nb"], leaf_node_holder=c["nl"],
                         size_minimum=min(min(i) for i in c["items"]), stream=case_stream(c, 8800, 4, c["steps"] + 64), lnes=c["lnes"])
    got = _lockstep_record(orc, c, c.get("pseed", 8800), 4, c["steps"])
    _equal_records({k: G["case_%s_%s" % (name, k)] for k in got}, got)


@pytest.mark.parametrize("name", sorted(CONT_CASES))
def test_continuous_cases_lockstep_with_reference(name):
    from harness import cont_case_stream
    from pct_oracle import OracleContinuous
    c = dict(CONT_CASES[name], steps=CONT_CASE_STEPS)
    orc = OracleContinuous(c["setting"], container_size=c["container"], internal_node_holder=c["nb"], leaf_node_holder=c["nl"],
                           size_minimum=c["low"], stream=cont_case_stream(c, 8801, 5, c["steps"] + 64))
    got = _lockstep_record(orc, c, 8801, 5, c["steps"])
    _equal_records({k: G["ccase_%s_%s" % (name, k)] for k in got}, got)


def test_the_known_divergence_is_lapack_rounding_at_a_geometric_tie():
    """The one disagreement a 130k-env-step fresh-seed soak found (setting 1, seed 135409): a 4x2x1 item resting on three boxes whose
    common edge passes exactly under its centre of mass -> no direct edge -> np.linalg.lstsq (LAPACK gelsd) splits the load.  The oracle's
    solver agrees with gelsd to 4e-16, but the next box's centre of mass then lies exactly ON the border between two of ITS supports, and
    the strict `centre > area` tests (D:space.py:186-187) are decided by that last bit.  Demonstrated on the reference's own code when the
    record was made: fed the oracle solver's solution instead of LAPACK's, ITS verdict flips too.  (gelsd's last bits depend on the BLAS
    build, so this tie is not reproducible across machines even by the reference itself.)"""
    from harness import case_stream
    c = CASES["holders_s1"]
    orc = OracleDiscrete(1, internal_node_holder=c["nb"], leaf_node_holder=c["nl"], stream=case_stream(c, TIE_SEED, TIE_ENV, 200))
    o = orc.reset()
    for t in range(TIE_STEPS):
        assert obs_digest(o) == G["tie_pre"][t], t
        _, row = policy_pick(o, c["nb"], c["nl"], TIE_SEED, TIE_ENV, t)
        o, _, d, _ = orc.step(row)
        if d:
            o = orc.reset()
    assert not G["tie_with_lapack"][0]  # LAPACK's last bits: infeasible
    if obs_digest(o) != G["tie_final"][0]:  # on this machine's BLAS the tie falls the other way for the oracle: the documented divergence
        gap = G["tie_solver_gap"]
        assert G["tie_with_oracle_solver"][0] and len(gap) == 1 and 0 < gap[0] < 1e-15
