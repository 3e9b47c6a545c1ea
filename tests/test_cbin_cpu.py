"""CPU: the continuous env on containers other than the unit cube (harness.CONT_BINS).  The C oracle and the restated baselines must
reproduce the records of the unmodified reference (tests/golden/cbin_*.npz, tests/golden/make_cbin_golden.py) exactly: step trajectories,
heuristic episodes and Space.drop_box_virtual answers.  The coverage checks keep the records doing what they are for: the millimetre bin
reaches the exact-division branch of the 6-decimal rounding, the pallet's baselines place boxes against both side walls, and every
baseline ends an episode on "no placement"."""
import glob
import os

import numpy as np
import pytest

import pct_oracle_heuristics as OH
from harness import CONT_BINS, cont_item_set
from pct_oracle import OracleContinuous

G = os.path.join(os.path.dirname(__file__), "golden")
PATHS = sorted(glob.glob(os.path.join(G, "cbin_*.npz")))
IDS = [os.path.basename(p)[5:-4] for p in PATHS]
NAMES = ("LSAH", "OnlineBPH", "BR")


def load(name):
    """-> (case, record) of cbin_<name>.npz"""
    return CONT_BINS[name], np.load(os.path.join(G, "cbin_%s.npz" % name))


def oracle(c, stream):
    return OracleContinuous(c["setting"], container_size=c["container"], internal_node_holder=c["nb"], leaf_node_holder=c["nl"],
                            size_minimum=c["low"], stream=stream)


def trajectory(g, k):
    return {f: g["t%d_%s" % (k, f)] for f in ("stream", "rows", "obs", "reward", "done", "counter", "ratio")}


def episodes(g, name):
    off = np.concatenate([[0], np.cumsum(g["len_" + name])])
    return [g["flat_" + name][off[i]:off[i + 1]].tolist() for i in range(len(off) - 1)]


def test_files_present():
    assert IDS == sorted(CONT_BINS) and sum(os.path.getsize(p) for p in PATHS) < 1200 * 1024


@pytest.mark.parametrize("name", IDS)
def test_oracle_replays_the_trajectories(name):
    c, g = load(name)
    for k in (0, 1):
        tr = trajectory(g, k)
        env, obs, j = oracle(c, tr["stream"]), tr["obs"], 0
        assert np.array_equal(env.reset(), obs[j]), "t%d reset" % k
        j += 1
        for t in range(len(tr["rows"])):
            o, r, d, info = env.step(tr["rows"][t])
            assert np.array_equal(o, obs[j]), "t%d observation after step %d (done=%s)" % (k, t, d)
            j += 1
            assert r == tr["reward"][t] and d == bool(tr["done"][t]) and info["counter"] == tr["counter"][t] and "error" not in info, (k, t)
            if d:
                assert info["ratio"] == tr["ratio"][t]
                assert np.array_equal(env.reset(), obs[j]), "t%d observation after the reset following step %d" % (k, t)
                j += 1
        assert j == len(obs)
    assert g["t0_done"].any() and g["t1_done"].any(), "each trajectory finishes an episode"


@pytest.mark.parametrize("name", IDS)
def test_restated_baselines_replay_the_records(name):
    c, g = load(name)
    for h in NAMES:
        want = episodes(g, h)
        got = OH.run_episodes(h, oracle(c, g["h_stream"]), len(want), item_set=cont_item_set(c))
        assert [e[2] for e in got] == want, h
        assert max(len(e) for e in want) < c["nb"], "an episode reached the box holder"


@pytest.mark.parametrize("name", IDS)
def test_oracle_answers_the_recorded_queries(name):
    c, g = load(name)
    tr = trajectory(g, 0)
    env = oracle(c, tr["stream"])
    env.reset()
    n = 0
    for t in range(len(tr["rows"])):
        for i in np.nonzero(g["q_step"] == t)[0]:
            x = g["q"][i]
            assert env.next_den == g["q_den"][i]
            assert env.drop_box_virtual(x[:3], x[3], x[4]) == (bool(g["q_feas"][i]), float(g["q_h"][i])), (t, i, x)
            n += 1
        if env.step(tr["rows"][t])[2]:
            env.reset()
    assert n == len(g["q"]) and len(set(g["q_step"].tolist())) >= 10
    assert g["q_feas"].any() and not g["q_feas"].all() and (g["q_h"] > 0).any()


# ---- coverage ------------------------------------------------------------------------------------------------------------------------
def _tolerance_split(g, c, axis):
    """for the probes of one axis (0: lx + sx vs W, 1: ly + sy vs L) at a 0 / 5e-7 / 2e-6 distance: the verdicts at the wall and 5e-7
    outside of it must be feasible ones at least once, 2e-6 outside never"""
    W = c["container"][axis]
    end = g["q"][:, 3 + axis] + g["q"][:, axis]
    over = end - W
    inside = g["q_feas"][np.abs(over) < 1e-9].any() and g["q_feas"][np.abs(over - 5e-7) < 1e-9].any()
    outside = not g["q_feas"][np.abs(over - 2e-6) < 1e-9].any() and (np.abs(over - 2e-6) < 1e-9).any()
    return inside, outside


@pytest.mark.parametrize("name", IDS)
def test_queries_hit_the_tolerances_on_each_axis(name):
    c, g = load(name)
    for axis in (0, 1):
        assert _tolerance_split(g, c, axis) == (True, True), "axis %d" % axis
    top = g["q_h"] + g["q"][:, 2]
    H = c["container"][2]
    assert (np.abs(top - H) < 1e-9).any() and not g["q_feas"][np.abs(top - H - 2e-6) < 1e-9].any()
    assert ((g["q"][:, 3] < 0) & (g["q"][:, 3] > -1e-6) & g["q_feas"]).any()
    assert (g["q"][:, :3] == 0).any(1).sum() >= 30


def test_mm_bin_reaches_the_exact_division():
    """coordinates above 2200 (|v| * 1e6 > 2.2e9): around6 divides exactly there (csrc/pct_geom_continuous.cuh).  Every mm record places
    boxes whose x + dx is past 2200 and has EMS corners past 2200 (the walls x = 2400 and z = 2300, which GENEMS rounds like any
    intersection); at least one record also has an EMS corner past 2200 strictly inside the bin (a box's face)."""
    inner = 0
    for setting in (1, 2, 3):
        c, g = load("mm_s%d" % setting)
        far = ems_far = 0
        for k in (0, 1):
            tr = trajectory(g, k)
            boxes = tr["obs"].reshape(len(tr["obs"]), -1, 9)[:, :c["nb"]]
            far += int((boxes[:, :, 3] > 2200).sum())
            env = oracle(c, tr["stream"])
            env.reset()
            for t in range(len(tr["rows"])):
                e = env.ems()
                ems_far += int((e > 2200).any(1).sum())
                inner += int(((e > 2200) & (e < np.array(c["container"] * 2))).sum())
                if env.step(tr["rows"][t])[2]:
                    env.reset()
        assert far > 0 and ems_far > 0, (setting, far, ems_far)
    assert inner > 0


@pytest.mark.parametrize("setting", [1, 2, 3])
def test_pallet_baselines_touch_both_walls(setting):
    c, g = load("pallet_s%d" % setting)
    W, L = c["container"][:2]
    p = np.concatenate([g["flat_" + h] for h in NAMES])
    assert (np.abs(p[:, 0] + p[:, 3] - W) < 1e-9).any(), "no chosen placement touches x = W"
    assert (np.abs(p[:, 1] + p[:, 4] - L) < 1e-9).any(), "no chosen placement touches y = L"


@pytest.mark.parametrize("name", IDS)
def test_every_baseline_ends_an_episode_on_no_placement(name):
    c, g = load(name)
    items = cont_item_set(c)
    for h in NAMES:
        env = oracle(c, g["h_stream"])
        env.reset()
        state, ends, n_ep = OH.fresh_state(env.container), [], len(g["len_" + h])
        while len(ends) < n_ep:
            ch = OH.choose(h, env, state, items)
            d = env.step(OH.action_row(ch, env.container, True))[2]
            if ch is not None:
                OH.note_placement(state, ch)
            if d:
                ends.append(ch is None)
                env.reset()
                state = OH.fresh_state(env.container)
        assert any(ends), h
