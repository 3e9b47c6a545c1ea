"""Heuristic baselines on containers other than 10x10x10, on both sides of the 32-cell side where HM / MACS / RANDOM switch to the
large-container instantiation of the selection kernel (DESIGN.md section 14).

CPU: the restatement (oracle/pct_oracle_heuristics.py) replays the reference's unmodified heuristic.py recorded on 20x18x24 and
40x36x16 (tests/golden/heur_case_*.npz, tests/golden/make_heuristic_golden_cases.py).
GPU: the batched kernel replays the same records, and agrees with the restatement step by step on device-drawn items on 40x36x16,
an asymmetric 33x200 bin and the 255x255x255 limit container."""
import glob
import os

import numpy as np
import pytest

import pct_oracle_heuristics as OH
from harness import case_stream
from pct_oracle import OracleDiscrete
from test_heuristics import dataset_stream

# OracleDiscrete takes the env's size_minimum explicitly: below it is np.min(item_set), as in the reference (D:bin3D.py:23) and PctBatch

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "heur_case_*.npz")))
RECORDED = ("LSAH", "OnlineBPH", "BR", "MACS", "DBL", "HM")
BIG40_ITEMS = [(i, j, k) for i in (3, 7, 12) for j in (4, 9) for k in (3, 8, 11)]
# the limit container: large items, so that the height-map sums and the MACS histograms reach their ranges in few steps
LIMIT = (255, 255, 255)
LIMIT_ITEMS = [(255, 255, 255), (250, 60, 6), (40, 40, 5), (200, 180, 120), (90, 240, 100)]


def golden(path, name):
    g = np.load(path)
    off = np.concatenate([[0], np.cumsum(g["len_" + name])])
    items = [tuple(int(v) for v in it) for it in g["items"]]
    packed = [g["flat_" + name][off[i]:off[i + 1]].tolist() for i in range(len(off) - 1)]
    return int(g["setting"]), tuple(int(c) for c in g["container"]), items, g["data"], packed


def _id(path):
    return os.path.basename(path)[len("heur_case_"):-len(".npz")]


def test_golden_cases_present():
    names = [_id(p) for p in GOLDEN]
    assert names == ["big40_s1", "big40_s2", "big40_s3", "big_s1", "big_s2", "big_s3"]
    for p in GOLDEN:  # both sides of the 32-cell side of the static height map
        assert (max(np.load(p)["container"][:2]) > 32) == _id(p).startswith("big40")


@pytest.mark.parametrize("name", RECORDED)
@pytest.mark.parametrize("path", GOLDEN, ids=_id)
def test_restated_heuristics_replay_reference_cases(path, name):
    setting, container, items, data, packed = golden(path, name)
    env = OracleDiscrete(setting, container_size=container, size_minimum=min(map(min, items)), stream=dataset_stream(data, 0, len(packed) + 1))
    env.set_trajectory_length(data.shape[1] + 1)
    rec = OH.run_episodes(name, env, len(packed), item_set=items)
    assert [r[2] for r in rec] == packed


# ---- GPU --------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", RECORDED)
@pytest.mark.parametrize("path", GOLDEN, ids=_id)
def test_batched_heuristic_replays_reference_cases(path, name):
    """dataset mode, 2 envs sharing the episodes: packed lists, mean, variance and length equal the unmodified reference's"""
    from pct_b200.heuristics import run_heuristic
    setting, container, items, data, packed = golden(path, name)
    (mean, var, length), rec = run_heuristic(name, setting, len(packed), container_size=container, item_set=items, data=list(data),
                                             n_envs=2, return_episodes=True)
    assert rec["packed"] == packed
    ratios = [sum(p[0] * p[1] * p[2] for p in ep) / float(np.prod(container)) for ep in packed]
    assert abs(mean - np.mean(ratios)) < 1e-12 and abs(var - np.var(ratios)) < 1e-12 and length == np.mean([len(ep) for ep in packed])


def lockstep(name, setting, container, items, n_envs, steps, seed=5, prefix=None):
    """n_envs envs on the device next to one oracle env each on the same items: at every step the kernel's action row equals the
    restatement's choice, and both step with it (episodes end and restart alike).  No step raises a flag other than the one of the
    "no feasible placement" row.  Items: drawn by the device generator from `items`; with prefix (one list of items per env), each
    env's stream starts with its prefix and continues with those draws.  -> the placements made (restatement choices)."""
    from pct_b200 import PctBatch
    case = dict(setting=setting, items=items)
    streams = [case_stream(case, seed, e, 400) for e in range(n_envs)]
    if prefix:
        for e, pre in enumerate(prefix):
            streams[e][:len(pre), :3] = pre
    b = PctBatch(n_envs, setting, container_size=container, item_set=items, seed=seed, item_stream=np.stack(streams) if prefix else None)
    envs = [OracleDiscrete(setting, container_size=container, size_minimum=min(map(min, items)), stream=s) for s in streams]
    states = [OH.fresh_state(container) for _ in envs]
    b.reset()
    for env in envs:
        env.reset()
    placed = []
    for t in range(steps):
        rows = b.heuristic_actions(name, seed=seed, t=t)
        got = rows.cpu().numpy()
        choices = [OH.choose(name, env, states[e], items, seed, e, t) for e, env in enumerate(envs)]
        for e, c in enumerate(choices):
            assert np.array_equal(got[e], OH.action_row(c, container).astype(np.float32)), (name, container, t, e, got[e], c)
        _, _, done, info = b.step(actions=rows)
        PctBatch.check_flags(PctBatch.decode_info(info)["flags"], ignore=2, what="lockstep")
        done = done.cpu().numpy().astype(bool)
        for e, (env, c) in enumerate(zip(envs, choices)):
            _, _, d, _ = env.step(OH.action_row(c, container))
            assert bool(d) == done[e], (name, t, e)
            if c is not None:
                OH.note_placement(states[e], c)
                placed.append(c)
            if d:
                env.reset()
                states[e] = OH.fresh_state(container)
    b.close()
    return placed


@pytest.mark.gpu
@pytest.mark.parametrize("name,setting", [("HM", 1), ("HM", 2), ("MACS", 1), ("MACS", 2), ("RANDOM", 1), ("RANDOM", 2), ("RANDOM", 3),
                                          ("DBL", 2), ("LSAH", 1)])
def test_device_items_big40(name, setting):
    """40 x 36 x 16: device-drawn items, 4 envs against the restatement over a whole episode and into the next"""
    assert len(lockstep(name, setting, (40, 36, 16), BIG40_ITEMS, 4, 60)) > 100


@pytest.mark.gpu
@pytest.mark.parametrize("name,setting,steps", [("HM", 1, 30), ("MACS", 2, 30), ("RANDOM", 2, 15), ("DBL", 1, 30)])
def test_device_items_asymmetric(name, setting, steps):
    """33 x 200 x 12: one side just above 32, the other far above: a map indexed with W and L swapped disagrees at once.  RANDOM scatters
    its boxes, so after 15 steps its EMS and candidate lists approach the env's capacities (128 EMS, 1228 candidates): it stops there."""
    assert len(lockstep(name, setting, (33, 200, 12), BIG40_ITEMS, 2, steps)) >= steps


@pytest.mark.gpu
@pytest.mark.parametrize("name,setting", [("HM", 1), ("HM", 2), ("DBL", 2), ("RANDOM", 1), ("RANDOM", 2), ("MACS", 1)])
def test_device_items_limit_container(name, setting):
    """255 x 255 x 255, the first steps.  Env 0 starts with the 255^3 item: its only placement fills the bin, the HM score of 100 * 255^3
    and a height-map sum of 255^3.  Env 1 starts with a 250 x 60 slab: the MACS candidates on top of it see histogram columns of 255
    free cells.  RANDOM bitmaps hold up to 216 * 216 * 6 bits."""
    prefix = [[(255, 255, 255)], [(250, 60, 6), (40, 40, 5)]]
    assert len(lockstep(name, setting, LIMIT, LIMIT_ITEMS, 2, 3, prefix=prefix)) >= 3


@pytest.mark.gpu
def test_random_chooses_among_all_feasible_placements():
    """64 x 64 x 16, setting 2, empty bins, a 3 x 4 x 5 item: 62 * 61 * 6 = 22692 feasible placements, beyond the 6144-bit bitmap of the
    static instantiation (lx <= 16).  Over 32 envs the kernel picks what the restatement picks among all of them."""
    placed = lockstep("RANDOM", 2, (64, 64, 16), [(3, 4, 5)], 32, 1, seed=11)
    assert len(placed) == 32 and max(c[1] for c in placed) > 16


class _View(object):
    """the env surface pct_oracle_heuristics.choose reads, served by the single-env facade the way heuristic.py calls it"""

    def __init__(self, env):
        self.env, self.container, self.setting = env, tuple(env.bin_size), env.setting

    def ems(self):
        return [[int(v) for v in e] for e in self.env.space.EMS]

    def drop_box_virtual(self, d, lx, ly):
        return self.env.space.drop_box_virtual(list(d), (lx, ly), False, self.env.next_den, self.env.setting, returnH=True)

    def plain(self):
        return np.array(self.env.space.plain)

    @property
    def next_box(self):
        return self.env.next_box


def _facade(path, tmp_path):
    import torch
    import pct_b200
    setting, container, items, data, _ = golden(path, "HM")
    ds = os.path.join(str(tmp_path), "set.pt")
    torch.save([t.tolist() for t in data], ds)
    env = pct_b200.PackingDiscrete(setting=setting, container_size=list(container), item_set=items, data_name=ds, load_test_data=True)
    return env, setting, container, items, data


@pytest.mark.gpu
def test_facade_queries_on_a_wide_bin(tmp_path):
    """40 x 36: space.drop_box_virtual (returnH, returnMap) and space.plain equal the oracle's, along an episode and at positions
    around and outside the bin"""
    path = [p for p in GOLDEN if _id(p) == "big40_s1"][0]
    env, setting, container, items, data = _facade(path, tmp_path)
    _, _, _, _, packed = golden(path, "DBL")
    ora = OracleDiscrete(setting, container_size=container, size_minimum=min(map(min, items)), stream=dataset_stream(data, 0, 2))
    ora.set_trajectory_length(data.shape[1] + 1)
    env.reset()
    ora.reset()
    rng = np.random.default_rng(3)
    W, L, _ = container
    for p in packed[0][:25]:
        plain = np.array(ora.plain())
        assert np.array_equal(np.array(env.space.plain), plain)
        for _ in range(20):
            d = [int(v) for v in rng.choice([3, 4, 7, 9, 11, 12], 3)]
            lx, ly = int(rng.integers(-2, W + 2)), int(rng.integers(-2, L + 2))
            ok, h = ora.drop_box_virtual(d, lx, ly)
            assert env.space.drop_box_virtual(d, (lx, ly), False, env.next_den, setting, returnH=True) == (ok, h)
            feas, hmap = env.space.drop_box_virtual(d, (lx, ly), False, env.next_den, setting, False, True)
            if 0 <= lx < W and 0 <= ly < L:  # update_height_graph on a copy: the footprint inside the bin becomes rest height + z
                want = plain.copy()
                want[lx:lx + d[0], ly:ly + d[1]] = h + d[2]
                assert feas == ok and np.array_equal(hmap, want)
        env.next_box = list(p[:3])
        env.step([0, p[3], p[4]])
        ora.step(np.array([p[3], p[4], 0, p[3] + p[0], p[4] + p[1], 0, 0, 0, 1.0]))
    env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,episodes", [("LSAH", 2), ("HM", 1)])
def test_facade_serves_the_reference_heuristic_loop_on_a_wide_bin(name, episodes, tmp_path):
    """env.space.drop_box_virtual / env.space.EMS / env.space.plain / env.next_box = [...] / env.step([0, lx, ly]) on a 40 x 36
    PackingDiscrete replay the reference's records (HM: one episode, as it asks one synchronous query per grid placement)"""
    path = [p for p in GOLDEN if _id(p) == "big40_s1"][0]
    env, setting, container, items, data = _facade(path, tmp_path)
    _, _, _, _, packed = golden(path, name)
    view = _View(env)
    env.reset()
    state, got = OH.fresh_state(view.container), []
    while len(got) < episodes:
        c = OH.choose(name, view, state, items)
        if c is None:
            got.append(env.packed)
            env.reset()
            state = OH.fresh_state(view.container)
            continue
        env.next_box = c[0]
        env.step([0, c[1], c[2]])
        OH.note_placement(state, c)
    assert got == packed[:episodes]
    env.close()
