"""CPU: the buffered baselines (tests/buffer_heuristics.py; DESIGN.md section 22) against the plain oracle baseline, and the B-sentinel
padding of the dataset streams (pct_b200.evaluation._streams) that lets a buffered env play a trajectory dataset."""
import numpy as np
import pytest

import pct_oracle_heuristics as H
from buffer_heuristics import LOWER, RowBufferedOracle, buffered_choose
from buffer_oracle import config
from harness import CONT_ITEM_SET, ITEM_SET

DISC = ("LSAH", "OnlineBPH", "BR", "MACS", "DBL", "HM", "RANDOM")
CONT = ("LSAH", "OnlineBPH", "BR")
SEED, ENV = 5, 3


def _run(name, cfg, B, steps):
    """steps of the buffered baseline on a RowBufferedOracle of configuration `cfg`; yields, before every step, (t, model, its items, LSAH
    state, slot, choice, per-slot choices, scores, ranks, item set)"""
    c, mk = config(cfg, nl=50)
    items = CONT_ITEM_SET if c["domain"] == "continuous" else ITEM_SET
    m = RowBufferedOracle(c, mk(SEED, ENV, 600), B)
    m.reset()
    for t in range(steps):
        buf = m.buf.copy()
        state = {"max": list(m.hstate["max"]), "min": list(m.hstate["min"])}
        out = buffered_choose(name, m.orc, buf, state, items, SEED, ENV, t)
        yield (t, m, buf, state) + tuple(out) + (items,)
        slot, row, _, _, _ = m.heuristic(name, items, SEED, ENV, t)
        assert slot == out[0]
        m.step_row(slot, row)


@pytest.mark.parametrize("cfg,name", [("d", n) for n in DISC] + [("c", n) for n in CONT])
@pytest.mark.parametrize("setting", [1, 2, 3])
def test_b1_is_the_plain_choice(cfg, name, setting):
    """B = 1: the buffered choice is the plain `choose` for the slot's item, on every step of a buffered run"""
    for t, m, buf, state, slot, c, _, _, _, items in _run(name, "%s%d" % (cfg, setting), 1, 14):
        m.orc.set_next(buf[0])
        assert slot == 0
        assert c == H.choose(name, m.orc, state, items, SEED, ENV, t), "step %d" % t


@pytest.mark.parametrize("B", [3, 16])
@pytest.mark.parametrize("cfg,name", [("d1", n) for n in DISC] + [("d2", "LSAH"), ("d2", "HM"), ("c1", "LSAH"), ("c2", "OnlineBPH"), ("c3", "BR")])
def test_the_chosen_slot_is_the_best(cfg, name, B):
    """B = 3 / 16: the chosen slot is the best under the stated rule (ties to the lowest slot), and its row is the plain choice for its item"""
    steps = 10 if B == 16 else 16
    seen_choice = False
    for t, m, buf, state, slot, c, choices, scores, ranks, items in _run(name, cfg, B, steps):
        live = [j for j in range(B) if choices[j] is not None]
        if not live:
            assert slot == 0 and c is None
            continue
        seen_choice = True
        assert slot in live
        m.orc.set_next(buf[slot])
        assert c == H.choose(name, m.orc, state, items, SEED, ENV, t) == choices[slot]
        if name == "RANDOM":
            continue
        key = ranks if name == "OnlineBPH" else scores
        best = min(key[j] for j in live) if name in LOWER + ("OnlineBPH",) else max(key[j] for j in live)
        assert key[slot] == best and all(key[j] != best for j in live if j < slot), "step %d: %s %s" % (t, slot, key)
    assert seen_choice


def _trajs(rng, n, lo=3, hi=9):
    return [np.array([[rng.integers(1, 6), rng.integers(1, 6), rng.integers(1, 6)] for _ in range(rng.integers(lo, hi))], dtype=np.float64)
            for _ in range(n)]


def _streams_b1(trajs, episodes, n_envs):
    """the padding of _streams before buffered envs: one sentinel per trajectory"""
    traj_len = max(len(t) for t in trajs) + 1
    quota = [(episodes - e + n_envs - 1) // n_envs for e in range(n_envs)]
    s = np.full((n_envs, max(quota) + 1, traj_len, 4), 100.0)
    s[..., 3] = 1.0
    for e in range(n_envs):
        for j in range(quota[e]):
            t = trajs[e + j * n_envs + 1]
            s[e, j, :len(t), :t.shape[1]] = t
    return s.reshape(n_envs, -1, 4), traj_len, np.array(quota)


def test_streams_b1_unchanged():
    """_streams at B = 1 (and without pad) is byte for byte the one-sentinel padding"""
    pytest.importorskip("torch")
    from pct_b200.evaluation import _streams
    trajs = _trajs(np.random.default_rng(7), 12)
    want = _streams_b1(trajs, 9, 4)
    for got in (_streams(trajs, 9, 4), _streams(trajs, 9, 4, pad=1)):
        assert got[0].tobytes() == want[0].tobytes() and got[1] == want[1] and np.array_equal(got[2], want[2])


@pytest.mark.parametrize("name", ["LSAH", "OnlineBPH", "DBL"])
@pytest.mark.parametrize("B", [1, 3, 16])
def test_buffered_episodes_stay_in_their_trajectory(name, B):
    """Whole buffered episodes over B-sentinel padded dataset streams: every item a slot holds is the episode's own trajectory's or a
    sentinel, every episode ends, and at B = 1 the episodes are the plain oracle baseline's"""
    pytest.importorskip("torch")
    from pct_b200.evaluation import _streams
    trajs = _trajs(np.random.default_rng(11), 8, lo=20, hi=40)
    n_envs, episodes = 2, 6
    stream, traj_len, quota = _streams(trajs, episodes, n_envs, pad=B)
    assert traj_len == max(len(t) for t in trajs) + B
    c, _ = config("d1")
    for e in range(n_envs):
        m = RowBufferedOracle(c, stream[e], B, traj=traj_len)
        m.reset()
        ep, t = 0, 0
        while ep < quota[e]:
            traj = trajs[e + ep * n_envs + 1]
            own = {tuple(r) for r in traj[:, :3]} | {(100.0, 100.0, 100.0)}
            assert all(tuple(b[:3]) in own for b in m.buf), "env %d episode %d holds an item of another trajectory" % (e, ep)
            slot, row, _, _, _ = m.heuristic(name, ITEM_SET, SEED, e, t)
            _, _, d, rec = m.step_row(slot, row)
            t += 1
            assert t < 2000
            if d:
                assert rec["counter"] <= len(traj)
                if B == 1:  # the plain oracle baseline on the same trajectory
                    from pct_oracle import OracleDiscrete
                    s1 = np.full((traj_len, 4), 100.0)
                    s1[:, 3] = 1.0
                    s1[:len(traj), :3] = traj
                    ref = H.run_episodes(name, OracleDiscrete(1, container_size=(10, 10, 10), stream=s1), 1, ITEM_SET, SEED, e)
                    assert ref[0][1] == rec["counter"]
                ep += 1
