"""GPU: the continuous env on containers other than the unit cube (harness.CONT_BINS): a 1.2 x 0.8 x 1.0 pallet (non-dyadic sides,
W != L != H), the reference constructor's 10 x 10 x 10 default and a 2400 x 1700 x 2300 bin in millimetres (coordinates past 2200, where
the 6-decimal rounding divides exactly).  In the unit cube a swapped W / L / H, a hard-coded 1.0 or a bound from the wrong axis changes
nothing, and no trajectory reaches the exact-division branch; here each of them changes answers.

Per bin and setting: the step (records of the unmodified reference, tests/golden/cbin_*.npz, and a 64-env lock-step against one oracle
per env with the support graphs compared), device-drawn items, the LSAH / OnlineBPH / BR baselines, the placement queries, and the
item / reset / snapshot calls.  Everything is compared exactly; the only tolerance is the facade's ratio / reward (numpy sum vs reduce)."""
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
import pct_oracle_heuristics as OH  # noqa: E402
from harness import CONT_BINS, compare_graphs, cont_case_stream, cont_item_set, expected_flags, oracle_counts, policy_pick  # noqa: E402
from pct_oracle import OracleContinuous  # noqa: E402

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
NAMES = sorted(CONT_BINS)
BASELINES = ("LSAH", "OnlineBPH", "BR")
PSEED = 4321


def _pb():
    import pct_b200
    return pct_b200


def load(name):
    return CONT_BINS[name], np.load(os.path.join(G, "cbin_%s.npz" % name))


def trajectory(g, k):
    return {f: g["t%d_%s" % (k, f)] for f in ("stream", "rows", "obs", "reward", "done", "counter", "ratio")}


def episodes(g, name):
    off = np.concatenate([[0], np.cumsum(g["len_" + name])])
    return [g["flat_" + name][off[i]:off[i + 1]].tolist() for i in range(len(off) - 1)]


def oracle(c, stream):
    return OracleContinuous(c["setting"], container_size=c["container"], internal_node_holder=c["nb"], leaf_node_holder=c["nl"],
                            size_minimum=c["low"], stream=stream)


def batch(c, streams, **kw):
    """a float64-observation batch of the case's container on per-env item streams"""
    return _pb().PctBatch(len(streams), c["setting"], container_size=c["container"], continuous=True, internal_node_holder=c["nb"],
                          leaf_node_holder=c["nl"], obs_dtype=torch.float64, item_stream=np.stack(streams), size_minimum=c["low"], **kw)


def streams(c, n, seed, length=400):
    return [cont_case_stream(c, seed, e, length) for e in range(n)]


def _np(t):
    return t.cpu().numpy().copy()


# ---- step ----------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_facade_replays_the_records(name):
    c, g = load(name)
    for k in (0, 1):
        tr = trajectory(g, k)
        env = _pb().PackingContinuous(setting=c["setting"], container_size=list(c["container"]), item_set=None, sample_from_distribution=False,
                                      internal_node_holder=c["nb"], leaf_node_holder=c["nl"], item_stream=tr["stream"][None],
                                      size_minimum=c["low"])
        obs, j = tr["obs"], 0
        o = env.reset()
        assert o.dtype == np.float64 and np.array_equal(o, obs[j]), "t%d reset" % k
        j += 1
        for t in range(len(tr["rows"])):
            o, r, d, info = env.step(tr["rows"][t])
            assert np.array_equal(o, obs[j]), "t%d observation after step %d: %s" % (k, t, np.argwhere(o != obs[j])[:6].ravel())
            j += 1
            assert d == bool(tr["done"][t]) and info["counter"] == tr["counter"][t] and "flags" not in info, (k, t, info)
            assert abs(r - tr["reward"][t]) < 1e-12
            if d:
                assert abs(info["ratio"] - tr["ratio"][t]) < 1e-12
                o = env.reset()
                assert np.array_equal(o, obs[j]), "t%d observation after the reset following step %d" % (k, t)
                j += 1
        assert j == len(obs)
        env.close()


@pytest.mark.parametrize("mode", ["idx", "rows"])
@pytest.mark.parametrize("name", NAMES)
def test_lockstep_with_support_graphs(name, mode):
    """64 envs, 120 steps of the shared policy, leaf indices or float64 rows; after every step the flags are the ones the oracle's list
    lengths call for, and for every env not flagged so far the observations, rewards, dones and counters equal the oracles' and the
    support graph of every fourth env (a different quarter each step) is the oracle's"""
    c = CONT_BINS[name]
    n, seed = 64, 17
    s = streams(c, n, seed)
    orcs = [oracle(c, x) for x in s]
    gpu = batch(c, s)
    o_ref, o = np.stack([x.reset() for x in orcs]), _np(gpu.reset())
    assert np.array_equal(o, o_ref), "reset"
    live = np.ones(n, dtype=bool)  # envs not yet flagged
    dones = 0
    for t in range(120):
        picks = [policy_pick(o_ref[e], c["nb"], c["nl"], seed, e, t) for e in range(n)]
        res = [x.step(p[1]) for x, p in zip(orcs, picks)]
        # the capacity flags the oracle's list lengths call for (harness.CAPS): setting 2 on these bins can pass the 1228-candidate list
        want = np.array([expected_flags(dict(domain="continuous"), oracle_counts(x), r[3]) for x, r in zip(orcs, res)])
        if mode == "idx":
            ob, r, d, info = gpu.step(leaf_idx=torch.tensor([p[0] for p in picks], dtype=torch.int32, device="cuda"))
        else:
            ob, r, d, info = gpu.step(actions=torch.from_numpy(np.stack([p[1] for p in picks])).cuda())
        inf = gpu.decode_info(_np(info))
        assert np.array_equal(inf["flags"][live], want[live]), "step %d flags %s, oracle counts call for %s" % (t, inf["flags"], want)
        live &= want == 0  # a flagged env's results are not the reference's from here on
        d_ref = np.array([x[2] for x in res])
        assert np.array_equal(_np(d).astype(bool)[live], d_ref[live]), "step %d done" % t
        assert np.array_equal(_np(r)[live], np.array([x[1] for x in res]).astype(np.float32)[live]), "step %d reward" % t
        assert np.array_equal(inf["counter"][live], np.array([x[3]["counter"] for x in res])[live]), "step %d counter" % t
        o_ref = np.stack([orc.reset() if x[2] else x[0] for orc, x in zip(orcs, res)])
        bad = np.argwhere(_np(ob)[live] != o_ref[live])
        assert len(bad) == 0, "step %d: observation of env %d, entry %d" % (t, np.nonzero(live)[0][bad[0][0]], bad[0][1])
        for e in range(t % 4, n, 4):
            if live[e]:
                compare_graphs(gpu.support_graph(e), orcs[e].support_graph(), "step %d env %d:" % (t, e))
        dones += int(d_ref[live].sum())
    assert dones >= n // 2 and live.sum() >= n - 8, "finished episodes %d, envs never flagged %d" % (dones, live.sum())
    gpu.close()


# ---- device-drawn items ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_device_drawn_items(name):
    """sample_from_distribution with the default bounds (0.1 / 0.5 x min side, tools.py:178-181): x, y carry 3 decimals within the bounds;
    z likewise in setting 2, else one of the LITERAL levels 0.1 ... 0.5 whatever the container (C:bin3D.py:108-110); and the envs follow
    oracles drawing from the same counter-based generator"""
    c = CONT_BINS[name]
    n, seed = 32, 77
    lo, hi = 0.1 * min(c["container"]), 0.5 * min(c["container"])
    b = _pb().PctBatch(n, c["setting"], container_size=c["container"], continuous=True, obs_dtype=torch.float64, sample_from_distribution=True,
                       seed=seed)
    orcs = [oracle(c, None) for _ in range(n)]
    for e, x in enumerate(orcs):
        x.set_random_sample(seed, e, lo, hi)
    o_ref, o = np.stack([x.reset() for x in orcs]), _np(b.reset())
    drawn = []
    for t in range(30):
        assert np.array_equal(o, o_ref), "step %d" % t
        drawn.append(_np(b.preview_items(1))[:, 0])
        picks = [policy_pick(o_ref[e], c["nb"], c["nl"], seed, e, t) for e in range(n)]
        res = [x.step(p[1]) for x, p in zip(orcs, picks)]
        ob, _, _, info = b.step(leaf_idx=torch.tensor([p[0] for p in picks], dtype=torch.int32, device="cuda"))
        assert not b.decode_info(_np(info))["flags"].any()
        o, o_ref = _np(ob), np.stack([orc.reset() if x[2] else x[0] for orc, x in zip(orcs, res)])
    it = np.concatenate(drawn)
    xy = it[:, :3] if c["setting"] == 2 else it[:, :2]
    assert xy.min() >= round(lo, 3) and xy.max() <= round(hi, 3)
    assert np.array_equal(np.round(xy, 3), xy), "sizes with more than 3 decimals"
    if c["setting"] != 2:
        assert set(np.unique(it[:, 2]).tolist()) == {0.1, 0.2, 0.3, 0.4, 0.5}
    b.close()


# ---- baselines -------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_baselines_replay_the_records(name):
    from pct_b200.heuristics import run_heuristic
    c, g = load(name)
    for h in BASELINES:
        want = episodes(g, h)
        _, rec = run_heuristic(h, c["setting"], len(want), container_size=c["container"], item_set=cont_item_set(c), continuous=True,
                               item_stream=g["h_stream"][None], n_envs=1, return_episodes=True)
        assert rec["packed"] == want, h


@pytest.mark.parametrize("name", NAMES)
def test_baselines_equal_the_restatement(name):
    """24 envs on their own item streams, two episodes each, against pct_oracle_heuristics over one oracle per env"""
    from pct_b200.heuristics import run_heuristic
    c = CONT_BINS[name]
    n, items = 24, cont_item_set(c)
    s = streams(c, n, 311 + c["setting"])
    for h in BASELINES:
        _, rec = run_heuristic(h, c["setting"], 2 * n, container_size=c["container"], item_set=items, continuous=True, item_stream=np.stack(s),
                               n_envs=n, return_episodes=True)
        for e in range(n):
            ref = OH.run_episodes(h, oracle(c, s[e]), 2, item_set=items)
            for j in range(2):
                assert rec["packed"][e + j * n] == ref[j][2], (h, e, j)
                assert abs(rec["ratio"][e + j * n] - ref[j][0]) < 1e-12


@pytest.mark.parametrize("setting", [1, 2, 3])
def test_pallet_no_placement_row(setting):
    """when no placement is left the row is [W+1, 0, 0, W+1, 0, 0, 0, 0, 1] (out of the container along x), and the step it is given to
    ends the episode with the record's length"""
    c, g = load("pallet_s%d" % setting)
    W = c["container"][0]
    want = [len(e) for e in episodes(g, "LSAH")]
    b = _pb().PctBatch(1, c["setting"], container_size=c["container"], item_set=cont_item_set(c), continuous=True, obs_dtype=torch.float64,
                       item_stream=g["h_stream"][None])
    b.reset()
    ends = []
    while len(ends) < len(want):
        row = b.heuristic_actions("LSAH").clone()
        _, _, d, info = b.step(actions=row)
        if bool(_np(d)[0]):
            assert _np(row)[0].tolist() == [W + 1.0, 0, 0, W + 1.0, 0, 0, 0, 0, 1], _np(row)[0]
            ends.append(int(b.decode_info(_np(info))["counter"][0]))
        else:
            assert _np(row)[0, 3] < W + 1e-6
    assert ends == want
    b.close()


# ---- queries ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_queries_replay_the_records(name):
    """the reference's drop_box_virtual answers at W, L, H and 5e-7 / 2e-6 either side, below 0 and for zero sizes, at ten states of t0:
    the batched query and the single query, feasibility and rest height bit for bit"""
    c, g = load(name)
    tr = trajectory(g, 0)
    b = batch(c, [tr["stream"]])
    b.reset()
    n = 0
    for t in range(len(tr["rows"])):
        sel = np.nonzero(g["q_step"] == t)[0]
        if len(sel):
            q, den = g["q"][sel], g["q_den"][sel]
            f, h = b.query_placements(q[None], density=den[None])
            f, h = _np(f)[0], _np(h)[0]
            assert np.array_equal(f, g["q_feas"][sel]), "step %d: feasible %s" % (t, np.nonzero(f != g["q_feas"][sel])[0])
            assert np.array_equal(h.view(np.uint64), g["q_h"][sel].view(np.uint64)), "step %d: rest height" % t
            for i, x in enumerate(q):
                assert b.query_placement(0, x[:3], x[3], x[4], density=den[i]) == (bool(g["q_feas"][sel[i]]), g["q_h"][sel[i]]), (t, x)
            n += len(sel)
        b.step(actions=torch.from_numpy(tr["rows"][t][None]).cuda())
    assert n == len(g["q"])
    b.close()


def _orient(nb, row):
    """LeafNode2Action: the oriented sizes of a leaf row (the item entries matching its x and y extents, z the remaining one)"""
    rest, out = list(nb), []
    for ext in (row[3] - row[0], row[4] - row[1]):
        out.append(rest.pop(int(np.argmin([abs(v - ext) for v in rest]))))
    return out + rest


def _queries(c, orc, leaves, rng, k=96):
    """test_gpu_queries' recipe scaled to the bin: leaf rows, the 1e-6 tolerances at 0, W and L, zero sizes, over-tall items, random
    positions over [-0.1 m, W + 0.05 m] x [-0.1 m, L + 0.05 m] with random sizes in [0.05 m, 0.6 m] (m = min side)"""
    W, L, H = c["container"]
    m = min(c["container"])
    nb, q = orc.next_box, []
    for row in leaves[:40]:
        q.append(_orient(nb, row) + [row[0], row[1]])
    for row in leaves[:6]:
        d = _orient(nb, row)
        q += [d + [row[0] - 5e-7, row[1]], d + [W - d[0] + 5e-7, row[1]], d + [row[0], L - d[1] + 2e-6]]
    size = lambda: [round(v, 3) for v in rng.uniform(0.05 * m, 0.6 * m, 3)]
    pos = lambda: [round(rng.uniform(-0.1 * m, W + 0.05 * m), 3), round(rng.uniform(-0.1 * m, L + 0.05 * m), 3)]
    for _ in range(3):
        s = size()
        q += [[0, s[1], s[2]] + pos(), [s[0], 0, s[2]] + pos()]
    for _ in range(4):
        s = size()
        q.append([s[0], s[1], H + 0.25 * m] + pos())
    while len(q) < k:
        q.append(size() + pos())
    return q[:k]


@pytest.mark.parametrize("name", NAMES)
def test_queries_equal_the_oracle(name):
    """96 placements per env at states every 6 steps of a 64-env lock-step: the batched answers equal the oracle's drop_box_virtual, and a
    sample of them the single query"""
    c = CONT_BINS[name]
    n, seed = 64, 23
    s = streams(c, n, seed)
    orcs = [oracle(c, x) for x in s]
    b = batch(c, s)
    obs = _np(b.reset())
    assert np.array_equal(obs, np.stack([x.reset() for x in orcs])), "reset"
    rng = np.random.default_rng(c["setting"])
    feasible, live = 0, np.ones(n, dtype=bool)  # a flagged env is not the reference's from then on (test_lockstep_with_support_graphs)
    for t in range(48):
        if t % 6 == 3:
            leaves = [obs[e].reshape(-1, 9)[c["nb"]:c["nb"] + c["nl"]] for e in range(n)]
            q = np.asarray([_queries(c, orcs[e], lv[lv[:, 8] == 1], rng) for e, lv in enumerate(leaves)])
            f, h = b.query_placements(q)
            f, h = _np(f), _np(h)
            for e in np.nonzero(live)[0]:
                for j, x in enumerate(q[e]):
                    assert (bool(f[e, j]), h[e, j]) == orcs[e].drop_box_virtual(x[:3], x[3], x[4]), (t, e, j, x)
            for e in range(0, n, 7):
                for j in range(0, q.shape[1], 9):
                    x = q[e, j]
                    assert b.query_placement(e, x[:3], x[3], x[4], density=orcs[e].next_den) == (bool(f[e, j]), h[e, j]), (t, e, j)
            feasible += int(f.sum())
            assert not f.all()
        o_ref = []
        for e in range(n):
            _, row = policy_pick(obs[e], c["nb"], c["nl"], PSEED, e, t)
            o, _, d, _ = orcs[e].step(row)
            o_ref.append(orcs[e].reset() if d else o)
        ob, _, _, info = b.step(leaf_idx=b.random_policy(PSEED, t))
        obs = _np(ob)
        live &= b.decode_info(_np(info))["flags"] == 0
        assert np.array_equal(obs[live], np.stack(o_ref)[live]), "step %d" % t
    assert feasible > 0 and live.sum() >= n - 8
    b.close()


# ---- items, reset, snapshot --------------------------------------------------------------------------------------------------------------
ITEM_CASES = ["pallet_s1", "pallet_s2", "mm_s1", "mm_s2"]


@pytest.mark.parametrize("name", ITEM_CASES)
def test_preview_and_set_items(name):
    """preview_items(8) lists the current item and the next 7 stream draws; a batch on a perturbed stream, corrected by set_items to the
    plain batch's current items before every step, follows the plain batch for two episodes of every env"""
    c = CONT_BINS[name]
    n, L = 32, 300
    s = streams(c, n, 41, L)
    A = batch(c, s)
    A.reset()
    for t in range(5):
        A.step(leaf_idx=A.random_policy(PSEED, t))
    pv = _np(A.preview_items(8))
    for e in range(n):
        st = A.state(e)
        assert list(pv[e, 0, :3]) == list(st["next_box"]) and pv[e, 0, 3] == st["next_den"], e
        for j in range(1, 8):
            it = s[e][(st["draw_pos"] + j - 1) % L]
            assert list(pv[e, j, :3]) == list(it[:3]) and pv[e, j, 3] == (it[3] if c["setting"] == 3 else 1.0), (e, j)
    A.close()
    other = streams(c, n, 99, L)
    rs = np.random.RandomState(5)
    s2 = [np.where((rs.rand(L) < 0.3)[:, None], o, x) for x, o in zip(s, other)]
    A, B = batch(c, s), batch(c, s2)
    A.reset()
    B.reset()
    eps, changed = np.zeros(n, dtype=int), 0
    for t in range(400):
        pa, pb = A.preview_items(1)[:, 0], B.preview_items(1)[:, 0]
        diff = torch.nonzero((pa != pb).any(1)).flatten().to(torch.int32)
        obs_b = B.set_items(pa[diff.long(), :3], env_idx=diff, density=pa[diff.long(), 3])
        changed += int(diff.numel())
        assert torch.equal(obs_b, A._obs), "observation after set_items differs at step %d" % t
        idx = A.random_policy(PSEED, t)
        oa = [_np(x) for x in A.step(leaf_idx=idx)]
        ob = [_np(x) for x in B.step(leaf_idx=idx)]
        for k, nm in ((1, "reward"), (2, "done")):
            assert np.array_equal(oa[k], ob[k]), "%s differs at step %d" % (nm, t)
        # counter, ratio, episode reward and length; not the flags: B's expansion of its own (perturbed) item before set_items can pass the
        # candidate capacity where A's item does not
        assert np.array_equal(oa[3][:, [0, 2, 3, 4]], ob[3][:, [0, 2, 3, 4]]), "info at step %d" % t
        eps += oa[2].astype(int)
        if eps.min() >= 2:
            break
    assert eps.min() >= 2 and changed > 0
    A.close()
    B.close()


@pytest.mark.parametrize("name", ITEM_CASES)
def test_reset_mask_and_snapshot(name):
    """a batch without auto-reset that calls reset(mask=done) after every step equals its auto-resetting twin for two episodes of every env;
    a snapshot taken mid-episode, restored into a fresh handle, continues like the original"""
    c = CONT_BINS[name]
    n = 32
    s = streams(c, n, 53)
    A, B = batch(c, s), batch(c, s, auto_reset=False)
    assert torch.equal(A.reset(), B.reset())
    eps, snap, t = np.zeros(n, dtype=int), None, 0
    while eps.min() < 2:
        idx = A.random_policy(PSEED, t)
        ra = [_np(x) for x in A.step(leaf_idx=idx)]
        rb = [_np(x) for x in B.step(leaf_idx=idx)]
        done = ra[2] != 0
        for k, nm in ((1, "reward"), (2, "done")):
            assert np.array_equal(ra[k], rb[k]), "%s differs at step %d" % (nm, t)
        assert np.array_equal(ra[3][:, :5], rb[3][:, :5]) and np.array_equal(ra[3][~done], rb[3][~done]), "info differs at step %d" % t
        ob = _np(B.reset(mask=torch.from_numpy(done).cuda()))
        assert np.array_equal(ra[0], ob), "observation after reset(mask) at step %d" % t
        eps += done.astype(int)
        t += 1
        assert t < 500
        if t == 12:
            snap = A.snapshot().clone()
            obs_snap = A._obs.clone()
    B.close()
    C = batch(c, s)
    C.reset()
    C.restore(snap)
    assert torch.equal(C._obs, obs_snap)
    A.restore(snap)
    for t in range(12, 60):
        idx = A.random_policy(PSEED, t)
        ra = [_np(x) for x in A.step(leaf_idx=idx)]
        rc = [_np(x) for x in C.step(leaf_idx=idx)]
        for u, v, nm in zip(ra, rc, ("obs", "reward", "done", "info")):
            assert np.array_equal(u, v), "restored handle: %s differs at step %d" % (nm, t)
    A.close()
    C.close()
