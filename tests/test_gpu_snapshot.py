"""GPU: snapshot / restore of env states (pct_snapshot / pct_restore, PctBatch.snapshot / restore, copy.deepcopy of the facades).

Branches are checked against the reference's own records (tests/golden/) and against the library itself, bit for bit: a restored env
must continue exactly as the env it was taken from.  Every step must carry zero flags unless a test expects one.
"""
import copy
import glob
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
from harness import CASES, CONT_CASES, ITEM_SET  # noqa: E402

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
DISCRETE = sorted(glob.glob(os.path.join(G, "discrete_*.npz"))) + sorted(glob.glob(os.path.join(G, "case_*.npz")))
CONTINUOUS = sorted(glob.glob(os.path.join(G, "continuous_s*.npz"))) + sorted(glob.glob(os.path.join(G, "ccase_*.npz")))
PARTING = {"alias_d1_e126": 39, "alias_d1_e835": 167, "alias_d3_e92": 103}  # step of the first alias / snapshot difference (tests/test_zzz_gpu_alias.py)
BAD_SNAPSHOT = 128


def _pb():
    import pct_b200
    return pct_b200


def _outputs(b, out):
    """host copies of what one step returned"""
    obs, rew, done, info = out
    return obs.cpu().numpy().copy(), rew.cpu().numpy().copy(), done.cpu().numpy().copy(), info.cpu().numpy().copy()


def _same(a, b, what):
    for x, y, nm in zip(a, b, ("obs", "reward", "done", "info")):
        assert np.array_equal(x, y), "%s: %s differ" % (what, nm)


def _no_flags(info):
    assert not (np.asarray(info)[:, 1]).any(), "flags %s" % np.unique(np.asarray(info)[:, 1])


def _random_batch(n, setting, continuous, **kw):
    pct_b200 = _pb()
    if continuous:
        return pct_b200.PctBatch(n, setting, container_size=(1.0, 1.0, 1.0), continuous=True, sample_from_distribution=True, seed=1234, **kw)
    return pct_b200.PctBatch(n, setting, item_set=ITEM_SET, seed=1234, **kw)


def _run(b, steps, t0=0, pseed=4321):
    for t in range(t0, t0 + steps):
        _, _, _, info = b.step(leaf_idx=b.random_policy(pseed, t))
        _no_flags(info.cpu().numpy())


# ---- 1. branching against the reference's records --------------------------------------------------------------------------------
def _expected(g):
    """per step t: observation before / after the step in auto-reset (ShmemVecEnv) semantics"""
    obs, before, after, k = g["obs"], [], [], 1
    cur = obs[0]
    for t in range(len(g["rows"])):
        before.append(cur)
        cur = obs[k + 1] if g["done"][t] else obs[k]
        k += 2 if g["done"][t] else 1
        after.append(cur)
    assert k == len(obs)
    return before, after


def _cuts(g, name):
    n = len(g["rows"])
    d = [int(t) for t in np.nonzero(g["done"])[0]]
    cuts = {1, n // 3, (2 * n) // 3, n - 1}
    if d:
        cuts.add(d[0])           # the snapshot is taken just before the step that ends the episode
        cuts.add(d[-1])
    if name in PARTING:
        p = PARTING[name]
        cuts.update({p - 1, p})  # just before the step where the two load semantics part
    return sorted(c for c in cuts if 0 < c < n)


def _branch_record(g, c, continuous, name):
    pct_b200 = _pb()
    cuts = _cuts(g, name)
    K = 1 + len(cuts)
    stream = np.repeat(np.asarray(g["stream"])[None], K, axis=0)
    if continuous:
        b = pct_b200.PctBatch(K, c["setting"], container_size=tuple(c["container"]), continuous=True, internal_node_holder=c["nb"],
                              leaf_node_holder=c["nl"], obs_dtype=torch.float64, item_stream=stream, size_minimum=c["low"])
    else:
        b = pct_b200.PctBatch(K, c["setting"], container_size=tuple(c["container"]), item_set=c["items"], internal_node_holder=c["nb"],
                              leaf_node_holder=c["nl"], obs_dtype=torch.float64, item_stream=stream, LNES=c["lnes"])
    before, after = _expected(g)
    nb, nl = c["nb"], c["nl"]
    cut_of = [0] + cuts
    o = b.reset().cpu().numpy()
    assert np.array_equal(o[0], before[0])
    for t in range(len(g["rows"])):
        for i in range(1, K):
            if cut_of[i] == t:
                fresh = torch.zeros_like(b._obs)
                b.restore(b.snapshot(env_idx=[0]), env_idx=[i], out=fresh)
                f = fresh.cpu().numpy()
                assert np.array_equal(f[i], before[t]), "restore rows of env %d at step %d" % (i, t)
                assert not np.delete(f, i, axis=0).any(), "rows of other envs written"
        rows = np.zeros((K, 9))
        for i in range(K):
            if cut_of[i] <= t:
                rows[i] = g["rows"][t]
            else:  # not branched yet: its own, different trajectory (first valid leaf of its own observation)
                leaves = o[i].reshape(-1, 9)[nb:nb + nl]
                valid = np.nonzero(leaves[:, 8])[0]
                if len(valid):
                    rows[i] = leaves[valid[(t * 7 + i) % len(valid)]]
        ob, rew, done, info = _outputs(b, b.step(actions=torch.from_numpy(rows).to(b.device)))
        _no_flags(info)
        for i in range(K):
            if cut_of[i] > t:
                continue
            assert np.array_equal(ob[i], after[t]), "env %d (cut %d): observation after step %d" % (i, cut_of[i], t)
            assert bool(done[i]) == bool(g["done"][t]) and info[i, 0] == g["counter"][t], (i, t)
            if continuous:
                assert abs(float(rew[i]) - float(np.float32(g["reward"][t]))) <= 1e-6 * max(1.0, abs(g["reward"][t])), (i, t)
            else:
                assert rew[i] == np.float32(g["reward"][t]), (i, t)
            if done[i]:
                ratio = info[i:i + 1].view(np.float32)[0, 2]
                assert abs(float(ratio) - float(g["ratio"][t])) <= 1e-6, (i, t)
        o = ob
    b.close()


@pytest.mark.parametrize("path", DISCRETE, ids=[os.path.basename(p) for p in DISCRETE])
def test_branches_follow_reference_record_discrete(path):
    g = np.load(path)
    name = str(g["name"]) if "name" in g.files else ""
    if name:
        c = CASES[name]
    else:
        c = dict(setting=int(g["setting"]), container=(10, 10, 10), items=ITEM_SET, nb=80, nl=50, lnes=str(g["lnes"]) if "lnes" in g.files else "EMS")
    _branch_record(g, c, False, name)


@pytest.mark.parametrize("path", CONTINUOUS, ids=[os.path.basename(p) for p in CONTINUOUS])
def test_branches_follow_reference_record_continuous(path):
    g = np.load(path)
    name = str(g["name"]) if "name" in g.files else ""
    c = CONT_CASES[name] if name else dict(setting=int(g["setting"]), container=(1.0, 1.0, 1.0), nb=80, nl=50, low=0.1)
    _branch_record(g, c, True, name)


# ---- 2. round trip at scale, PCT_ITEMS_RANDOM --------------------------------------------------------------------------------------
DOMAINS = [(s, False) for s in (1, 2, 3)] + [(s, True) for s in (1, 2, 3)]
DOM_IDS = ["d%d" % s if not c else "c%d" % s for s, c in DOMAINS]


@pytest.mark.parametrize("setting,continuous", DOMAINS, ids=DOM_IDS)
def test_round_trip_replays_the_same_future(setting, continuous):
    n = 1024
    b = _random_batch(n, setting, continuous)
    b.reset()
    _run(b, 40)
    snap = b.snapshot()
    obs_at = b._obs.cpu().numpy().copy()
    probe = list(range(0, n, 61))
    st0 = [b.state(e) for e in probe]
    rec, idx = [], []
    for t in range(40, 70):
        i = b.random_policy(4321, t).clone()
        idx.append(i)
        rec.append(_outputs(b, b.step(leaf_idx=i)))
        _no_flags(rec[-1][3])
    assert any(r[2].any() for r in rec), "the window should contain auto-resets"
    fresh = torch.full_like(b._obs, float("nan"))
    b.restore(snap, out=fresh)
    assert np.array_equal(fresh.cpu().numpy(), obs_at)
    for e, s0 in zip(probe, st0):
        s = b.state(e)
        for k in s0:
            assert np.array_equal(np.asarray(s[k]), np.asarray(s0[k])), "state %s of env %d" % (k, e)
    for t in range(30):
        _same(rec[t], _outputs(b, b.step(leaf_idx=idx[t])), "step %d after the restore" % t)
    b.close()


# ---- 3. stale destinations ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", DOMAINS, ids=DOM_IDS)
def test_restore_over_stale_state_equals_restore_into_fresh_handle(setting, continuous):
    n = 256
    a = _random_batch(n, setting, continuous)
    a.reset()
    _run(a, 6, pseed=11)
    snap = a.snapshot()
    rich = _random_batch(n, setting, continuous)
    rich.reset()
    _run(rich, 150, pseed=12)
    fresh = _random_batch(n, setting, continuous)
    fresh.reset()
    o1, o2 = torch.zeros_like(rich._obs), torch.zeros_like(fresh._obs)
    rich.restore(snap, out=o1)
    fresh.restore(snap, out=o2)
    assert torch.equal(o1, o2)
    for t in range(30):
        i = rich.random_policy(13, t).clone()
        r1, r2 = _outputs(rich, rich.step(leaf_idx=i)), _outputs(fresh, fresh.step(leaf_idx=i))
        _no_flags(r1[3])
        _same(r1, r2, "step %d" % t)
    for x in (a, rich, fresh):
        x.close()


# ---- 4. across handles ---------------------------------------------------------------------------------------------------------------
def _streams(n, length, seed, continuous):
    rng = np.random.default_rng(seed)
    if continuous:
        s = np.round(rng.uniform(0.1, 0.5, size=(n, length, 3)), 3)
    else:
        s = np.asarray(ITEM_SET, dtype=np.float64)[rng.integers(0, len(ITEM_SET), size=(n, length))]
    return np.concatenate([s, rng.uniform(0.5, 1.5, size=(n, length, 1))], axis=2)


def _stream_batch(n, setting, continuous, stream, **kw):
    pct_b200 = _pb()
    if continuous:
        return pct_b200.PctBatch(n, setting, container_size=kw.pop("container_size", (1.0, 1.0, 1.0)), continuous=True, item_stream=stream,
                                 size_minimum=0.1, **kw)
    return pct_b200.PctBatch(n, setting, container_size=kw.pop("container_size", (10, 10, 10)), item_set=ITEM_SET, item_stream=stream, **kw)


@pytest.mark.parametrize("continuous", [False, True], ids=["discrete", "continuous"])
def test_restore_into_another_handle(continuous):
    pct_b200 = _pb()
    n, setting = 64, 1
    stream = _streams(n, 300, 5, continuous)
    a = _stream_batch(n, setting, continuous, stream, env_id_base=0)
    b = _stream_batch(n, setting, continuous, stream, env_id_base=1000)
    a.reset()
    b.reset()
    for t in range(20):
        _no_flags(a.step(leaf_idx=a.random_policy(3, t))[3].cpu().numpy())
    snap = a.snapshot()
    ob_a, ob_b = torch.zeros_like(a._obs), torch.zeros_like(b._obs)
    a.restore(snap, out=ob_a)
    b.restore(snap, out=ob_b)
    assert torch.equal(ob_a, ob_b)
    for t in range(20, 60):
        i = a.random_policy(3, t).clone()
        ra, rb = _outputs(a, a.step(leaf_idx=i)), _outputs(b, b.step(leaf_idx=i))
        _no_flags(ra[3])
        _same(ra, rb, "step %d" % t)
    # another configuration: the record is refused, the env keeps its state and the next step reports the flag
    for kw in (dict(container_size=(1.0, 1.0, 1.25) if continuous else (10, 10, 11)), dict(leaf_node_holder=40), dict(internal_node_holder=60)):
        c = _stream_batch(n, setting, continuous, stream, **kw)
        c.reset()
        for t in range(5):
            c.step(leaf_idx=c.random_policy(3, t))
        before = [c.state(e) for e in (0, 7)]
        rows = torch.zeros_like(c._obs)
        c.restore(snap, out=rows)
        assert not rows.any(), "rows written for a refused record"
        for e, s0 in zip((0, 7), before):
            s = c.state(e)
            assert s["n_boxes"] == s0["n_boxes"] and np.array_equal(s["boxes"], s0["boxes"]) and s["draw_pos"] == s0["draw_pos"]
            assert s["flags"] == BAD_SNAPSHOT
        _, _, _, info = c.step(leaf_idx=c.random_policy(3, 5))
        flags = info.cpu().numpy()[:, 1]
        assert (flags & BAD_SNAPSHOT).all()
        with pytest.raises(pct_b200.PctError, match="bad_snapshot"):
            pct_b200.PctBatch.check_flags(flags)
        c.close()
    a.close()
    b.close()


def test_argument_errors():
    pct_b200 = _pb()
    b = _random_batch(4, 1, False)
    with pytest.raises(pct_b200.PctError, match="before pct_reset"):
        b.snapshot()
    L = b.L
    assert L.pct_snapshot(b.h, None, -1, None, None) == -1
    b.reset()
    assert L.pct_snapshot(b.h, None, 4, None, None) == -1
    assert L.pct_restore(b.h, None, None, -1, None, None, None) == -1
    s = b.snapshot()
    assert s.shape == (4, b.snapshot_bytes) and b.snapshot_bytes % 16 == 0
    # out-of-range indices are skipped: nothing is written out of bounds
    obs0 = b._obs.clone()
    b.restore(s, env_idx=[-1, 4, 1000], rec_idx=[0, 1, 2], out=torch.zeros_like(b._obs))
    b.restore(s, env_idx=[0, 1], rec_idx=[7, -3])
    assert torch.equal(b._obs, obs0)
    torch.cuda.synchronize()
    b.close()


# ---- 5. fan-out with leaf indices ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("continuous", [False, True], ids=["discrete", "continuous"])
def test_fan_out_leaf_indices_equal_leaf_rows(continuous):
    n = 16
    b = _random_batch(n, 1, continuous, obs_dtype=torch.float64)
    b.reset()
    _run(b, 25)
    rec = b.snapshot(env_idx=[3])
    _run(b, 7, t0=25, pseed=99)  # the children's own states differ from the record's
    src = torch.zeros(n, dtype=torch.int32)
    rows_obs = b.restore(rec, rec_idx=src, out=torch.zeros_like(b._obs)).clone()
    r_idx = _outputs(b, b.step(leaf_idx=torch.arange(n, dtype=torch.int32, device=b.device)))
    b.restore(rec, rec_idx=src, out=torch.zeros_like(b._obs))
    leaf_rows = rows_obs.view(n, -1, 9)[:, b.nb:b.nb + b.nl]
    act = leaf_rows[torch.arange(n), torch.arange(n).clamp(max=b.nl - 1)].contiguous()
    r_act = _outputs(b, b.step(actions=act))
    assert (rows_obs.view(n, -1, 9)[:, b.nb:b.nb + b.nl, 8].sum(1) > 1).all()
    _same(r_idx, r_act, "leaf index vs leaf row")
    b.close()


# ---- 6. delta rows ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("continuous", [False, True], ids=["discrete", "continuous"])
@pytest.mark.parametrize("rows", ["none", "tracked"])
def test_restore_keeps_the_observation_buffer_contract(continuous, rows):
    n = 128
    b = _random_batch(n, 1, continuous)
    b.reset()
    _run(b, 5)
    early = b.snapshot()
    _run(b, 40, t0=5)  # the tracked buffer now holds many more rows than the early states have
    late = b.snapshot()
    if rows == "none":
        assert b.restore(early, write_obs=False) is None
    else:
        b.restore(early)
    i = b.random_policy(7, 0).clone()
    tracked = _outputs(b, b.step(leaf_idx=i))
    b.restore(late, write_obs=False)
    b.restore(early, write_obs=False)
    out = torch.full_like(b._obs, 7.0)
    fresh = _outputs(b, b.step(leaf_idx=i, out=out))
    _no_flags(fresh[3])
    _same(tracked, fresh, "tracked vs fresh buffer")
    b.close()


# ---- 7. LSAH continuation ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("continuous", [False, True], ids=["discrete", "continuous"])
def test_lsah_continues_after_restore(continuous):
    b = _random_batch(64, 1, continuous)
    b.reset()

    def lsah(steps):
        out = []
        for _ in range(steps):
            rows = b.heuristic_actions("LSAH").clone()
            out.append((rows.cpu().numpy(),) + _outputs(b, b.step(actions=rows)))
        return out

    lsah(12)
    snap = b.snapshot()
    first = lsah(20)
    b.restore(snap)
    again = lsah(20)
    for t, (x, y) in enumerate(zip(first, again)):
        for u, v in zip(x, y):
            assert np.array_equal(u, v), "LSAH step %d" % t
    b.close()


# ---- 8. graph capture ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("continuous", [False, True], ids=["discrete", "continuous"])
def test_restore_and_step_in_a_cuda_graph(continuous):
    n = 256
    b = _random_batch(n, 1, continuous)
    b.reset()
    _run(b, 10)
    snap = b.snapshot()
    _run(b, 10, t0=10)
    idx = b.random_policy(5, 3).clone()
    buf = torch.zeros_like(b._obs)
    b.restore(snap, out=buf)
    eager = _outputs(b, b.step(leaf_idx=idx, out=buf))
    _run(b, 5, t0=30)
    gbuf = torch.zeros_like(b._obs)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        b.restore(snap, out=gbuf)
        res = b.step(leaf_idx=idx, out=gbuf)
    for rep in range(2):
        graph.replay()
        torch.cuda.synchronize()
        _same(eager, _outputs(b, res), "graph replay %d" % rep)
    b.close()


# ---- 9. facades ---------------------------------------------------------------------------------------------------------------------------
def _first_leaf(env, o):
    leaves = o.reshape(-1, 9)[env.internal_node_holder:env.internal_node_holder + env.leaf_node_holder]
    v = np.nonzero(leaves[:, 8])[0]
    return leaves[v[len(v) // 2]] if len(v) else np.zeros(9)


def _facades(tmp_path):
    pct_b200 = _pb()
    rng = np.random.default_rng(3)
    ds = os.path.join(str(tmp_path), "set.pt")
    torch.save([np.asarray(ITEM_SET)[rng.integers(0, len(ITEM_SET), 60)].tolist() for _ in range(8)], ds)
    return {
        "stream": lambda: pct_b200.PackingDiscrete(setting=1, container_size=[10, 10, 10], item_set=ITEM_SET, data_name=ds, load_test_data=True),
        "random": lambda: pct_b200.PackingDiscrete(setting=3, container_size=[10, 10, 10], item_set=ITEM_SET, seed=9),
        "continuous": lambda: pct_b200.PackingContinuous(setting=1, container_size=[1, 1, 1], item_set=None, seed=9),
    }


@pytest.mark.parametrize("kind", ["stream", "random", "continuous"])
def test_deepcopy_of_the_facade(kind, tmp_path):
    make = _facades(tmp_path)[kind]
    env = make()
    o = env.reset()
    for _ in range(15):
        o, _, d, _ = env.step(_first_leaf(env, o))
        if d:
            o = env.reset()
    env.next_box = list(env.next_box)  # a Python attribute travels with the copy
    cp = copy.deepcopy(env)
    assert cp._next_box_override == env._next_box_override and cp._batch is not env._batch
    env._next_box_override = cp._next_box_override = None
    # independent: stepping the copy leaves the original unchanged
    st = env._state()
    oc = o
    for _ in range(5):
        oc, _, d, _ = cp.step(_first_leaf(cp, oc))
        if d:
            oc = cp.reset()
    st2 = env._state()
    assert st2["n_boxes"] == st["n_boxes"] and np.array_equal(st2["boxes"], st["boxes"]) and st2["draw_pos"] == st["draw_pos"]
    # same state, same future items: identical outputs under the same rows
    cp = copy.deepcopy(env)
    oc = o
    for t in range(60):
        row = _first_leaf(env, o)
        o, r, d, info = env.step(row)
        oc, rc, dc, infoc = cp.step(row)
        assert np.array_equal(o, oc) and r == rc and d == dc and info == infoc, "step %d" % t
        assert "flags" not in info
        if d:
            o, oc = env.reset(), cp.reset()
            assert np.array_equal(o, oc)
    env.close()
    cp.close()


@pytest.mark.parametrize("kind", ["stream", "random", "continuous"])
def test_deepcopy_before_the_first_reset(kind, tmp_path):
    make = _facades(tmp_path)[kind]
    env = make()
    cp = copy.deepcopy(env)
    o, oc = env.reset(), cp.reset()
    assert np.array_equal(o, oc)
    for t in range(30):
        row = _first_leaf(env, o)
        o, _, d, _ = env.step(row)
        oc, _, dc, _ = cp.step(row)
        assert np.array_equal(o, oc) and d == dc, t
        if d:
            o, oc = env.reset(), cp.reset()
    env.close()
    cp.close()
