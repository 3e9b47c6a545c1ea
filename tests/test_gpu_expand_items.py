"""GPU: read-only leaf expansion of caller-given items (pct_expand_items, PctBatch.expand_items).

The expansion is pinned to the reference's own leaves (the item override records of tests/golden/make_item_golden.py) and to the library's
item override, bit for bit: for every row and item, the leaf rows and the info record equal what set_items writes for that item on a twin
restored from a snapshot.  The call must leave every env exactly as it was (snapshots, observation buffer, the following steps), and a
buffer-packing loop built on it must replay as a plain stream on the library and on the oracle.
"""
import ctypes as C
import glob
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
from buffer_compose import BufferDriver  # noqa: E402
from harness import CASES, ITEM_SET, NEEDS_ALIAS_D, OracleDiscrete, case_stream, load_capacity_cases, make_stream  # noqa: E402
import many_supports as M  # noqa: E402
from pct_oracle import OracleContinuous, make_continuous_stream  # noqa: E402

pytestmark = pytest.mark.gpu
PSEED = 4321
DOMAINS = [(s, False) for s in (1, 2, 3)] + [(s, True) for s in (1, 2, 3)]
DOM_IDS = ["d%d" % s if not c else "c%d" % s for s, c in DOMAINS]
FLAG_CAND = 8


def _pb():
    import pct_b200
    return pct_b200


def _np(t):
    return t.cpu().numpy().copy()


def _streams(n, setting, continuous, length, seed=11):
    if continuous:
        return np.stack([make_continuous_stream(seed, e, length, setting) for e in range(n)])
    return np.stack([make_stream(seed, e, length, setting) for e in range(n)])


def _batch(n, setting, continuous, stream=None, **kw):
    pct_b200 = _pb()
    if continuous:
        if stream is not None:
            return pct_b200.PctBatch(n, setting, container_size=(1.0, 1.0, 1.0), continuous=True, obs_dtype=torch.float64, item_stream=stream,
                                     size_minimum=0.1, **kw)
        return pct_b200.PctBatch(n, setting, container_size=(1.0, 1.0, 1.0), continuous=True, obs_dtype=torch.float64,
                                 sample_from_distribution=True, seed=1234, **kw)
    if stream is not None:
        return pct_b200.PctBatch(n, setting, item_set=ITEM_SET, obs_dtype=torch.float64, item_stream=stream, **kw)
    return pct_b200.PctBatch(n, setting, item_set=ITEM_SET, obs_dtype=torch.float64, seed=1234, **kw)


def _snap(b):
    return _np(b.snapshot(out=torch.zeros((b.n_envs, b.snapshot_bytes), dtype=torch.uint8, device=b.device)))


def _leaf_rows(b, obs):
    return obs[:, b.nb * 9:(b.nb + b.nl) * 9].reshape(obs.shape[0], b.nl, 9)


def _items(n, k, continuous, rng, degenerate=True):
    """(n, k, 3) random items; with `degenerate`, column 1.. of a few rows hold the sentinel, an item larger than the bin, an item as tall
    as the bin and (discrete) sizes outside [0, 255].  (No zero side: the reference's drop_box_virtual raises on it, an empty height-map slice.)"""
    if continuous:
        it = rng.uniform(0.1, 0.5, size=(n, k, 3))
        odd = [(100.0, 100.0, 100.0), (1.5, 0.2, 0.2), (0.5, 0.5, 1.0)]
    else:
        it = np.array(ITEM_SET, dtype=np.int64)[rng.randint(0, len(ITEM_SET), size=(n, k))].astype(np.float64)
        odd = [(100, 100, 100), (11, 2, 2), (2, 3, 10), (300, -5, 2)]
    if degenerate and k > 1:
        for i, o in enumerate(odd):
            it[i::len(odd) * 3, 1 + i % (k - 1)] = o
    return torch.as_tensor(it)


def _compare(b, twin, items, den=None, env_idx=None):
    """expand_items on b against set_items(items[:, j]) on `twin` restored from b's snapshot, column by column: identical leaf-row bytes and
    identical records (counter, flags, n_leaf, n_cand, n_ems); -> (leaves, info) of the expansion"""
    n, k = int(items.shape[0]), int(items.shape[1])
    snap = b.snapshot()
    leaves, info = b.expand_items(items, env_idx=env_idx, density=den)
    leaves, info = _np(leaves), _np(info)
    rows = np.arange(n) if env_idx is None else np.asarray(env_idx)
    for j in range(k):
        twin.restore(snap, write_obs=False)
        ti = torch.zeros((twin.n_envs, 8), dtype=torch.int32, device=twin.device)
        out = torch.zeros((twin.n_envs, twin.obs_len), dtype=twin.obs_dtype, device=twin.device)
        obs = _np(twin.set_items(items[:, j], env_idx=env_idx, density=None if den is None else den[:, j], out=out, info=ti))
        want = _leaf_rows(twin, obs)[rows]
        assert np.array_equal(want.view(np.uint8), leaves[:, j].view(np.uint8)), "leaf rows of item column %d differ" % j
        ti = _np(ti)[rows]
        assert np.array_equal(info[:, j][:, [0, 1, 5, 6, 7]], ti[:, [0, 1, 5, 6, 7]]), "records of item column %d differ" % j
        assert not info[:, j, 2:5].any()
    return leaves, info


def _walk_and_compare(b, twin, continuous, rng, checkpoints=(0, 5, 20, 60), density=False):
    b.reset()
    twin.reset()
    n, t, seen = b.n_envs, 0, 0
    for cp in checkpoints:
        while t < cp:
            b.step(leaf_idx=b.random_policy(PSEED, t))
            t += 1
        items = _items(n, 8, continuous, rng)
        den = torch.as_tensor(rng.uniform(0.5, 2.0, size=(n, 8))) if density else None
        leaves, info = _compare(b, twin, items, den)
        seen += int(info[:, :, 5].sum())
        for k in (1, 3):  # fewer items per row: the same entries
            l2, i2 = b.expand_items(items[:, :k], density=None if den is None else den[:, :k])
            assert np.array_equal(_np(l2).view(np.uint8), leaves[:, :k].view(np.uint8)) and np.array_equal(_np(i2), info[:, :k])
    assert seen > 0
    return t


# ---- 1. the reference's leaves -----------------------------------------------------------------------------------------------------
GOLD = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "items_s*.npz")))
GOLD += sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "citems_s*.npz")))


@pytest.mark.parametrize("path", GOLD, ids=[os.path.basename(p) for p in GOLD])
def test_reference_leaves(path):
    """before every recorded step, the expansion of the item the reference expanded there (the override or the current item) equals the
    reference's leaf rows, rows 80..129 of the observation it saw; two other items ride along in the same call"""
    g = np.load(path)
    setting, continuous = int(g["setting"]), os.path.basename(path).startswith("c")
    b = _batch(1, setting, continuous, g["stream"][None])
    b.reset()
    rng = np.random.RandomState(3)
    checked = 0
    for t in range(len(g["rows"])):
        cur = _np(b.preview_items(1))[0, 0]
        first = g["item"][t] if g["override"][t] else cur
        others = _items(1, 2, continuous, rng, degenerate=False)[0].numpy()
        items = torch.as_tensor(np.concatenate([first[None, :3], others], 0)[None])
        den = torch.tensor([[first[3] if setting == 3 else 1.0, 1.0, 1.0]], dtype=torch.float64)
        leaves, info = b.expand_items(items, density=den)
        assert np.array_equal(_np(leaves)[0, 0].reshape(-1), g["seen"][t][80 * 9:130 * 9]), "leaves of step %d (override=%s)" % (t, bool(g["override"][t]))
        assert not _np(info)[0, :, 1].any()
        checked += int(_np(info)[0, 0, 5] > 0)
        if g["override"][t]:
            it = g["item"][t]
            b.set_items(torch.as_tensor(it[None, :3]), density=torch.tensor([it[3] if setting == 3 else 1.0]))
        b.step(actions=torch.as_tensor(g["rows"][t][None]).to(b.device))
    assert checked > len(g["rows"]) // 2
    b.close()


# ---- 2. equal to set_items ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", DOMAINS, ids=DOM_IDS)
@pytest.mark.parametrize("source", ["random", "stream"])
def test_equals_set_items(setting, continuous, source):
    n = 64
    s = _streams(n, setting, continuous, 300) if source == "stream" else None
    b, twin = _batch(n, setting, continuous, s), _batch(n, setting, continuous, s)
    _walk_and_compare(b, twin, continuous, np.random.RandomState(setting + 10 * continuous), density=setting == 3)
    b.close(); twin.close()


@pytest.mark.parametrize("lnes,shuffle", [("EV", False), ("EP", False), ("CP", False), ("FC", False), ("EMS", True), ("CP", True)])
def test_equals_set_items_lnes_shuffle(lnes, shuffle):
    n, setting = 32, 1
    s = _streams(n, setting, False, 300)
    b, twin = _batch(n, setting, False, s, LNES=lnes, shuffle=shuffle), _batch(n, setting, False, s, LNES=lnes, shuffle=shuffle)
    _walk_and_compare(b, twin, False, np.random.RandomState(7))
    b.close(); twin.close()


@pytest.mark.parametrize("name", NEEDS_ALIAS_D)
def test_equals_set_items_alias_cases(name):
    """the recorded trajectories on which the reference's object aliasing decides a placement, expanded along the way"""
    c = CASES[name]
    n = 8
    s = np.stack([case_stream(c, c["seed"], c["env"] + e, 400) for e in range(n)])
    pct_b200 = _pb()
    mk = lambda: pct_b200.PctBatch(n, c["setting"], container_size=c["container"], item_set=c["items"], internal_node_holder=c["nb"],
                                   leaf_node_holder=c["nl"], obs_dtype=torch.float64, item_stream=s, env_id_base=c["env"])
    b, twin = mk(), mk()
    cps = sorted({0, 5, 20, 60, c["steps"] // 2, c["steps"] - 1})
    _walk_and_compare(b, twin, False, np.random.RandomState(5), checkpoints=cps)
    b.close(); twin.close()


@pytest.mark.parametrize("cont,setting", [(False, 1), (False, 3), (True, 1)], ids=["d1", "d3", "c1"])
def test_equals_set_items_many_supports(cont, setting):
    """the many-support floors: stability tests on 9 .. 32 supports use the env's large-case scratch under the block's lock"""
    n = 16
    pct_b200 = _pb()
    mk = lambda: pct_b200.PctBatch(n, setting, container_size=M.container(cont), continuous=cont, internal_node_holder=M.NB,
                                   leaf_node_holder=M.NL, obs_dtype=torch.float64, item_stream=M.streams(cont, setting, n), size_minimum=M.unit(cont))
    b, twin = mk(), mk()
    b.reset(); twin.reset()
    rng = np.random.RandomState(9)
    pol = np.array(M.POLICY_ITEMS, dtype=np.float64) * M.unit(cont)
    build = [M.plan(cont, setting, e)[1] for e in range(n)]  # each env's build-up placement rows: the floors of small columns
    T = max(len(r) for r in build)
    ar = torch.arange(n, device=b.device)
    for t in range(T + 6):
        if t in (T, T + 5):  # every floor is in place
            items = torch.as_tensor(pol[rng.randint(0, len(pol), size=(n, 8))])
            _compare(b, twin, items, torch.as_tensor(rng.uniform(0.5, 2.0, size=(n, 8))) if setting == 3 else None)
        rows = _leaf_rows(b, b._obs)[ar, b.random_policy(M.PSEED, t).long()].clone()  # envs past their build-up: a random leaf
        for e in range(n):
            if t < len(build[e]):
                rows[e] = torch.as_tensor(build[e][t], dtype=rows.dtype)
        _, _, _, inf = b.step(actions=rows)
        assert not _np(inf)[:, 1].any()
    b.close(); twin.close()


def test_candidate_overflow_is_reported_not_kept():
    """an item whose full-coordinate candidate list crosses 1228 entries: its record carries cand_overflow, the env's flags stay 0 and
    the next step reports none"""
    c = load_capacity_cases()["d_cand_fc20_s2"]
    pct_b200 = _pb()
    n = 8
    mk = lambda: pct_b200.PctBatch(n, c["setting"], container_size=c["container"], item_set=c["items"], internal_node_holder=c["nb"],
                                   leaf_node_holder=c["nl"], obs_dtype=torch.float64, item_stream=np.stack([c["stream"]] * n),
                                   size_minimum=c["size_minimum"], LNES=c["lnes"])
    b, twin = mk(), mk()
    b.reset(); twin.reset()
    items = torch.tensor([[(1, 2, 3), (2, 3, 4), (1, 1, 2), (3, 3, 3)]] * n, dtype=torch.int32)
    _, info = _compare(b, twin, items)
    assert (info[:, 0, 1] & FLAG_CAND).all(), info[:, :, 1]
    assert not any(b.state(e)["flags"] for e in range(n))
    _, _, _, si = b.step(leaf_idx=torch.zeros(n, dtype=torch.int32, device=b.device))
    assert not _np(si)[:, 1].any()
    b.close(); twin.close()


# ---- 3. read-only ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", DOMAINS, ids=DOM_IDS)
def test_read_only(setting, continuous):
    """snapshots and the observation buffer are untouched, and a twin stepped without the call gives the same observations, rewards,
    dones and infos, with leaf-index and row actions, under the default delta rows"""
    n = 64
    s = _streams(n, setting, continuous, 300)
    A, B = _batch(n, setting, continuous, s), _batch(n, setting, continuous, s)
    A.reset(); B.reset()
    rng = np.random.RandomState(1)
    for t in range(80):
        snap0, obs0 = _snap(A), _np(A._obs)
        A.expand_items(_items(n, 3, continuous, rng))
        assert np.array_equal(_snap(A), snap0), "expand_items changed env records at step %d" % t
        assert np.array_equal(_np(A._obs), obs0), "expand_items wrote into the observation buffer at step %d" % t
        idx = A.random_policy(PSEED, t)
        if t % 2:
            rows = _leaf_rows(A, A._obs)[torch.arange(n, device=A.device), idx.long()].clone()
            oa, ob = A.step(actions=rows), B.step(actions=rows)
        else:
            oa, ob = A.step(leaf_idx=idx), B.step(leaf_idx=idx)
        for u, v in zip(oa, ob):
            assert torch.equal(u, v), t
    A.close(); B.close()


# ---- 4. indexing and errors --------------------------------------------------------------------------------------------------------
def test_env_idx_and_errors():
    pct_b200 = _pb()
    n = 16
    b = _batch(n, 1, False)
    items = torch.full((n, 2, 3), 2, dtype=torch.int32)
    L, h = b.L, b.h
    ptr = lambda t: C.c_void_p(t.data_ptr())
    dl = torch.zeros((n, 2, b.nl, 9), dtype=b.obs_dtype, device=b.device)
    di = items.to(b.device)
    assert L.pct_expand_items(h, None, n, 2, ptr(di), None, ptr(dl), None, None) == -4  # PCT_ERR_STATE before pct_reset
    with pytest.raises(pct_b200.PctError):
        b.expand_items(items)
    b.reset()
    for t in range(6):
        b.step(leaf_idx=b.random_policy(PSEED, t))
    rng = np.random.RandomState(2)
    items = _items(n, 3, False, rng)
    full_l, full_i = [_np(x) for x in b.expand_items(items)]
    perm = np.random.RandomState(4).permutation(n)[:10].astype(np.int32)
    l, i = [_np(x) for x in b.expand_items(items[perm], env_idx=perm)]
    assert np.array_equal(l, full_l[perm]) and np.array_equal(i, full_i[perm])
    idx = torch.tensor([5, -1, 3, n], dtype=torch.int32)
    l, i = [_np(x) for x in b.expand_items(items[[5, 0, 3, 1]], env_idx=idx)]
    assert np.array_equal(l[0], full_l[5]) and np.array_equal(l[2], full_l[3]) and np.array_equal(i[2], full_i[3])
    assert not l[1].any() and not l[3].any() and not i[1].any() and not i[3].any(), "out-of-range rows are zeros"
    dec = b.decode_info(torch.as_tensor(full_i).reshape(-1, 8))
    assert (dec["counter"] == np.repeat([b.state(e)["n_boxes"] for e in range(n)], 3)).all()
    # C ABI
    assert L.pct_expand_items(h, None, -1, 2, ptr(di), None, ptr(dl), None, None) == -1
    assert L.pct_expand_items(h, None, n, 0, ptr(di), None, ptr(dl), None, None) == -1
    assert L.pct_expand_items(h, None, 1 << 12, 1 << 12, ptr(di), None, ptr(dl), None, None) == -1  # n * k * nl * 9 > INT32_MAX
    assert L.pct_expand_items(h, None, 0, 2, None, None, None, None, None) == 0
    assert L.pct_expand_items(h, None, n, 2, None, None, ptr(dl), None, None) == -1
    # Python checks
    for bad in (torch.ones((n, 3)), torch.ones((n, 2, 2)), torch.ones((n, 0, 3))):
        with pytest.raises(pct_b200.PctError):
            b.expand_items(bad)
    with pytest.raises(pct_b200.PctError):
        b.expand_items(torch.ones((2, 1, 3)), env_idx=[0, 1, 2])
    with pytest.raises(pct_b200.PctError):
        b.expand_items(torch.ones((n + 1, 1, 3)))
    with pytest.raises(pct_b200.PctError):
        b.expand_items(torch.ones((2, 2, 3)), density=torch.ones(2))
    with pytest.raises(pct_b200.PctError):
        b.expand_items(torch.ones((2, 2, 3)), out=(torch.zeros((2, 2, b.nl, 9), dtype=torch.float32, device=b.device),
                                                   torch.zeros((2, 2, 8), dtype=torch.int32, device=b.device)))
    with pytest.raises(pct_b200.PctError):
        b.expand_items(torch.ones((2, 2, 3)), out=(dl[:2],))
    o = (torch.zeros((2, 3, b.nl, 9), dtype=b.obs_dtype, device=b.device), torch.zeros((2, 3, 8), dtype=torch.int32, device=b.device))
    r = b.expand_items(items[:2], out=o)
    assert r[0] is o[0] and r[1] is o[1] and np.array_equal(_np(o[0]), full_l[:2])
    e0 = b.expand_items(torch.zeros((0, 2, 3)))
    assert e0[0].shape == (0, 2, b.nl, 9) and e0[1].shape == (0, 2, 8)
    b.close()


# ---- 5. graph capture --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", [(1, False), (1, True)], ids=["d1", "c1"])
def test_graph_capture(setting, continuous):
    """preview -> expand -> choose (the item with more leaves, its first leaf) -> set_items -> step, captured once and replayed against
    the same loop run eagerly"""
    n = 64
    s = _streams(n, setting, continuous, 300)
    G, E = _batch(n, setting, continuous, s), _batch(n, setting, continuous, s)
    qd = torch.float64 if continuous else torch.int32
    bufs = {}
    for b in (G, E):
        b.reset()
        bufs[b] = dict(pv=torch.zeros((n, 2, 4), dtype=torch.float64, device=b.device), it=torch.zeros((n, 2, 3), dtype=qd, device=b.device),
                       lv=torch.zeros((n, 2, b.nl, 9), dtype=b.obs_dtype, device=b.device),
                       inf=torch.zeros((n, 2, 8), dtype=torch.int32, device=b.device), idx=torch.zeros((n,), dtype=torch.int32, device=b.device))

    def body(b):
        q = bufs[b]
        b.preview_items(2, out=q["pv"])
        q["it"].copy_(q["pv"][:, :, :3])
        b.expand_items(q["it"], density=q["pv"][:, :, 3].contiguous(), out=(q["lv"], q["inf"]))
        j = (q["inf"][:, 1, 5] > q["inf"][:, 0, 5]).long()
        ar = torch.arange(n, device=b.device)
        b.set_items(q["it"][ar, j], density=q["pv"][ar, j, 3].contiguous())
        return b.step(leaf_idx=q["idx"]) + (q["lv"], q["inf"])

    for b in (G, E):
        body(b)
    st = torch.cuda.Stream(device=G.device)
    st.wait_stream(torch.cuda.current_stream(G.device))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(st):
        with torch.cuda.graph(g, stream=st):
            out = body(G)
    torch.cuda.current_stream(G.device).wait_stream(st)
    for t in range(8):
        g.replay()
        ref = body(E)
        torch.cuda.synchronize()
        for u, v in zip(out, ref):
            assert torch.equal(u, v), t
    G.close(); E.close()


# ---- 6. buffer packing on the expansion -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", [(1, False), (2, False), (3, False), (1, True), (3, True)], ids=["d1", "d2", "d3", "c1", "c3"])
def test_buffer_policy_replays_as_a_stream(setting, continuous):
    """B = 3: a policy picks uniformly among the valid (item, leaf) pairs of the expansion, then set_items(item) and step(leaf); the
    set_items observation's leaf equals the expansion's row, and the packed items replay as a plain stream on the library and the oracle"""
    n, B, L = 256, 3, 400
    src = torch.as_tensor(_streams(n, setting, continuous, L, seed=21)).cuda()
    own = _streams(n, setting, continuous, L, seed=22)
    P = _batch(n, setting, continuous, own)
    P.reset()
    gen = torch.Generator(device=P.device)
    gen.manual_seed(17)
    buf, pos, ar = src[:, :B].clone(), B, torch.arange(n, device=P.device)
    nl = P.nl
    chosen, idxs, obs_set, rews, dones = [], [], [], [], []
    eps = np.zeros(n, dtype=int)
    for t in range(300):
        leaves, info = P.expand_items(buf[:, :, :3], density=buf[:, :, 3].contiguous())
        valid = (torch.arange(nl, device=P.device)[None, None, :] < info[:, :, 5:6]).reshape(n, B * nl).to(torch.float64)
        none = valid.sum(1) == 0
        valid[none, 0] = 1.0  # no placement for any buffered item: item 0, leaf 0 (an empty row; the episode ends)
        pick = torch.multinomial(valid, 1, generator=gen)[:, 0]
        j, leaf = pick // nl, (pick % nl).to(torch.int32)
        item = buf[ar, j].clone()
        obs = P.set_items(item[:, :3], density=item[:, 3].contiguous()).clone()
        assert torch.equal(_leaf_rows(P, obs)[ar, leaf.long()], leaves[ar, j, leaf.long()]), "set_items leaf differs from the expansion at step %d" % t
        _, r, d, inf = P.step(leaf_idx=leaf)
        assert not (_np(inf)[:, 1] & ~2).any(), "flags"
        chosen.append(_np(item)); idxs.append(_np(leaf)); obs_set.append(_np(obs)); rews.append(_np(r)); dones.append(_np(d))
        buf[ar, j] = src[:, pos % L]
        pos += 1
        eps += dones[-1].astype(int)
        if eps.min() >= 2:
            break
    assert eps.min() >= 2
    T = len(chosen)
    seq = np.concatenate([np.stack(chosen, 1), np.tile(_np(src[:, :1]), (1, 2, 1))], 1)
    if not continuous:
        seq[:, :, :3] = np.trunc(seq[:, :, :3])
    R = _batch(n, setting, continuous, seq)
    R.reset()
    for t in range(T):
        assert np.array_equal(_np(R._obs), obs_set[t]), "replay observation differs at step %d" % t
        _, r, d, _ = R.step(leaf_idx=torch.as_tensor(idxs[t]).to(R.device))
        assert np.array_equal(_np(r), rews[t]) and np.array_equal(_np(d), dones[t]), t
    R.close()
    for e in range(0, n, 32):  # the oracle on the same streams, with the chosen leaf rows as actions
        o = (OracleContinuous(setting, stream=seq[e]) if continuous else OracleDiscrete(setting, stream=seq[e]))
        ob = o.reset()
        for t in range(T):
            assert np.array_equal(ob, obs_set[t][e]), (e, t)
            ob, r, d, _ = o.step(_leaf_rows(P, obs_set[t][e][None])[0, idxs[t][e]].astype(np.float64))
            assert np.float32(r) == rews[t][e] and bool(d) == bool(dones[t][e]), (e, t)
            if d:
                ob = o.reset()
    P.close()


@pytest.mark.parametrize("setting,continuous", [(1, False), (3, False), (1, True)], ids=["d1", "d3", "c1"])
def test_equals_buffer_driver_fan_out(setting, continuous):
    """for every env and buffered item j, the expansion equals child j's leaf rows after BufferDriver's fan-out (snapshot -> restore into
    n * B envs -> set_items)"""
    n, B, L = 64, 3, 300
    src = torch.as_tensor(_streams(n, setting, continuous, L, seed=21))
    P = _batch(n, setting, continuous, _streams(n, setting, continuous, L, seed=22))
    Cb = _batch(n * B, setting, continuous, _streams(n * B, setting, continuous, 8, seed=23))
    P.reset(); Cb.reset()
    drv = BufferDriver(P, Cb, src, B)
    for t in range(40):
        leaves, info = P.expand_items(drv.buf[:, :, :3], density=drv.buf[:, :, 3].contiguous())
        chosen, act, j = drv.decide()  # fans out: Cb holds child (e, j) at row e * B + j
        got = _leaf_rows(Cb, Cb._obs).reshape(n, B, Cb.nl, 9)
        assert torch.equal(got, leaves), "step %d" % t
        P.set_items(chosen[:, :3], density=chosen[:, 3])
        P.step(actions=act)
        drv.buf[drv.envs, j] = drv.src[:, drv.pos % L]
        drv.pos += 1
    P.close(); Cb.close()
