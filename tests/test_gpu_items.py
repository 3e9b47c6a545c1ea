"""GPU: item preview and item override (pct_preview_items / pct_set_items, PctBatch.preview_items / set_items).

The preview is checked against each env's state, against the items later steps actually place and against the item streams.  The
override is checked against the library itself, bit for bit: a batch whose stream differs at random places, corrected by set_items
with the other batch's preview, must produce the other batch's observations, rewards, dones and infos.  A buffer-packing driver on
public calls only is replayed as a plain stream on a twin batch and on the oracle.
"""
import ctypes as C
import glob
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
from buffer_compose import BufferDriver  # noqa: E402
from harness import CASES, ITEM_SET, NEEDS_ALIAS_D, OracleDiscrete, case_stream, make_stream  # noqa: E402
from pct_oracle import OracleContinuous, make_continuous_stream  # noqa: E402

pytestmark = pytest.mark.gpu
PSEED = 4321
DOMAINS = [(s, False) for s in (1, 2, 3)] + [(s, True) for s in (1, 2, 3)]
DOM_IDS = ["d%d" % s if not c else "c%d" % s for s, c in DOMAINS]
BAD_ACTION = 2
NO_ROW = np.array((1, 0, 0, 1, 0, 0, 0, 0, 1), dtype=np.float32)  # heuristic_actions' "no placement" row (discrete)
SENTINEL = (100, 100, 100)  # LoadBoxCreator's end-of-trajectory item (D:binCreator.py:64): fits nowhere


def _pb():
    import pct_b200
    return pct_b200


def _streams(n, setting, continuous, length, seed=11, env_base=0):
    if continuous:
        return np.stack([make_continuous_stream(seed, env_base + e, length, setting) for e in range(n)])
    return np.stack([make_stream(seed, env_base + e, length, setting) for e in range(n)])


def _batch(n, setting, continuous, stream=None, **kw):
    """a float64-observation batch: per-env `stream`, else the random item source (item set / continuous sample_from_distribution)"""
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


def _np(t):
    return t.cpu().numpy().copy()


def _snap(b):
    """every env's record; a zeroed buffer, so that the bytes behind the live parts of the records compare equal too"""
    return _np(b.snapshot(out=torch.zeros((b.n_envs, b.snapshot_bytes), dtype=torch.uint8, device=b.device)))


def _step(b, t):
    return [_np(x) for x in b.step(leaf_idx=b.random_policy(PSEED, t))]


# ---- 1-3. preview ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", DOMAINS, ids=DOM_IDS)
@pytest.mark.parametrize("source", ["random", "stream"])
def test_preview_matches_state_and_later_steps(setting, continuous, source):
    n, K, L = 64, 6, 7  # a 7-item stream wraps within the episode
    stream = _streams(n, setting, continuous, L) if source == "stream" else None
    b = _batch(n, setting, continuous, stream)
    b.reset()
    for t in range(3):
        _step(b, t)
    snap0 = _snap(b)
    pv = _np(b.preview_items(K))
    assert np.array_equal(_snap(b), snap0), "preview_items changed env records"
    assert pv.shape == (n, K, 4)
    for e in range(n):  # column 0 = the state's current item
        s = b.state(e)
        assert list(pv[e, 0, :3]) == list(s["next_box"]) and pv[e, 0, 3] == s["next_den"], e
        if stream is not None:  # columns 1.. = the stream at draw_pos + j - 1, cyclically
            for j in range(1, K):
                it = stream[e, (s["draw_pos"] + j - 1) % L]
                want = np.trunc(it[:3]) if not continuous else it[:3]
                assert list(pv[e, j, :3]) == list(want) and pv[e, j, 3] == (it[3] if setting == 3 else 1.0), (e, j)
    alive = np.ones(n, dtype=bool)
    for j in range(1, K):  # columns 1.. = the current items of the following steps, for envs without a done in between
        _, _, done, _ = _step(b, 3 + j - 1)
        alive &= done == 0
        cur = _np(b.preview_items(1))[:, 0]
        assert np.array_equal(cur[alive], pv[alive, j]), j
    assert alive.sum() > n // 2
    if setting == 3:
        assert len(np.unique(pv[:, :, 3])) > n  # real densities, not 1.0
    b.close()


def test_preview_rows_and_env_idx():
    b = _batch(16, 1, False)
    b.reset()
    full = _np(b.preview_items(3))
    idx = torch.tensor([5, -1, 3, 16], dtype=torch.int32)
    pv = _np(b.preview_items(3, env_idx=idx))
    assert np.array_equal(pv[0], full[5]) and np.array_equal(pv[2], full[3])
    assert not pv[1].any() and not pv[3].any(), "out-of-range rows are zeros"
    b.close()


# ---- 4. twin streams ---------------------------------------------------------------------------------------------------------------
def _perturb(stream, continuous, setting, rate=0.3, seed=5):
    rng = np.random.RandomState(seed)
    s2 = stream.copy()
    m = rng.rand(*stream.shape[:2]) < rate
    if continuous:
        other = _streams(stream.shape[0], setting, True, stream.shape[1], seed=99)
    else:
        other = np.stack([make_stream(77, e, stream.shape[1], setting) for e in range(stream.shape[0])])
    s2[m] = other[m]
    return s2


def _twin(A, B, steps, episodes=2):
    """B follows A's current items through set_items; returns the number of set_items calls that changed something"""
    A.reset()
    B.reset()
    n, eps, changed = A.n_envs, np.zeros(A.n_envs, dtype=int), 0
    a_info, a_done = None, None
    for t in range(steps):
        pa, pb = A.preview_items(1)[:, 0], B.preview_items(1)[:, 0]
        diff = torch.nonzero((pa != pb).any(1)).flatten().to(torch.int32)
        binfo = torch.zeros((n, 8), dtype=torch.int32, device=B.device)
        obs_b = B.set_items(pa[diff.long(), :3], env_idx=diff, density=pa[diff.long(), 3], info=binfo)
        changed += int(diff.numel())
        assert torch.equal(obs_b, A._obs), "observation after set_items differs at step %d" % t
        if a_info is not None and diff.numel():  # (n == 0 is a no-op: no info records are written)
            assert np.array_equal(_np(binfo)[:, 5:], a_info[:, 5:]), "n_leaf / n_cand / n_ems differ at step %d" % t
            live = a_done == 0  # a finished env's step record describes the episode before its reset
            assert np.array_equal(_np(binfo)[live, :2], a_info[live, :2]), "counter / flags differ at step %d" % t
        assert not _np(binfo)[:, 1].any(), "flags"
        idx = A.random_policy(PSEED, t)
        oa = [_np(x) for x in A.step(leaf_idx=idx)]
        ob = [_np(x) for x in B.step(leaf_idx=idx)]
        for k, nm in ((1, "reward"), (2, "done")):
            assert np.array_equal(oa[k], ob[k]), "%s differs at step %d" % (nm, t)
        assert np.array_equal(oa[3][:, :5], ob[3][:, :5]), "info differs at step %d" % t
        a_info, a_done = oa[3], oa[2]
        eps += oa[2].astype(int)
        if eps.min() >= episodes:
            break
    assert eps.min() >= episodes, "not every env finished %d episodes" % episodes
    assert changed > 0
    return changed


@pytest.mark.parametrize("setting,continuous", DOMAINS, ids=DOM_IDS)
def test_twin_streams(setting, continuous):
    n, L = 64, 200
    s = _streams(n, setting, continuous, L)
    A, B = _batch(n, setting, continuous, s), _batch(n, setting, continuous, _perturb(s, continuous, setting))
    _twin(A, B, 400)
    A.close(); B.close()


@pytest.mark.parametrize("lnes,shuffle", [("EV", False), ("EP", False), ("CP", False), ("FC", False), ("EMS", True), ("CP", True)])
def test_twin_streams_lnes_shuffle(lnes, shuffle):
    n, L, setting = 32, 200, 1
    s = _streams(n, setting, False, L)
    A = _batch(n, setting, False, s, LNES=lnes, shuffle=shuffle)
    B = _batch(n, setting, False, _perturb(s, False, setting), LNES=lnes, shuffle=shuffle)
    _twin(A, B, 400)
    A.close(); B.close()


@pytest.mark.parametrize("name", NEEDS_ALIAS_D)
def test_twin_streams_alias_cases(name):
    """the recorded trajectories on which the reference's object aliasing decides a real placement: env 0 follows the recorded env"""
    c = CASES[name]
    n, L = 8, 400
    s = np.stack([case_stream(c, c["seed"], c["env"] + e, L) for e in range(n)])
    pct_b200 = _pb()
    mk = lambda st: pct_b200.PctBatch(n, c["setting"], container_size=c["container"], item_set=c["items"], internal_node_holder=c["nb"],
                                      leaf_node_holder=c["nl"], obs_dtype=torch.float64, item_stream=st, env_id_base=c["env"])
    A, B = mk(s), mk(_perturb(s, False, c["setting"]))
    _twin(A, B, max(400, c["steps"] + 40), episodes=1)
    A.close(); B.close()


VARIANTS = [("PCT_B200_WALK", "fork", False), ("PCT_B200_WALK", "fork", True), ("PCT_B200_K3", "block", False), ("PCT_B200_K3", "block", True),
            ("PCT_B200_GROUPS", "2", False), ("PCT_B200_OVERLAP", "0", False)]


@pytest.mark.parametrize("var,val,continuous", VARIANTS, ids=["%s=%s-%s" % (v, x, "c1" if c else "d1") for v, x, c in VARIANTS])
def test_twin_streams_launch_variants(monkeypatch, var, val, continuous):
    """the override path under the opt-in launch variants: fork-join walks, the block-per-env feasibility kernel, a step split over
    internal streams (set_items itself always runs the whole batch on the caller's stream), the non-overlapped step order"""
    monkeypatch.setenv(var, val)
    n, L, setting = 256, 200, 1
    s = _streams(n, setting, continuous, L)
    A, B = _batch(n, setting, continuous, s), _batch(n, setting, continuous, _perturb(s, continuous, setting))
    _twin(A, B, 400)
    A.close(); B.close()


# ---- 5. the reference's own overrides (tests/golden/make_item_golden.py) ----------------------------------------------------------
GOLD = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "items_s*.npz")))
GOLD += sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "citems_s*.npz")))


@pytest.mark.parametrize("path", GOLD, ids=[os.path.basename(p) for p in GOLD])
def test_reference_overrides_replay(path):
    """the recorded stream, with set_items at the recorded override steps, replays the reference's observations, rewards, dones and counters"""
    g = np.load(path)
    setting, continuous = int(g["setting"]), os.path.basename(path).startswith("c")
    b = _batch(1, setting, continuous, g["stream"][None])
    obs = _np(b.reset())[0]
    overridden = {int(g["draw"][t]) for t in np.nonzero(g["override"])[0]}
    for t in range(len(g["rows"])):
        if g["override"][t]:
            it = g["item"][t]
            obs = _np(b.set_items(torch.as_tensor(it[None, :3]), density=torch.tensor([it[3] if setting == 3 else 1.0])))[0]
        assert np.array_equal(obs, g["seen"][t]), "observation seen at step %d (override=%s)" % (t, bool(g["override"][t]))
        o, r, d, info = [_np(x) for x in b.step(actions=torch.as_tensor(g["rows"][t][None]).to(b.device))]
        assert r[0] == np.float32(g["reward"][t]) and bool(d[0]) == bool(g["done"][t]) and info[0, 0] == g["counter"][t], t
        assert not info[0, 1], "flags"
        obs = o[0]
        if int(g["draw"][t]) + 1 not in overridden:  # the next draw's observation (after the auto-reset on a done)
            assert np.array_equal(obs, g["after"][t]), "observation after step %d" % t
    b.close()


# ---- 6-7. envs not listed, snapshots after set_items -------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", DOMAINS, ids=DOM_IDS)
def test_unlisted_envs_unchanged_and_snapshot_after_set(setting, continuous):
    n = 48
    s = _streams(n, setting, continuous, 300)
    b = _batch(n, setting, continuous, s)
    b.reset()
    for t in range(5):
        _step(b, t)
    obs0, snap0 = _np(b._obs), _snap(b)
    listed = np.arange(0, n, 3).astype(np.int32)
    draws = [b.state(int(e))["draw_pos"] for e in listed]
    new = s[listed, 250]  # other items of the same kind
    obs1 = _np(b.set_items(torch.as_tensor(new[:, :3]), env_idx=listed, density=torch.as_tensor(new[:, 3])))
    snap1 = _snap(b)
    rest = np.setdiff1d(np.arange(n), listed)
    assert np.array_equal(obs1[rest], obs0[rest]) and np.array_equal(snap1[rest], snap0[rest])
    pv = _np(b.preview_items(1))[:, 0]
    want = np.trunc(new[:, :3]) if not continuous else new[:, :3]
    assert np.array_equal(pv[listed, :3], want)
    assert np.array_equal(pv[listed, 3], new[:, 3])
    assert [b.state(int(e))["draw_pos"] for e in listed] == draws, "set_items consumed a draw"
    # a snapshot taken after set_items restores into a fresh handle, which continues identically
    f = _batch(n, setting, continuous, s)
    f.reset()
    fo = _np(f.restore(b.snapshot()))
    assert np.array_equal(fo, obs1)
    for t in range(5, 25):
        idx = b.random_policy(PSEED, t)
        x, y = [_np(v) for v in b.step(leaf_idx=idx)], [_np(v) for v in f.step(leaf_idx=idx)]
        for u, v in zip(x, y):
            assert np.array_equal(u, v), t
    b.close(); f.close()


# ---- 8. delta rows -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", [(1, False), (2, False), (1, True)], ids=["d1", "d2", "c1"])
def test_delta_rows(setting, continuous, monkeypatch):
    n = 32
    s = _streams(n, setting, continuous, 300)
    X = _batch(n, setting, continuous, s)
    monkeypatch.setenv("PCT_B200_OBS_DELTA", "0")
    Y = _batch(n, setting, continuous, s)
    monkeypatch.delenv("PCT_B200_OBS_DELTA")
    Z = _batch(n, setting, continuous, s)
    bufs = [torch.zeros_like(X._obs), torch.zeros_like(X._obs)]
    X.reset(); Y.reset(); Z.reset(out=bufs[1])
    rng = np.random.RandomState(3)
    for t in range(60):
        sub = np.sort(rng.choice(n, 8, replace=False)).astype(np.int32)
        it = s[sub, rng.randint(0, 300)]
        args = (torch.as_tensor(it[:, :3]),)
        kw = dict(env_idx=sub, density=torch.as_tensor(it[:, 3]))
        ox, oy, oz = _np(X.set_items(*args, **kw)), _np(Y.set_items(*args, **kw)), _np(Z.set_items(*args, out=bufs[t % 2], **kw))
        assert np.array_equal(ox, oy) and np.array_equal(ox, oz), t
        idx = X.random_policy(PSEED, t)
        ox, oy, oz = _np(X.step(leaf_idx=idx)[0]), _np(Y.step(leaf_idx=idx)[0]), _np(Z.step(leaf_idx=idx, out=bufs[(t + 1) % 2])[0])
        assert np.array_equal(ox, oy) and np.array_equal(ox, oz), t
    X.close(); Y.close(); Z.close()


# ---- 9. edge cases -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", [(1, False), (1, True)], ids=["d1", "c1"])
def test_graph_capture(setting, continuous):
    """preview_items -> set_items (each env swaps in its next item: a one-step lookahead) -> step, captured once, replayed"""
    n = 64
    s = _streams(n, setting, continuous, 300)
    G, E = _batch(n, setting, continuous, s), _batch(n, setting, continuous, s)
    qd = torch.float64 if continuous else torch.int32
    bufs = {}
    for b in (G, E):
        b.reset()
        bufs[b] = dict(pv=torch.zeros((n, 2, 4), dtype=torch.float64, device=b.device), it=torch.zeros((n, 3), dtype=qd, device=b.device),
                       den=torch.zeros((n,), dtype=torch.float64, device=b.device), idx=torch.zeros((n,), dtype=torch.int32, device=b.device))

    def body(b):
        q = bufs[b]
        b.preview_items(2, out=q["pv"])
        q["it"].copy_(q["pv"][:, 1, :3])
        q["den"].copy_(q["pv"][:, 1, 3])
        b.set_items(q["it"], density=q["den"])
        return b.step(leaf_idx=q["idx"])

    for b in (G, E):  # warm-up outside the capture
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


@pytest.mark.parametrize("setting,continuous", [(1, False), (3, False), (1, True), (2, True)], ids=["d1", "d3", "c1", "c2"])
def test_oversize_item_ends_episode_like_a_stream_item(setting, continuous):
    n = 8
    s = _streams(n, setting, continuous, 100)
    s2 = s.copy()
    s2[0, 0, :3] = SENTINEL
    A, B = _batch(n, setting, continuous, s2), _batch(n, setting, continuous, s)
    oa = _np(A.reset())
    B.reset()
    info = torch.zeros((n, 8), dtype=torch.int32, device=B.device)
    ob = _np(B.set_items(torch.tensor([SENTINEL], dtype=torch.float64), env_idx=[0], info=info))
    assert np.array_equal(oa, ob)
    assert _np(info)[0, 5] == 0, "an item that fits nowhere has no leaves"
    idx = torch.zeros((n,), dtype=torch.int32, device=A.device)
    ra, rb = [_np(x) for x in A.step(leaf_idx=idx)], [_np(x) for x in B.step(leaf_idx=idx)]
    assert ra[2][0] == 1 and ra[1][0] == 0
    for u, v in zip(ra, rb):
        assert np.array_equal(u, v)
    A.close(); B.close()


@pytest.mark.parametrize("continuous", [False, True], ids=["d1", "c1"])
def test_failed_step_without_auto_reset_keeps_the_set_item(continuous):
    """documented difference: the reference's terminal observation re-reads the creator's head (the item the source delivered); here the
    env keeps the set item, so the terminal observation is the one set_items wrote for it"""
    n = 4
    s = _streams(n, 1, continuous, 50)
    b = _batch(n, 1, continuous, s, auto_reset=False)
    o0 = _np(b.reset())
    o_set = _np(b.set_items(torch.tensor([SENTINEL], dtype=torch.float64), env_idx=[0]))
    obs, rew, done, _ = [_np(x) for x in b.step(leaf_idx=torch.zeros((n,), dtype=torch.int32, device=b.device))]
    assert done[0] == 1 and rew[0] == 0
    assert np.array_equal(obs[0], o_set[0]), "terminal observation = the set item's observation"
    assert not np.array_equal(obs[0], o0[0]), "... not the one of the item the source delivered (the reference's)"
    assert list(_np(b.preview_items(1))[0, 0, :3]) == list(SENTINEL)
    b.close()


def test_errors():
    pct_b200 = _pb()
    b = _batch(4, 1, False)
    L, h = b.L, b.h
    buf = torch.zeros((4, 2, 4), dtype=torch.float64, device=b.device)
    items = torch.ones((4, 3), dtype=torch.int32, device=b.device)
    ptr = lambda t: C.c_void_p(t.data_ptr())
    assert L.pct_preview_items(h, None, 4, 2, ptr(buf), None) == -4  # PCT_ERR_STATE before pct_reset
    assert L.pct_set_items(h, None, 4, ptr(items), None, ptr(b._obs), None, None) == -4
    with pytest.raises(pct_b200.PctError):
        b.preview_items(2)
    b.reset()
    assert L.pct_preview_items(h, None, -1, 2, ptr(buf), None) == -1
    assert L.pct_preview_items(h, None, 4, 0, ptr(buf), None) == -1
    assert L.pct_preview_items(h, None, 1 << 16, 1 << 16, ptr(buf), None) == -1
    assert L.pct_preview_items(h, None, 0, 2, None, None) == 0
    assert L.pct_set_items(h, None, -1, ptr(items), None, ptr(b._obs), None, None) == -1
    assert L.pct_set_items(h, None, 0, None, None, None, None, None) == 0
    with pytest.raises(pct_b200.PctError):
        b.preview_items(0)
    with pytest.raises(pct_b200.PctError):
        b.set_items(torch.ones((4, 2)))
    with pytest.raises(pct_b200.PctError):
        b.set_items(torch.ones((2, 3)), env_idx=[0, 1, 2])
    with pytest.raises(pct_b200.PctError):
        b.set_items(torch.ones((5, 3)))
    with pytest.raises(pct_b200.PctError):
        b.set_items(torch.ones((2, 3)), density=torch.ones(3))
    # out-of-range envs are skipped
    before = _snap(b)
    b.set_items(torch.full((2, 3), 2), env_idx=[-1, 4])
    assert np.array_equal(_snap(b), before)
    b.close()


# ---- 10. buffer driver -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", [(1, False), (2, False), (3, False), (1, True), (3, True)], ids=["d1", "d2", "d3", "c1", "c3"])
def test_buffer_driver_replays_as_a_stream(setting, continuous):
    n, B, L = 256, 3, 400
    src = _streams(n, setting, continuous, L, seed=21)
    own = _streams(n, setting, continuous, L, seed=22)  # the parent's own source: every item it draws is overridden
    P, Cb = _batch(n, setting, continuous, own), _batch(n * B, setting, continuous, _streams(n * B, setting, continuous, 8, seed=23))
    P.reset(); Cb.reset()
    drv = BufferDriver(P, Cb, torch.as_tensor(src), B)
    chosen, acts, obs_set, rews, dones = [], [], [], [], []
    eps = np.zeros(n, dtype=int)
    for t in range(300):
        c, a, o, out = drv.step()
        chosen.append(_np(c)); acts.append(_np(a)); obs_set.append(o.cpu().numpy()); rews.append(_np(out[1])); dones.append(_np(out[2]))
        assert not (_np(out[3])[:, 1] & ~BAD_ACTION).any(), "flags"  # bad_action: the heuristic found no placement, the episode ends
        eps += dones[-1].astype(int)
        if eps.min() >= 2:
            break
    assert eps.min() >= 2
    T = len(chosen)
    seq = np.concatenate([np.stack(chosen, 1), np.tile(src[:, :1], (1, 2, 1))], 1)  # item of draw t = the item chosen at step t (+ padding)
    if not continuous:
        seq[:, :, :3] = np.trunc(seq[:, :, :3])
    R = _batch(n, setting, continuous, seq)
    R.reset()
    for t in range(T):
        assert np.array_equal(_np(R._obs), obs_set[t]), "replay observation differs at step %d" % t
        _, r, d, _ = R.step(actions=torch.as_tensor(acts[t]).to(R.device))
        assert np.array_equal(_np(r), rews[t]) and np.array_equal(_np(d), dones[t]), t
    R.close()
    for e in range(0, n, 16):  # the oracle on the same streams and rows
        o = (OracleContinuous(setting, stream=seq[e]) if continuous else OracleDiscrete(setting, stream=seq[e]))
        ob = o.reset()
        for t in range(T):
            assert np.array_equal(ob, obs_set[t][e]), (e, t)
            if not continuous and np.array_equal(acts[t][e], NO_ROW):  # no placement: the reference ends the episode without stepping
                assert dones[t][e] and rews[t][e] == 0, (e, t)
                ob = o.reset()
                continue
            ob, r, d, _ = o.step(acts[t][e].astype(np.float64))
            assert np.float32(r) == rews[t][e] and bool(d) == bool(dones[t][e]), (e, t)
            if d:
                ob = o.reset()
    P.close(); Cb.close()
