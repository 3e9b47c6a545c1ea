"""GPU: per-env reset (pct_reset_envs, PctBatch.reset(env_idx=..., mask=...)).

A batch without auto-reset that calls reset(mask=done) after every step must reproduce, bit for bit, the batch with the auto-reset
(the reference's ShmemVecEnv worker calls env.reset() right after a finished step, wrapper/shmem_vec_env.py:139-143).  Terminal
observations and mid-episode resets are checked against one oracle env per env; the rest checks that unlisted envs stay untouched,
the delta-row buffer contract, the interaction with set_items and LSAH, graph capture and the error cases.
"""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
from harness import CASES, ITEM_SET, NEEDS_ALIAS_D, case_stream, make_stream, policy_pick  # noqa: E402
from pct_oracle import OracleContinuous, OracleDiscrete, make_continuous_stream  # noqa: E402

pytestmark = pytest.mark.gpu
PSEED = 4321
DOMAINS = [(s, False) for s in (1, 2, 3)] + [(s, True) for s in (1, 2, 3)]
DOM_IDS = ["d%d" % s if not c else "c%d" % s for s, c in DOMAINS]
SENTINEL = (100, 100, 100)  # an item that fits nowhere


def _pb():
    import pct_b200
    return pct_b200


def _streams(n, setting, continuous, length, seed=11):
    if continuous:
        return np.stack([make_continuous_stream(seed, e, length, setting) for e in range(n)])
    return np.stack([make_stream(seed, e, length, setting) for e in range(n)])


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


# ---- 1. twin batches: auto-reset against reset(mask=done) -----------------------------------------------------------------------
def _twin(A, B, steps, episodes=2):
    """A auto-resets; B (auto_reset=False) runs reset(mask=done) on the step's own done buffer after every step"""
    assert torch.equal(A.reset(), B.reset())
    n, eps = A.n_envs, np.zeros(A.n_envs, dtype=int)
    rinfo = torch.zeros((n, 8), dtype=torch.int32, device=B.device)
    for t in range(steps):
        idx = A.random_policy(PSEED, t)
        oa = [_np(x) for x in A.step(leaf_idx=idx)]
        ob = [_np(x) for x in B.step(leaf_idx=idx)]
        for k, nm in ((1, "reward"), (2, "done")):
            assert np.array_equal(oa[k], ob[k]), "%s differs at step %d" % (nm, t)
        done = oa[2] != 0
        assert np.array_equal(oa[3][:, :5], ob[3][:, :5]), "info differs at step %d" % t  # the terminal records
        assert np.array_equal(oa[3][~done, 5:], ob[3][~done, 5:]), "n_leaf / n_cand / n_ems differ at step %d" % t
        assert np.array_equal(ob[0][~done], oa[0][~done]), "observation of a live env differs at step %d" % t
        obs_b = B.reset(mask=B._done, info=rinfo)
        assert torch.equal(obs_b, A._obs), "observation after reset(mask=done) differs at step %d" % t
        ri = _np(rinfo)
        assert np.array_equal(ri[:, 5:], oa[3][:, 5:]), "n_leaf / n_cand / n_ems of the reset differ at step %d" % t
        assert np.array_equal(ri[~done, :2], oa[3][~done, :2]) and not ri[done, :2].any() and not ri[:, 2:5].any(), t
        eps += done.astype(int)
        if eps.min() >= episodes:
            break
    assert eps.min() >= episodes, "not every env finished %d episodes" % episodes


@pytest.mark.parametrize("setting,continuous", DOMAINS, ids=DOM_IDS)
@pytest.mark.parametrize("source", ["random", "traj"])
def test_twin_auto_reset(setting, continuous, source):
    n = 64
    s = _streams(n, setting, continuous, 200) if source == "traj" else None
    A, B = _batch(n, setting, continuous, s), _batch(n, setting, continuous, s, auto_reset=False)
    if source == "traj":
        A.set_trajectory_length(30)
        B.set_trajectory_length(30)
    _twin(A, B, 400)
    A.close(); B.close()


@pytest.mark.parametrize("lnes,shuffle", [("EV", False), ("EP", False), ("CP", False), ("FC", False), ("EMS", True), ("CP", True)])
def test_twin_auto_reset_lnes_shuffle(lnes, shuffle):
    n, setting = 32, 1
    s = _streams(n, setting, False, 200)
    A = _batch(n, setting, False, s, LNES=lnes, shuffle=shuffle)
    B = _batch(n, setting, False, s, LNES=lnes, shuffle=shuffle, auto_reset=False)
    _twin(A, B, 400)
    A.close(); B.close()


@pytest.mark.parametrize("name", NEEDS_ALIAS_D)
def test_twin_auto_reset_alias_cases(name):
    """the recorded trajectories on which the reference's object aliasing decides a real placement: env 0 follows the recorded env"""
    c = CASES[name]
    n = 8
    s = np.stack([case_stream(c, c["seed"], c["env"] + e, 400) for e in range(n)])
    pct_b200 = _pb()
    mk = lambda **kw: pct_b200.PctBatch(n, c["setting"], container_size=c["container"], item_set=c["items"], internal_node_holder=c["nb"],
                                        leaf_node_holder=c["nl"], obs_dtype=torch.float64, item_stream=s, env_id_base=c["env"], **kw)
    A, B = mk(), mk(auto_reset=False)
    _twin(A, B, max(400, c["steps"] + 40), episodes=1)
    A.close(); B.close()


VARIANTS = [("PCT_B200_WALK", "fork", False), ("PCT_B200_WALK", "fork", True), ("PCT_B200_K3", "block", False), ("PCT_B200_K3", "block", True),
            ("PCT_B200_GROUPS", "2", False), ("PCT_B200_OVERLAP", "0", False)]


@pytest.mark.parametrize("var,val,continuous", VARIANTS, ids=["%s=%s-%s" % (v, x, "c1" if c else "d1") for v, x, c in VARIANTS])
def test_twin_auto_reset_launch_variants(monkeypatch, var, val, continuous):
    """the reset path under the opt-in launch variants: fork-join walks, the block-per-env feasibility kernel, a step split over internal
    streams (the reset itself always runs the whole batch on the caller's stream), the non-overlapped step order"""
    monkeypatch.setenv(var, val)
    n, setting = 256, 1
    s = _streams(n, setting, continuous, 200)
    A, B = _batch(n, setting, continuous, s), _batch(n, setting, continuous, s, auto_reset=False)
    _twin(A, B, 400)
    A.close(); B.close()


# ---- 2. terminal observations and mid-episode resets against the oracle -----------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", DOMAINS, ids=DOM_IDS)
@pytest.mark.parametrize("mode", ["done", "mid"])
def test_oracle_terminal_and_mid_episode(setting, continuous, mode):
    """mode done: reset(mask=done) after every step, as gym callers do; mode mid: env_idx lists the finished envs plus random live ones,
    under a trajectory length (so a mid-episode reset jumps to the next trajectory).  The oracle env calls reset() for the same envs."""
    n, L, T = 16, 1200, 120
    traj = 40 if mode == "mid" else 0
    s = _streams(n, setting, continuous, L)
    B = _batch(n, setting, continuous, s, auto_reset=False)
    orc = [OracleContinuous(setting, stream=s[e]) if continuous else OracleDiscrete(setting, stream=s[e]) for e in range(n)]
    if traj:
        B.set_trajectory_length(traj)
        for o in orc:
            o.set_trajectory_length(traj)
    ref = [o.reset() for o in orc]
    obs = _np(B.reset())
    rng = np.random.RandomState(5)
    dones = mids = 0
    for t in range(T):
        assert np.array_equal(obs, np.stack(ref)), "observation before step %d" % t
        picks = [policy_pick(ref[e], B.nb, B.nl, PSEED, e, t) for e in range(n)]
        idx = torch.tensor([k for k, _ in picks], dtype=torch.int32, device=B.device)
        obs, rew, done, _ = [_np(x) for x in B.step(leaf_idx=idx)]
        for e in range(n):
            ref[e], r, d, _ = orc[e].step(picks[e][1])
            assert np.float32(r) == rew[e] and bool(d) == bool(done[e]), (e, t)
        assert np.array_equal(obs, np.stack(ref)), "observation after step %d (terminal ones included)" % t
        sel = done != 0
        dones += int(sel.sum())
        if mode == "mid":
            extra = (rng.rand(n) < 0.08) & ~sel
            mids += int(extra.sum())
            sel |= extra
        for e in np.nonzero(sel)[0]:
            ref[e] = orc[e].reset()
        if mode == "done":
            obs = _np(B.reset(mask=B._done))
        else:
            obs = _np(B.reset(env_idx=np.nonzero(sel)[0].astype(np.int32)))
    assert np.array_equal(obs, np.stack(ref))
    assert dones >= n and (mode == "done" or mids >= n)
    B.close()


# ---- 3. envs not listed; snapshots after a reset -------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", DOMAINS, ids=DOM_IDS)
def test_unlisted_envs_unchanged_and_snapshot_after_reset(setting, continuous):
    n = 48
    s = _streams(n, setting, continuous, 300)
    b = _batch(n, setting, continuous, s)
    b.reset()
    for t in range(6):
        b.step(leaf_idx=b.random_policy(PSEED, t))
    obs0, snap0 = _np(b._obs), _snap(b)
    listed = np.arange(1, n, 3).astype(np.int32)
    draws = [b.state(int(e))["draw_pos"] for e in listed]
    obs1 = _np(b.reset(env_idx=listed))
    snap1 = _snap(b)
    rest = np.setdiff1d(np.arange(n), listed)
    assert np.array_equal(obs1[rest], obs0[rest]) and np.array_equal(snap1[rest], snap0[rest])
    for e, d in zip(listed, draws):
        st = b.state(int(e))
        assert st["n_boxes"] == 0 and st["n_ems"] == 1 and st["flags"] == 0 and st["draw_pos"] == d + 1, e
        it = s[e, d % 300]
        assert list(st["next_box"]) == list(np.trunc(it[:3]) if not continuous else it[:3]), e
    # a snapshot taken after the reset restores into a fresh handle, which continues identically
    f = _batch(n, setting, continuous, s)
    f.reset()
    assert np.array_equal(_np(f.restore(b.snapshot())), obs1)
    for t in range(6, 30):
        idx = b.random_policy(PSEED, t)
        x, y = [_np(v) for v in b.step(leaf_idx=idx)], [_np(v) for v in f.step(leaf_idx=idx)]
        for u, v in zip(x, y):
            assert np.array_equal(u, v), t
    b.close(); f.close()


# ---- 4. delta rows ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", [(1, False), (2, False), (1, True)], ids=["d1", "d2", "c1"])
def test_delta_rows(setting, continuous, monkeypatch):
    """delta rows (X) = full rewrites (Y) = alternating buffers (Z: each reset gets another buffer than the step before it, each step
    the buffer of the reset before it); a reset env's internal rows are zero but row 0's valid flag"""
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
    row0 = np.zeros(9)
    row0[8] = 1
    for t in range(60):
        idx = X.random_policy(PSEED, t)
        ox, oy, oz = _np(X.step(leaf_idx=idx)[0]), _np(Y.step(leaf_idx=idx)[0]), _np(Z.step(leaf_idx=idx, out=bufs[t % 2])[0])
        assert np.array_equal(ox, oy) and np.array_equal(ox, oz), t
        sub = np.sort(rng.choice(n, 6, replace=False)).astype(np.int32)
        if t % 3 == 0:  # a mask instead of a list
            m = np.zeros(n, dtype=bool)
            m[sub] = True
            kw = dict(mask=torch.as_tensor(m, device=X.device))
        else:
            kw = dict(env_idx=sub)
        ox, oy, oz = _np(X.reset(**kw)), _np(Y.reset(**kw)), _np(Z.reset(out=bufs[(t + 1) % 2], **kw))
        assert np.array_equal(ox, oy) and np.array_equal(ox, oz), t
        internal = ox.reshape(n, -1, 9)[sub, :X.nb]
        assert np.array_equal(internal[:, 0], np.tile(row0, (len(sub), 1))) and not internal[:, 1:].any(), t
    X.close(); Y.close(); Z.close()


# ---- 5. interaction with set_items and LSAH -----------------------------------------------------------------------------------
@pytest.mark.parametrize("continuous", [False, True], ids=["d1", "c1"])
def test_reset_discards_a_set_item(continuous):
    n = 8
    s = _streams(n, 1, continuous, 100)
    A, B = _batch(n, 1, continuous, s), _batch(n, 1, continuous, s)
    A.reset(); B.reset()
    for t in range(4):
        idx = A.random_policy(PSEED, t)
        A.step(leaf_idx=idx); B.step(leaf_idx=idx)
    B.set_items(torch.tensor([SENTINEL, SENTINEL], dtype=torch.float64), env_idx=[2, 5])
    assert list(_np(B.preview_items(1))[2, 0, :3]) == list(SENTINEL)
    oa, ob = _np(A.reset(env_idx=[2, 5, 6])), _np(B.reset(env_idx=[2, 5, 6]))
    assert np.array_equal(oa, ob), "the reset drew the same fresh item with or without set_items"
    assert np.array_equal(_snap(A), _snap(B))
    A.close(); B.close()


@pytest.mark.parametrize("continuous", [False, True], ids=["discrete", "continuous"])
def test_lsah_after_mid_episode_reset(continuous):
    """LSAH's footprint restarts with the episode: after a mid-episode reset at draw d, an env follows a fresh batch whose stream starts at d"""
    n, L = 32, 400
    s = _streams(n, 1, continuous, L)
    b = _batch(n, 1, continuous, s)
    b.reset()
    for _ in range(5):
        b.step(actions=b.heuristic_actions("LSAH"))
    listed = np.arange(0, n, 2).astype(np.int32)
    d = np.array([b.state(e)["draw_pos"] for e in range(n)])
    b.reset(env_idx=listed)
    f = _batch(n, 1, continuous, np.stack([np.roll(s[e], -d[e], axis=0) for e in range(n)]))
    fo = _np(f.reset())
    assert np.array_equal(_np(b._obs)[listed], fo[listed])
    dones = 0
    for t in range(60):
        rb, rf = b.heuristic_actions("LSAH").clone(), f.heuristic_actions("LSAH").clone()
        assert np.array_equal(_np(rb)[listed], _np(rf)[listed]), "LSAH rows differ at step %d" % t
        x, y = [_np(v) for v in b.step(actions=rb)], [_np(v) for v in f.step(actions=rf)]
        for u, v in zip(x, y):
            assert np.array_equal(u[listed], v[listed]), t
        dones += int(x[2][listed].sum())
    assert dones > 0
    b.close(); f.close()


# ---- 6. graph capture ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", [(1, False), (1, True)], ids=["d1", "c1"])
def test_graph_capture(setting, continuous):
    """random policy -> step -> reset(mask=done) on a batch without auto-reset, captured once, replayed; against the same loop run eagerly"""
    n = 64
    s = _streams(n, setting, continuous, 300)
    G, E = _batch(n, setting, continuous, s, auto_reset=False), _batch(n, setting, continuous, s, auto_reset=False)
    info = {}
    for b in (G, E):
        b.reset()
        info[b] = torch.zeros((n, 8), dtype=torch.int32, device=b.device)

    def body(b):
        _, rew, done, _ = b.step(leaf_idx=b.random_policy(PSEED, 0))
        obs = b.reset(mask=done, info=info[b])
        return obs, rew, done, info[b]

    for b in (G, E):  # warm-up outside the capture
        body(b)
    st = torch.cuda.Stream(device=G.device)
    st.wait_stream(torch.cuda.current_stream(G.device))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(st):
        with torch.cuda.graph(g, stream=st):
            out = body(G)
    torch.cuda.current_stream(G.device).wait_stream(st)
    dones = 0
    for t in range(40):
        g.replay()
        ref = body(E)
        torch.cuda.synchronize()
        for u, v in zip(out, ref):
            assert torch.equal(u, v), t
        dones += int(ref[2].sum())
    assert dones > 0, "the replays exercised no reset"
    G.close(); E.close()


# ---- 7. errors and edge cases ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("continuous", [False, True], ids=["d1", "c1"])
def test_errors_and_edge_cases(continuous):
    pct_b200 = _pb()
    n = 8
    b = _batch(n, 1, continuous, _streams(n, 1, continuous, 100), auto_reset=False)
    L, h = b.L, b.h
    idx = torch.arange(n, dtype=torch.int32, device=b.device)
    mask = torch.ones((n,), dtype=torch.uint8, device=b.device)
    ptr = lambda t: C.c_void_p(t.data_ptr())
    assert L.pct_reset_envs(h, ptr(idx), 2, None, ptr(b._obs), None, None) == -4  # PCT_ERR_STATE before pct_reset
    assert L.pct_reset_envs(h, None, n, ptr(mask), ptr(b._obs), None, None) == -4
    with pytest.raises(pct_b200.PctError):
        b.reset(env_idx=[0])
    b.reset()
    assert L.pct_reset_envs(h, ptr(idx), n, ptr(mask), ptr(b._obs), None, None) == -1  # both
    assert L.pct_reset_envs(h, None, n, None, ptr(b._obs), None, None) == -1           # neither
    assert L.pct_reset_envs(h, ptr(idx), -1, None, ptr(b._obs), None, None) == -1
    assert L.pct_reset_envs(h, None, n - 1, ptr(mask), ptr(b._obs), None, None) == -1  # mask length
    assert L.pct_reset_envs(h, None, n, ptr(mask), None, None, None) == -1             # no observation buffer
    for kw in (dict(env_idx=[0], mask=mask), dict(mask=mask[:-1]), dict(mask=mask.float()), dict(env_idx=[[0]]),
               dict(env_idx=[0], info=torch.zeros((n, 7), dtype=torch.int32, device=b.device)), dict(info=torch.zeros((n, 8), dtype=torch.int32))):
        with pytest.raises(pct_b200.PctError):
            b.reset(**kw)
    for t in range(3):
        b.step(leaf_idx=b.random_policy(PSEED, t))
    obs0, snap0 = _np(b._obs), _snap(b)
    launches = b.kernel_launches
    assert L.pct_reset_envs(h, ptr(idx), 0, None, ptr(b._obs), None, None) == 0       # n == 0: no-op
    b.reset(env_idx=[])
    assert b.kernel_launches == launches, "n == 0 enqueued work"
    b.reset(env_idx=[-1, n, 1 << 20])                                                  # out-of-range indices are skipped
    assert np.array_equal(_snap(b), snap0) and np.array_equal(_np(b._obs), obs0)
    b.reset(mask=torch.zeros((n,), dtype=torch.bool, device=b.device))                 # an all-zero mask leaves every env unchanged
    assert np.array_equal(_snap(b), snap0) and np.array_equal(_np(b._obs), obs0)
    b.reset(mask=np.arange(n) % 2 == 0)                                                # a host mask is copied to the device
    assert [b.state(e)["n_boxes"] for e in range(0, n, 2)] == [0] * (n // 2)
    assert np.array_equal(_snap(b)[1::2], snap0[1::2])
    b.close()
