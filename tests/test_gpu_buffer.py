"""GPU: buffered packing (pct_set_buffer / pct_buffer_*, PctBatch(..., buffer=B); DESIGN.md section 18).

A buffered step is defined by composition: pct_set_items(item j) followed by pct_step(leaf l) on a plain handle.  So a buffered batch is
checked against a plain twin driven by set_items(whole_batch=False) + step(env_idx=...) with the same choices, and its observation against
expand_items of its own buffered items.  With B = 1 it must be the plain step, bit for bit.  Its items follow the env's draw sequence, and the
chosen items replay as a plain stream on the oracle.
"""
import ctypes as C
import os
import types

import numpy as np
import pytest

torch = pytest.importorskip("torch")
from harness import ITEM_SET, case_stream, cont_case_stream, load_capacity_cases, make_stream  # noqa: E402
from pct_oracle import OracleContinuous, OracleDiscrete, make_continuous_stream  # noqa: E402

pytestmark = pytest.mark.gpu
PSEED = 97
INVALID, STATE = -1, -4  # PCT_ERR_INVALID, PCT_ERR_STATE
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "baseline", "_ref")


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
    kw.setdefault("obs_dtype", torch.float64)
    if continuous:
        if stream is not None:
            return pct_b200.PctBatch(n, setting, container_size=(1.0, 1.0, 1.0), continuous=True, item_stream=stream, size_minimum=0.1, **kw)
        return pct_b200.PctBatch(n, setting, container_size=(1.0, 1.0, 1.0), continuous=True, sample_from_distribution=True, seed=1234, **kw)
    if stream is not None:
        return pct_b200.PctBatch(n, setting, item_set=ITEM_SET, item_stream=stream, **kw)
    return pct_b200.PctBatch(n, setting, item_set=ITEM_SET, seed=1234, **kw)


def _blocks(P, obs):
    """(internal rows (n, NB, 9), leaf blocks (n, B, NL, 9), item rows (n, B, 9)) of a buffered observation"""
    n, nb, nl, B = obs.shape[0], P.nb, P.nl, P.buffer
    return obs[:, :nb * 9].reshape(n, nb, 9), obs[:, nb * 9:(nb + B * nl) * 9].reshape(n, B, nl, 9), obs[:, (nb + B * nl) * 9:].reshape(n, B, 9)


def _item_rows(items, dtype):
    """the item rows pct_set_items writes for (n, B, 4) items: [density, 0, 0, sorted sizes, 0, 0, 1]"""
    n, B = items.shape[:2]
    r = np.zeros((n, B, 9))
    r[:, :, 0] = items[:, :, 3]
    r[:, :, 3:6] = np.sort(items[:, :, :3], axis=2)
    r[:, :, 8] = 1
    return r.astype(dtype)


def _bytes_equal(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


# ---- 1. B = 1 is pct_step ----------------------------------------------------------------------------------------------------------------
B1_CASES = [(s, c, src, {}) for c in (False, True) for s in (1, 2, 3) for src in ("random", "stream")]
B1_CASES += [(1, False, "stream", dict(traj=7)), (3, True, "stream", dict(traj=9))]
B1_CASES += [(s, False, "random", dict(LNES=l)) for s, l in ((1, "EV"), (2, "EP"), (1, "CP"), (2, "FC"))]
B1_CASES += [(1, False, "random", dict(shuffle=True)), (2, False, "stream", dict(shuffle=True, LNES="EP")), (1, True, "random", dict(shuffle=True)),
             (1, False, "random", dict(obs_dtype=torch.float32)), (3, True, "stream", dict(obs_dtype=torch.float32))]


def _b1_id(c):
    s, cont, src, kw = c
    return "%s%d-%s%s" % ("c" if cont else "d", s, src, "".join("-%s=%s" % (k, str(v).replace("torch.", "")) for k, v in sorted(kw.items())))


@pytest.mark.parametrize("setting,continuous,source,kw", B1_CASES, ids=[_b1_id(c) for c in B1_CASES])
def test_b1_is_pct_step(setting, continuous, source, kw):
    """a buffered batch with B = 1 equals a plain batch of the same configuration at every step: observation, reward, done and record"""
    kw = dict(kw)
    traj = kw.pop("traj", 0)
    n, T = 64, 160
    st = _streams(n, setting, continuous, 400) if source == "stream" else None
    P, Q = _batch(n, setting, continuous, st, buffer=1, **kw), _batch(n, setting, continuous, st, **kw)
    assert P.obs_len == Q.obs_len
    if traj:
        P.set_trajectory_length(traj); Q.set_trajectory_length(traj)
    P.reset(); Q.reset()
    assert _bytes_equal(_np(P._obs), _np(Q._obs))
    t_dev = torch.zeros((), dtype=torch.int64, device=P.device)
    done_total = 0
    for t in range(T):
        a = P.random_policy_dev(PSEED, t_dev).clone()
        b = Q.random_policy_dev(PSEED, t_dev) if not continuous else Q.random_policy(PSEED, t)
        assert torch.equal(a, b), t
        if t % 11 == 5:
            a[::7] = -1  # out of range: the zero action of a plain step (placement at the origin)
            a[3::13] = 10 ** 6
        op, rp, dp, ip = P.step(leaf_idx=a)
        oq, rq, dq, iq = Q.step(leaf_idx=a)
        assert _bytes_equal(_np(op), _np(oq)), "observation at step %d" % t
        assert torch.equal(rp, rq) and torch.equal(dp, dq) and torch.equal(ip, iq), "reward / done / record at step %d" % t
        done_total += int(dp.sum())
        t_dev += 1
    assert done_total > n
    P.close(); Q.close()


# ---- 2. the composition twin -------------------------------------------------------------------------------------------------------------
def _twin_run(P, Q, episodes=2, max_steps=600, bad_every=0, strict_flags=True):
    """steps buffered P with random valid flat indices and plain twin Q with set_items_only(item j) + step_envs(leaf l), comparing them
    (and P's leaf blocks with expand_items of P's own buffered items) after every step; -> steps taken.  episodes = 0: max_steps steps.
    strict_flags: the records' flags are equal; otherwise (capacity cases, where the twin's own expansions raise flags of items P never
    expands) P's flags hold every slot expansion's and BAD_ACTION agrees"""
    n, B, nl = P.n_envs, P.buffer, P.nl
    ar = torch.arange(n, device=P.device)
    t_dev = torch.zeros((), dtype=torch.int64, device=P.device)
    eps = np.zeros(n, dtype=int)
    obs = P._obs.clone()
    shuffle = bool(P.cfg.shuffle)
    t = 0
    while t < max_steps:
        items = P.buffer_items()
        _, blocks, irows = _blocks(P, obs)
        # P's leaf blocks are expand_items of its buffered items on P itself (same shuffle keys), its item rows those of set_items
        lv, li = P.expand_items(items[:, :, :3], density=items[:, :, 3].contiguous())
        assert _bytes_equal(_np(lv), _np(blocks)), "leaf blocks at step %d" % t
        assert _bytes_equal(_item_rows(_np(items), _np(irows).dtype), _np(irows)), "item rows at step %d" % t
        flat = P.random_policy_dev(PSEED, t_dev).clone()
        if bad_every and t % bad_every == 3:
            flat[::5] = -3
            flat[2::9] = B * nl + 4
            flat[4::11] = (B - 1) * nl + nl - 1  # the last leaf of the last slot: usually past its leaf count
        f = flat.long()
        inside = (f >= 0) & (f < B * nl)
        j = torch.where(inside, f // nl, torch.zeros_like(f))
        leaf = torch.where(inside, f % nl, torch.full_like(f, -1)).to(torch.int32)
        chosen = items[ar, j]
        oq = Q.set_items(chosen[:, :3], density=chosen[:, 3].contiguous(), whole_batch=False).clone()
        if not shuffle:  # the twin's leaf rows for the chosen item are P's leaf block j
            assert _bytes_equal(_np(oq[:, P.nb * 9:(P.nb + nl) * 9].reshape(n, nl, 9)), _np(blocks[ar, j])), "twin leaf rows at step %d" % t
        obs, r, d, info = P.step(leaf_idx=flat)
        obs = obs.clone()
        if shuffle:  # the twin's list is shuffled with its own draw position: it gets the chosen leaf row (zeros: the zero action) instead
            lrow = torch.where((leaf >= 0)[:, None], blocks[ar, j, leaf.clamp(min=0).long()], torch.zeros_like(blocks[:, 0, 0]))
            o2, r2, d2, i2 = Q.step(actions=lrow.contiguous(), env_idx=ar)
        else:
            o2, r2, d2, i2 = Q.step(leaf_idx=leaf, env_idx=ar)
        assert torch.equal(r, r2) and torch.equal(d, d2), "reward / done at step %d" % t
        ip, iq = _np(info), _np(i2)
        assert np.array_equal(ip[:, [0, 2, 3, 4, 7]], iq[:, [0, 2, 3, 4, 7]]), "record at step %d" % t
        # flags: the twin's are its own expansion's too; P's are the apply kernel's and every slot's expansion's
        items = P.buffer_items()
        lv, li = P.expand_items(items[:, :, :3], density=items[:, :, 3].contiguous())
        li = _np(li)
        assert np.array_equal(ip[:, 5], li[:, :, 5].sum(1)) and np.array_equal(ip[:, 6], li[:, :, 6].sum(1)), "summed counts at step %d" % t
        orli = np.bitwise_or.reduce(li[:, :, 1], axis=1)
        assert np.array_equal(ip[:, 1] | orli, ip[:, 1]) and np.array_equal(ip[:, 1] & 2, iq[:, 1] & 2), "flags at step %d" % t
        if strict_flags:
            assert np.array_equal(ip[:, 1], iq[:, 1]), "flags at step %d" % t
        assert _bytes_equal(_np(obs[:, :P.nb * 9]), _np(o2[:, :Q.nb * 9])), "internal rows at step %d" % t
        eps += _np(d).astype(int)
        t += 1
        t_dev += 1
        if episodes and eps.min() >= episodes:
            break
    assert eps.min() >= episodes, "every env finishes %d episodes within %d steps" % (episodes, max_steps)
    # the read-only calls see the same placed boxes
    if not P.continuous:
        assert torch.equal(P.height_maps(), Q.height_maps())
    q = torch.as_tensor(np.array([[[2, 2, 2, 0, 0], [3, 1, 2, 4, 5], [1, 1, 1, 9, 9]]] * n, dtype=np.float64))
    if P.continuous:
        q = q / 10.0
    den = torch.ones(q.shape[:2], dtype=torch.float64)
    fp, rp_ = P.query_placements(q, density=den)
    fq, rq_ = Q.query_placements(q, density=den)
    assert torch.equal(fp, fq) and torch.equal(rp_, rq_)
    its = P.buffer_items()
    assert _bytes_equal(_np(P.expand_items(its[:, :, :3], density=its[:, :, 3].contiguous())[0]),
                        _np(Q.expand_items(its[:, :, :3], density=its[:, :, 3].contiguous())[0])) or shuffle
    return t


TWIN = [(s, c, B) for B in (3, 5) for s, c in ((1, False), (2, False), (3, False), (1, True), (3, True))]


@pytest.mark.parametrize("setting,continuous,B", TWIN, ids=["%s%d-B%d" % ("c" if c else "d", s, B) for s, c, B in TWIN])
def test_composition_twin(setting, continuous, B):
    n = 48
    st = _streams(n, setting, continuous, 600, seed=5)
    own = _streams(n, setting, continuous, 600, seed=6)
    P, Q = _batch(n, setting, continuous, st, buffer=B), _batch(n, setting, continuous, own)
    P.reset(); Q.reset()
    _twin_run(P, Q, bad_every=7)
    P.close(); Q.close()


@pytest.mark.parametrize("kw", [dict(LNES="EV"), dict(LNES="CP"), dict(shuffle=True), dict(shuffle=True, LNES="FC")], ids=["EV", "CP", "shuffle", "shuffle-FC"])
def test_composition_twin_lnes_shuffle(kw):
    n, B = 48, 3
    P, Q = _batch(n, 1, False, buffer=B, **kw), _batch(n, 1, False, **kw)
    P.reset(); Q.reset()
    _twin_run(P, Q)
    P.close(); Q.close()


def _mild_streams(c, n):
    if c["domain"] == "continuous":
        return [cont_case_stream(dict(c, lo=0.1, hi=0.5), 500 + e, 0, len(c["stream"])) for e in range(n)]
    mild = [(a, b, h) for a in (5, 7) for b in (5, 8) for h in (4, 6)]
    return [case_stream(dict(c, items=mild), 500 + e, 0, len(c["stream"])) for e in range(n)]


def test_composition_twin_capacity_cases():
    """the capacity cases' configurations and streams (tests/golden/capacity_cases.npz) through buffered B = 3 envs and their twins"""
    cases = load_capacity_cases()
    pct_b200 = _pb()
    for name in sorted(cases):
        c = cases[name]
        s = np.stack([c["stream"]] * 2 + _mild_streams(c, 2))
        n = len(s)
        mk = lambda **kw: pct_b200.PctBatch(n, c["setting"], container_size=c["container"], continuous=c["domain"] == "continuous",
                                            item_set=None if c["domain"] == "continuous" else c["items"], internal_node_holder=c["nb"],
                                            leaf_node_holder=c["nl"], obs_dtype=torch.float64, item_stream=s, size_minimum=c["size_minimum"],
                                            LNES=c["lnes"], **kw)
        P, Q = mk(buffer=3), mk()
        P.reset(); Q.reset()
        _twin_run(P, Q, episodes=0, max_steps=min(int(c["steps"]) + 40, len(c["stream"]) - 40), strict_flags=False)
        P.close(); Q.close()


# ---- 3. item order ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous,traj", [(1, False, 0), (3, False, 0), (1, False, 9), (2, True, 0), (3, True, 8)],
                         ids=["d1", "d3", "d1-traj", "c2", "c3-traj"])
def test_items_follow_the_stream(setting, continuous, traj):
    """buffer_items() against the draw sequence computed on the host: slot j takes the draw the step consumed; a finished episode
    refills slots 0 .. B-1 with the next B draws (under a trajectory length: the first B items of the next trajectory)"""
    n, B, L = 32, 4, 2000
    st = _streams(n, setting, continuous, L, seed=3)
    P = _batch(n, setting, continuous, st, buffer=B)
    if traj:
        P.set_trajectory_length(traj)
    P.reset()
    pos = np.full(n, B)
    buf = st[:, :B].copy()
    t_dev = torch.zeros((), dtype=torch.int64, device=P.device)
    eps = np.zeros(n, dtype=int)
    for t in range(400):
        assert np.array_equal(_np(P.buffer_items()), buf), t
        flat = P.random_policy_dev(PSEED, t_dev)
        f = _np(flat)
        _, _, d, _ = P.step(leaf_idx=flat)
        d = _np(d)
        for e in range(n):
            if d[e]:
                p0 = pos[e]
                if traj and p0 % traj:
                    p0 += traj - p0 % traj
                buf[e] = st[e, [(p0 + k) % L for k in range(B)]]
                pos[e] = p0 + B
            else:
                buf[e, f[e] // P.nl] = st[e, pos[e] % L]
                pos[e] += 1
        eps += d.astype(int)
        t_dev += 1
    assert eps.min() >= 2
    P.close()


@pytest.mark.parametrize("setting,continuous", [(1, False), (3, False), (1, True), (3, True)], ids=["d1", "d3", "c1", "c3"])
def test_items_random_source(setting, continuous):
    """the random sources (item set / continuous sampler): after a reset slot j holds draw j, what preview_items(B) shows on a plain batch"""
    n, B = 64, 5
    P, Q = _batch(n, setting, continuous, buffer=B), _batch(n, setting, continuous)
    P.reset(); Q.reset()
    assert np.array_equal(_np(P.buffer_items()), _np(Q.preview_items(B)))
    idx = torch.as_tensor(np.array([3, -1, 70, 0], dtype=np.int32))
    got = _np(P.buffer_items(env_idx=idx))
    assert np.array_equal(got[0], _np(Q.preview_items(B))[3]) and not got[1].any() and not got[2].any()
    P.close(); Q.close()


# ---- 4. the oracle -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", [(1, False), (2, False), (3, False), (1, True), (3, True)], ids=["d1", "d2", "d3", "c1", "c3"])
def test_chosen_items_replay_on_the_oracle(setting, continuous):
    """the items a B = 3 policy chose, replayed as a plain stream on the oracle with the chosen leaf rows as actions: the internal rows,
    the chosen item's leaf rows, rewards and dones equal the buffered batch's"""
    n, B = 64, 3
    st = _streams(n, setting, continuous, 600, seed=21)
    P = _batch(n, setting, continuous, st, buffer=B)
    obs = P.reset().clone()
    nb, nl = P.nb, P.nl
    t_dev = torch.zeros((), dtype=torch.int64, device=P.device)
    chosen, blocks, flats, rews, dones, obs_hist = [], [], [], [], [], []
    eps = np.zeros(n, dtype=int)
    for t in range(400):
        items = _np(P.buffer_items())
        flat = _np(P.random_policy_dev(PSEED, t_dev))
        j = flat // nl
        chosen.append(items[np.arange(n), j]); flats.append(flat); obs_hist.append(_np(obs))
        o, r, d, _ = P.step(leaf_idx=torch.as_tensor(flat).to(P.device))
        obs = o.clone()
        rews.append(_np(r)); dones.append(_np(d))
        eps += dones[-1].astype(int)
        t_dev += 1
        if eps.min() >= 2:
            break
    assert eps.min() >= 2
    T = len(chosen)
    seq = np.concatenate([np.stack(chosen, 1), np.tile(st[:, :1], (1, 2, 1))], 1)
    for e in range(0, n, 8):
        o = OracleContinuous(setting, stream=seq[e]) if continuous else OracleDiscrete(setting, stream=seq[e])
        ob = o.reset()
        for t in range(T):
            ins, blk, _ = _blocks(P, obs_hist[t][e][None])
            j, l = flats[t][e] // nl, flats[t][e] % nl
            assert np.array_equal(ob[:nb * 9], ins[0].reshape(-1)), (e, t)
            assert np.array_equal(ob[nb * 9:(nb + nl) * 9].reshape(nl, 9), blk[0, j]), (e, t)
            ob, r, d, _ = o.step(blk[0, j, l].astype(np.float64))
            assert np.float32(r) == rews[t][e] and bool(d) == bool(dones[t][e]), (e, t)
            if d:
                ob = o.reset()
    P.close()


# ---- 5. refused calls and argument errors ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("continuous", [False, True], ids=["d", "c"])
def test_refused_calls_and_errors(continuous):
    pct_b200 = _pb()
    L = pct_b200._lib.lib()
    n, B = 8, 3
    P = _batch(n, 1, continuous, buffer=B)
    h = P.h
    vp = lambda t: C.c_void_p(t.data_ptr())
    obs = torch.zeros((n, P.obs_len), dtype=torch.float64, device=P.device)
    idx = torch.zeros(n, dtype=torch.int32, device=P.device)
    t_dev = torch.zeros((), dtype=torch.int64, device=P.device)
    out = torch.zeros((n, B, 4), dtype=torch.float64, device=P.device)
    # before the first reset
    assert L.pct_buffer_step(h, vp(idx), vp(obs), vp(P._rew), vp(P._done), None, None) == STATE
    assert L.pct_buffer_items(h, None, n, vp(out), None) == STATE
    assert L.pct_buffer_policy_random(h, vp(idx), 1, vp(t_dev), None) == STATE
    assert L.pct_set_buffer(h, 0) == INVALID and L.pct_set_buffer(h, 17) == INVALID
    P.reset()
    assert L.pct_set_buffer(h, 2) == STATE  # after a reset
    assert L.pct_buffer_step(h, None, vp(obs), vp(P._rew), vp(P._done), None, None) == INVALID
    assert L.pct_buffer_items(h, None, -1, vp(out), None) == INVALID
    assert L.pct_buffer_obs_len(h) == (P.nb + B * P.nl + B) * 9 == P.obs_len
    dims = torch.ones((n, 3), dtype=torch.float64 if continuous else torch.int32, device=P.device)
    plain_obs = torch.zeros((n, (P.nb + P.nl + 1) * 9), dtype=torch.float64, device=P.device)
    refused = [
        lambda: L.pct_reset(h, vp(plain_obs), None),
        lambda: L.pct_step(h, None, 0, vp(idx), vp(plain_obs), vp(P._rew), vp(P._done), None, None),
        lambda: L.pct_step_envs(h, vp(idx), 1, None, None, 0, vp(idx), vp(plain_obs), vp(P._rew), vp(P._done), None, None),
        lambda: L.pct_reset_host(h, plain_obs.cpu().numpy().ctypes.data),
        lambda: L.pct_step_host(h, None, 0, np.zeros(n, np.int32).ctypes.data, np.zeros((n, 9 * 200)).ctypes.data, np.zeros(n, np.float32).ctypes.data,
                                np.zeros(n, np.uint8).ctypes.data, None),
        lambda: L.pct_set_items(h, None, n, vp(dims), None, vp(plain_obs), None, None),
        lambda: L.pct_set_items_only(h, None, n, vp(dims), None, vp(plain_obs), None, None),
        lambda: L.pct_reset_envs(h, vp(idx), 1, None, vp(plain_obs), None, None),
        lambda: L.pct_reset_envs_only(h, vp(idx), 1, None, vp(plain_obs), None, None),
        lambda: L.pct_preview_items(h, None, n, 2, vp(out), None),
        lambda: L.pct_heuristic_actions(h, 0, vp(plain_obs), 0, 0, None),
        lambda: L.pct_heuristic_actions_f64(h, 0, vp(plain_obs), None),
        lambda: L.pct_snapshot(h, None, 1, vp(torch.zeros(P.snapshot_bytes, dtype=torch.uint8, device=P.device)), None),
        lambda: L.pct_restore(h, None, None, 1, vp(torch.zeros(P.snapshot_bytes, dtype=torch.uint8, device=P.device)), None, None),
    ]
    for i, f in enumerate(refused):
        assert f() == STATE, i
    for f in (lambda: P.set_items(_np(dims)), lambda: P.preview_items(2), lambda: P.snapshot(), lambda: P.heuristic_actions("LSAH"),
              lambda: P.reset(env_idx=[0]), lambda: P.step(leaf_idx=idx, env_idx=[0])):
        with pytest.raises(pct_b200.PctError):
            f()
    torch.cuda.synchronize()
    # the read-only calls work
    P.expand_items(_np(dims)[:, None, :].repeat(2, 1))
    P.query_placements(np.ones((n, 1, 5)))
    P.state(0)
    P.support_graph(0)
    P.close()
    Q = _batch(n, 1, continuous)
    assert L.pct_buffer_reset(Q.h, vp(obs), None, None) == STATE  # not a buffered handle
    assert L.pct_buffer_obs_len(Q.h) == 0
    with pytest.raises(pct_b200.PctError):
        Q.buffer_items()
    Q.close()
    with pytest.raises(pct_b200.PctError):
        _batch(n, 1, continuous, buffer=2, auto_reset=False)


# ---- 6. CUDA graphs ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", [(1, False), (2, False), (1, True)], ids=["d1", "d2", "c1"])
def test_graph_capture(setting, continuous):
    """a captured policy_random -> buffer_step loop and GraphedRollout with the built-in policy equal the eager loop"""
    pct_b200 = _pb()
    n, B, T = 64, 3, 6
    st = _streams(n, setting, continuous, 500, seed=8)
    G, E = _batch(n, setting, continuous, st, buffer=B), _batch(n, setting, continuous, st, buffer=B)
    G.reset(); E.reset()
    t_g = torch.zeros((), dtype=torch.int64, device=G.device)
    out_g = torch.zeros((T, n, G.obs_len), dtype=torch.float64, device=G.device)
    rew_g = torch.zeros((T, n), dtype=torch.float32, device=G.device)
    idx = torch.zeros(n, dtype=torch.int32, device=G.device)

    def body():
        for t in range(T):
            G.random_policy_dev(PSEED, t_g, out=idx)
            _, r, _, _ = G.step(leaf_idx=idx, out=out_g[t])
            rew_g[t].copy_(r)
            t_g.add_(1)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        body()
    t_e = torch.zeros((), dtype=torch.int64, device=E.device)
    for rep in range(4):
        g.replay()
        torch.cuda.synchronize()
        for t in range(T):
            flat = E.random_policy_dev(PSEED, t_e)
            o, r, _, _ = E.step(leaf_idx=flat)
            assert torch.equal(o, out_g[t]) and torch.equal(r, rew_g[t]), (rep, t)
            t_e += 1
    G.close(); E.close()
    R, E = _batch(n, setting, continuous, st, buffer=B), _batch(n, setting, continuous, st, buffer=B)
    roll = pct_b200.GraphedRollout(R, 5, policy_seed=PSEED)
    E.reset()
    t_e = torch.zeros((), dtype=torch.int64, device=E.device)
    for rep in range(3):
        obs, rew, done, act = roll.run()
        torch.cuda.synchronize()
        for t in range(5):
            assert torch.equal(obs[t], E._obs), (rep, t)
            flat = E.random_policy_dev(PSEED, t_e)
            assert torch.equal(flat, act[t])
            _, r, d, _ = E.step(leaf_idx=flat)
            assert torch.equal(r, rew[t]) and torch.equal(d, done[t])
            t_e += 1
    R.close(); E.close()


# ---- 7. the reference's network ----------------------------------------------------------------------------------------------------------
@pytest.mark.skipif(not os.path.isfile(os.path.join(REF, "attention_model.py")), reason="no copy of the reference's policy network under baseline/_ref")
def test_drl_gat_buffered_rollout_replays_on_the_oracle():
    """DRL_GAT built for B * NL leaves, through buffered_drl_gat, runs a captured buffered rollout; its sampled flat indices replay on the oracle"""
    pct_b200 = _pb()
    from pct_b200 import compat
    n, T, B, setting = 32, 6, 3, 1
    dev = torch.device("cuda", 0)
    model, tools = compat.load_policy_modules(REF, strip_asserts=True)
    args = types.SimpleNamespace(embedding_size=64, hidden_size=128, gat_layer_num=1, internal_node_holder=80, internal_node_length=6,
                                 leaf_node_holder=B * 50)
    torch.manual_seed(7)
    net = pct_b200.buffered_drl_gat(model.DRL_GAT(args).to(dev), B, 80, 50)
    st = _streams(n, setting, False, 600, seed=31)
    P = _batch(n, setting, False, st, buffer=B, obs_dtype=torch.float32)
    roll = pct_b200.GraphedRollout(P, T, policy=pct_b200.drl_gat_policy(net, tools, 80, B * 50, 0.1))
    acts, obs_hist, rews, dones = [], [], [], []
    with torch.no_grad():
        for r in range(3):
            obs, rew, done, act = roll.run()
            torch.cuda.synchronize()
            for t in range(T):
                obs_hist.append(_np(obs[t])); acts.append(_np(act[t])); rews.append(_np(rew[t])); dones.append(_np(done[t]))
    assert roll.graph is not None
    nb, nl = 80, 50
    # the sampled index is a valid flat leaf (when there is one) and the choices replay on the oracle
    for t in range(len(acts)):
        _, blk, _ = _blocks(P, obs_hist[t])
        f = acts[t]
        has = blk[:, :, :, 8].sum((1, 2)) > 0
        assert (blk[np.arange(n), f // nl, f % nl, 8] == 1)[has].all()
    for e in range(0, n, 4):
        # chosen item of step t: the item row of slot j at step t, as drawn = the stream's items in buffer order (host tracking)
        buf, pos = st[e, :B].copy(), B
        items = []
        for t in range(len(acts)):
            j = acts[t][e] // nl
            items.append(buf[j].copy())
            if dones[t][e]:
                buf, pos = st[e, pos:pos + B].copy(), pos + B
            else:
                buf[j] = st[e, pos]
                pos += 1
        seq = np.concatenate([np.stack(items), st[e, :2]])
        o = OracleDiscrete(setting, stream=seq)
        ob = o.reset()
        for t in range(len(acts)):
            ins, blk, _ = _blocks(P, obs_hist[t][e][None])
            j, l = acts[t][e] // nl, acts[t][e] % nl
            assert np.array_equal(ob[:nb * 9].astype(np.float32), ins[0].reshape(-1)), (e, t)
            ob, rr, d, _ = o.step(blk[0, j, l].astype(np.float64))
            assert np.float32(rr) == rews[t][e] and bool(d) == bool(dones[t][e]), (e, t)
            if d:
                ob = o.reset()
    P.close()
