"""GPU: selected envs and snapshots of buffered batches (pct_buffer_step_envs, pct_buffer_reset_envs, pct_buffer_snapshot / _restore;
PctBatch.buffer_*; DESIGN.md section 20).

A buffered batch driven by random selections is compared with a twin that takes full buffered steps: after its t-th selected step, an env
equals the twin's env after full step t, bit for bit (rows, reward, done, record, buffered items, buffered snapshot record), and envs not
selected are not written.  With B = 1 the calls are the plain selected calls.  Resets of chosen envs equal pct_buffer_reset's.  Records
round-trip, fan out and refuse other configurations; the lookahead example of tests/buffer_search.py commits what a direct step commits.
"""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
from harness import CASES, ITEM_SET, NEEDS_ALIAS_D, case_stream, load_capacity_cases, make_stream  # noqa: E402
from pct_oracle import OracleContinuous, OracleDiscrete, make_continuous_stream, rnd_u64  # noqa: E402
import buffer_search  # noqa: E402

pytestmark = pytest.mark.gpu
SENT_REW, SENT_DONE, SENT_INFO = -7.0, 0xAB, 0x5A5A5A5A
INVALID, STATE = -1, -4  # PCT_ERR_INVALID, PCT_ERR_STATE
BAD_SNAPSHOT = 128
PSEED = 97
SIZES = ["0", "1", "1%", "50%", "all"]


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


def _snap(P, env_idx=None):
    n = P.n_envs if env_idx is None else len(env_idx)
    out = torch.zeros((n, P.buffer_snapshot_bytes), dtype=torch.uint8, device=P.device)  # zero-filled: only live prefixes are written
    return _np(P.buffer_snapshot(env_idx=env_idx, out=out))


def _valid(P, obs):
    """(n, B * NL) valid flat leaf indices of buffered observations (host array)"""
    n = obs.shape[0]
    return obs[:, P.nb * 9:(P.nb + P.buffer * P.nl) * 9].reshape(n, P.buffer * P.nl, 9)[:, :, 8] == 1


def policy_pick(P, obs, e, k, seed=5):
    """the flat index of env e at its k-th step: a keyed choice among the valid flat indices of its own observation (0 when none)"""
    v = np.nonzero(_valid(P, obs[None])[0])[0]
    if len(v) == 0:
        return 0
    return int(v[rnd_u64(seed, int(e), int(k)) % len(v)])


def _pick(rng, live, n):
    s = SIZES[rng.randint(len(SIZES))]
    k = {"0": 0, "1": 1, "1%": max(1, n // 100), "50%": n // 2, "all": n}[s]
    return np.sort(rng.permutation(live)[:min(k, len(live))])


def _state(P):
    return _np(P._obs), _np(P._rew), _np(P._done), _np(P._info), _np(P.buffer_items()), _snap(P)


def _history(Z, episodes=2, max_steps=700, steps=None):
    """full buffered steps of twin Z with policy_pick until every env finished `episodes` episodes (or `steps` steps) -> states after
    reset, step 1, ..."""
    n = Z.n_envs
    Z.reset()
    hist = [_state(Z)]
    eps = np.zeros(n, dtype=int)
    t = 0
    while (eps.min() < episodes) if steps is None else (t < steps):
        assert steps is not None or t < max_steps, "the twin's envs finish %d episodes within %d steps" % (episodes, max_steps)
        obs = hist[-1][0]
        flat = torch.as_tensor(np.array([policy_pick(Z, obs[e], e, t) for e in range(n)], dtype=np.int32), device=Z.device)
        Z.step(leaf_idx=flat)
        hist.append(_state(Z))
        eps += hist[-1][2].astype(int)
        t += 1
    return hist


def _parity(A, Z, seed=0, snap_every=5, steps=None):
    """drive A by random selections (list and mask forms) until every env took as many steps as the twin's history, checking each
    selected env against the twin and every unselected env against its state before the call"""
    n = A.n_envs
    hist = _history(Z, steps=steps)
    T = len(hist) - 1
    A.reset()
    assert np.array_equal(_np(A._obs), hist[0][0])
    rng = np.random.RandomState(seed)
    ks = np.zeros(n, dtype=int)
    calls = 0
    while ks.min() < T:
        sel = _pick(rng, np.nonzero(ks < T)[0], n)
        flat = rng.randint(-5, A.buffer * A.nl + 5, n).astype(np.int32)  # garbage for the envs not selected
        for e in sel:
            flat[e] = policy_pick(A, hist[ks[e]][0][e], e, ks[e])
        A._rew.fill_(SENT_REW); A._done.fill_(SENT_DONE); A._info.fill_(SENT_INFO)
        before = _np(A._obs)
        check_snap = calls % snap_every == 0
        snap0 = _snap(A) if check_snap else None
        flat_t = torch.as_tensor(flat, device=A.device)
        if calls % 2:
            m = torch.zeros(n, dtype=torch.bool, device=A.device)
            m[torch.as_tensor(sel, dtype=torch.long, device=A.device)] = True
            o, r, d, i = A.buffer_step_envs(flat_t, mask=m)
        else:
            o, r, d, i = A.buffer_step_envs(flat_t, env_idx=sel)
        o, r, d, i = _np(o), _np(r), _np(d), _np(i)
        items = _np(A.buffer_items())
        snap = _snap(A) if check_snap else None
        un = np.ones(n, dtype=bool)
        un[sel] = False
        for e in sel:
            ho, hr, hd, hi, hit, hs = hist[ks[e] + 1]
            assert np.array_equal(o[e].view(np.uint8), ho[e].view(np.uint8)), "rows of env %d after its step %d (call %d)" % (e, ks[e] + 1, calls)
            assert r[e] == hr[e] and d[e] == hd[e] and np.array_equal(i[e], hi[e]), "reward / done / record of env %d, step %d" % (e, ks[e] + 1)
            assert np.array_equal(items[e], hit[e]), "buffered items of env %d, step %d" % (e, ks[e] + 1)
            if check_snap:
                assert np.array_equal(snap[e], hs[e]), "buffered record of env %d, step %d" % (e, ks[e] + 1)
        assert np.array_equal(o[un], before[un]), "an unselected env's rows were written (call %d)" % calls
        assert (r[un] == SENT_REW).all() and (d[un] == SENT_DONE).all() and (i[un] == SENT_INFO).all(), "unselected entries written (call %d)" % calls
        if check_snap:
            assert np.array_equal(snap[un], snap0[un]), "an unselected env's record changed (call %d)" % calls
        ks[sel] += 1
        calls += 1
    return T


# ---- 1. selection parity -----------------------------------------------------------------------------------------------------------------
PARITY = [(s, c, B, {}) for c in (False, True) for s in ((1, 2, 3) if not c else (1, 3)) for B in (3, 5)]
PARITY += [(1, False, 1, {}), (2, False, 3, dict(LNES="EP")), (1, False, 3, dict(shuffle=True)), (1, False, 5, dict(obs_dtype=torch.float32)),
           (1, True, 3, dict(obs_dtype=torch.float32)), (3, False, 3, dict(traj=9))]


def _pid(c):
    s, cont, B, kw = c
    return "%s%d-B%d%s" % ("c" if cont else "d", s, B, "".join("-%s=%s" % (k, str(v).replace("torch.", "")) for k, v in sorted(kw.items())))


@pytest.mark.parametrize("setting,continuous,B,kw", PARITY, ids=[_pid(c) for c in PARITY])
def test_selection_parity(setting, continuous, B, kw):
    kw = dict(kw)
    traj = kw.pop("traj", 0)
    n = 64
    st = _streams(n, setting, continuous, 1500, seed=17)
    A, Z = _batch(n, setting, continuous, st, buffer=B, **kw), _batch(n, setting, continuous, st, buffer=B, **kw)
    if traj:
        A.set_trajectory_length(traj); Z.set_trajectory_length(traj)
    _parity(A, Z)
    A.close(); Z.close()


def test_selection_parity_capacity_cases():
    """the capacity cases' configurations and streams (tests/golden/capacity_cases.npz) through selections, once each"""
    pct_b200 = _pb()
    cases = load_capacity_cases()
    for name in sorted(cases):
        c = cases[name]
        s = np.stack([c["stream"]] * 4)
        mk = lambda: pct_b200.PctBatch(len(s), c["setting"], container_size=c["container"], continuous=c["domain"] == "continuous",
                                       item_set=None if c["domain"] == "continuous" else c["items"], internal_node_holder=c["nb"],
                                       leaf_node_holder=c["nl"], obs_dtype=torch.float64, item_stream=s, size_minimum=c["size_minimum"],
                                       LNES=c["lnes"], buffer=3)
        A, Z = mk(), mk()
        _parity(A, Z, snap_every=3, steps=min(int(c["steps"]) + 40, len(c["stream"]) - 40))
        A.close(); Z.close()


# ---- 2. B = 1 is the plain selected call ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", [(1, False), (2, False), (3, False), (1, True), (3, True)], ids=["d1", "d2", "d3", "c1", "c3"])
def test_b1_is_the_plain_selected_call(setting, continuous):
    n = 64
    st = _streams(n, setting, continuous, 800, seed=4)
    P, Q = _batch(n, setting, continuous, st, buffer=1), _batch(n, setting, continuous, st)
    P.reset(); Q.reset()
    rng = np.random.RandomState(1)
    ip = torch.empty((n, 8), dtype=torch.int32, device=P.device)
    iq = torch.empty_like(ip)
    for call in range(120):
        sel = np.sort(rng.permutation(n)[:rng.randint(1, n + 1)])
        for X in (P, Q):
            X._rew.fill_(SENT_REW); X._done.fill_(SENT_DONE); X._info.fill_(SENT_INFO)
        if call % 9 == 8:
            ip.fill_(SENT_INFO); iq.fill_(SENT_INFO)
            op = P.buffer_reset_envs(env_idx=sel, info=ip)
            oq = Q.reset(env_idx=sel, info=iq, whole_batch=False)
            assert torch.equal(ip, iq), call
        else:
            flat = torch.as_tensor(np.array([policy_pick(P, _np(P._obs[e]), e, call) for e in range(n)], dtype=np.int32), device=P.device)
            op, rp, dp, i1 = P.buffer_step_envs(flat, env_idx=sel)
            oq, rq, dq, i2 = Q.step(leaf_idx=flat, env_idx=sel)
            assert torch.equal(rp, rq) and torch.equal(dp, dq) and torch.equal(i1, i2), call
        assert np.array_equal(_np(op).view(np.uint8), _np(oq).view(np.uint8)), call
    P.close(); Q.close()


# ---- 3. reset of chosen envs ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous,B,traj", [(1, False, 3, 0), (3, False, 5, 11), (2, False, 3, 0), (1, True, 5, 0), (3, True, 3, 9)],
                         ids=["d1-B3", "d3-B5-traj", "d2-B3", "c1-B5", "c3-B3-traj"])
def test_reset_envs_equal_the_full_reset(setting, continuous, B, traj):
    n, L = 48, 1200
    st = _streams(n, setting, continuous, L, seed=9)
    A, Z = _batch(n, setting, continuous, st, buffer=B), _batch(n, setting, continuous, st, buffer=B)
    for X in (A, Z):
        if traj:
            X.set_trajectory_length(traj)
        X.reset()
    rng = np.random.RandomState(2)
    t_dev = torch.zeros((), dtype=torch.int64, device=A.device)
    ia = torch.empty((n, 8), dtype=torch.int32, device=A.device)
    iz = torch.empty_like(ia)
    for rnd in range(4):
        for t in range(7 + 3 * rnd):  # identical histories
            flat = A.random_policy_dev(11, t_dev).clone()
            A.step(leaf_idx=flat); Z.step(leaf_idx=flat)
            t_dev += 1
        S = np.sort(rng.permutation(n)[:rng.randint(1, n // 2)])
        pos = np.array([A.state(e)["draw_pos"] for e in range(n)])
        before, items0, snap0 = _np(A._obs), _np(A.buffer_items()), _snap(A)
        ia.fill_(SENT_INFO)
        if rnd % 2:
            m = torch.zeros(n, dtype=torch.uint8, device=A.device)
            m[torch.as_tensor(S, dtype=torch.long, device=A.device)] = 1
            oa = _np(A.buffer_reset_envs(mask=m, info=ia))
        else:
            oa = _np(A.buffer_reset_envs(env_idx=S, info=ia))
        oz = _np(Z.reset(info=iz))
        un = np.ones(n, dtype=bool)
        un[S] = False
        sa, sz = _snap(A), _snap(Z)
        items_a, items_z = _np(A.buffer_items()), _np(Z.buffer_items())
        assert np.array_equal(oa[S].view(np.uint8), oz[S].view(np.uint8)), "rows of the reset envs"
        assert np.array_equal(_np(ia)[S], _np(iz)[S]), "records of the reset envs"
        assert np.array_equal(items_a[S], items_z[S]) and np.array_equal(sa[S], sz[S]), "buffers / records of the reset envs"
        assert np.array_equal(oa[un], before[un]) and (_np(ia)[un] == SENT_INFO).all(), "envs outside S written"
        assert np.array_equal(items_a[un], items0[un]) and np.array_equal(sa[un], snap0[un]), "envs outside S changed"
        for e in S:  # the next B draws of the env's stream (under a trajectory length: the first B of the next trajectory)
            p0 = int(pos[e])
            if traj and p0 % traj:
                p0 += traj - p0 % traj
            assert np.array_equal(items_a[e], st[e, [(p0 + k) % L for k in range(B)]]), e
        # the twin is now reset everywhere: make A equal it again
        A.buffer_restore(torch.as_tensor(sz, device=A.device))
    A.close(); Z.close()


@pytest.mark.parametrize("setting,continuous", [(1, False), (3, False), (1, True)], ids=["d1", "d3", "c1"])
def test_mid_episode_reset_replays_on_the_oracle(setting, continuous):
    """steps with mid-episode resets of chosen envs, replayed on the oracle as a plain stream of the chosen items (a reset consumes one
    draw of that stream: a placeholder item)"""
    n, B = 32, 3
    st = _streams(n, setting, continuous, 800, seed=23)
    P = _batch(n, setting, continuous, st, buffer=B)
    obs = P.reset().clone()
    nb, nl = P.nb, P.nl
    t_dev = torch.zeros((), dtype=torch.int64, device=P.device)
    rng = np.random.RandomState(3)
    log = []  # per step: (reset envs before it, obs, items, flat, reward, done)
    eps = np.zeros(n, dtype=int)
    for t in range(400):
        R = np.sort(rng.permutation(n)[:4]) if t % 6 == 4 else np.zeros(0, dtype=int)
        if len(R):
            obs = P.buffer_reset_envs(env_idx=R).clone()
        items = _np(P.buffer_items())
        flat = _np(P.random_policy_dev(PSEED, t_dev))
        o, r, d, _ = P.step(leaf_idx=torch.as_tensor(flat).to(P.device))
        log.append((set(R.tolist()), _np(obs), items, flat, _np(r), _np(d)))
        obs = o.clone()
        eps += log[-1][5].astype(int)
        t_dev += 1
        if eps.min() >= 2 and t > 40:
            break
    for e in range(0, n, 5):
        seq = []
        for R, _, items, flat, _, _ in log:
            it = items[e, flat[e] // nl]
            if e in R:
                seq.append(it)  # placeholder: the oracle's reset draws it
            seq.append(it)
        seq = np.concatenate([np.stack(seq), np.tile(st[e, :1], (2, 1))])
        o = OracleContinuous(setting, stream=seq) if continuous else OracleDiscrete(setting, stream=seq)
        ob = o.reset()
        for t, (R, ob_p, items, flat, rew, done) in enumerate(log):
            if e in R:
                ob = o.reset()
            blk = ob_p[e, nb * 9:(nb + B * nl) * 9].reshape(B, nl, 9)
            j, l = flat[e] // nl, flat[e] % nl
            assert np.array_equal(ob[:nb * 9], ob_p[e, :nb * 9]), (e, t)
            assert np.array_equal(ob[nb * 9:(nb + nl) * 9].reshape(nl, 9), blk[j]), (e, t)
            ob, r, d, _ = o.step(blk[j, l].astype(np.float64))
            assert np.float32(r) == rew[e] and bool(d) == bool(done[e]), (e, t)
            if d:
                ob = o.reset()
    P.close()



# ---- 4. snapshot / restore -----------------------------------------------------------------------------------------------------------------
def _drive(X, t_dev, steps, seed=PSEED):
    out = []
    for _ in range(steps):
        flat = X.random_policy_dev(seed, t_dev).clone()
        o, r, d, i = X.step(leaf_idx=flat)
        out.append((_np(o), _np(r), _np(d), _np(i)))
        t_dev += 1
    return out


@pytest.mark.parametrize("setting,continuous,B,kw", [(1, False, 3, {}), (2, False, 5, {}), (3, False, 3, dict(shuffle=True)), (1, True, 3, {}),
                                                      (3, True, 5, dict(obs_dtype=torch.float32)), (1, False, 1, dict(LNES="CP"))],
                         ids=["d1-B3", "d2-B5", "d3-B3-shuffle", "c1-B3", "c3-B5-f32", "d1-B1-CP"])
def test_snapshot_restore(setting, continuous, B, kw):
    n = 48
    st = _streams(n, setting, continuous, 900, seed=13)
    A, Z, F = (_batch(n, setting, continuous, st, buffer=B, **kw) for _ in range(3))
    A.reset(); Z.reset(); F.reset()
    ta = torch.zeros((), dtype=torch.int64, device=A.device)
    tz = torch.zeros((), dtype=torch.int64, device=A.device)
    _drive(A, ta, 25); _drive(Z, tz, 25)
    rec = A.buffer_snapshot()
    obs_at = _np(A._obs)
    assert np.array_equal(_snap(A), _snap(Z))
    _drive(A, ta, 13)  # diverge, then restore into the same slots
    stale = _np(A.buffer_restore(rec))
    assert np.array_equal(stale.view(np.uint8), obs_at.view(np.uint8)), "restored rows are the source's observation"
    s1 = _snap(A)
    A.buffer_restore(torch.as_tensor(s1, device=A.device), write_obs=False)
    assert np.array_equal(_snap(A), s1), "snapshot -> restore -> snapshot"
    assert np.array_equal(s1, _snap(Z))
    # restore over a richer, stale env equals restore into a fresh handle
    fresh = _np(F.buffer_restore(rec))
    assert np.array_equal(fresh.view(np.uint8), stale.view(np.uint8)) and np.array_equal(_snap(F), s1)
    # the same future as the untouched twin
    ta.fill_(int(tz)); tf = tz.clone()
    for (oa, ra, da, ia), (oz, rz, dz, iz), (of, rf, df, i_f) in zip(_drive(A, ta, 30), _drive(Z, tz, 30), _drive(F, tf, 30)):
        assert np.array_equal(oa.view(np.uint8), oz.view(np.uint8)) and np.array_equal(of.view(np.uint8), oz.view(np.uint8))
        assert np.array_equal(ra, rz) and np.array_equal(da, dz) and np.array_equal(ia, iz) and np.array_equal(rf, rz) and np.array_equal(i_f, iz)
    for X in (A, Z, F):
        X.close()


@pytest.mark.parametrize("continuous", [False, True], ids=["d", "c"])
def test_fan_out(continuous):
    """one record into many slots of another handle: identical rows; children with the same stream row and flat index step identically"""
    n, K, B, setting = 16, 24, 3, 1
    st = _streams(n, setting, continuous, 600, seed=29)
    P = _batch(n, setting, continuous, st, buffer=B)
    P.reset()
    t_dev = torch.zeros((), dtype=torch.int64, device=P.device)
    _drive(P, t_dev, 9)
    src = 5
    rec = P.buffer_snapshot(env_idx=[src])
    S = _batch(K, setting, continuous, np.stack([st[src]] * K), buffer=B)
    S.reset()
    o = _np(S.buffer_restore(rec, env_idx=np.arange(K), rec_idx=np.zeros(K, dtype=np.int32)))
    assert (o == o[:1]).all() and np.array_equal(o[0].view(np.uint8), _np(P._obs[src]).view(np.uint8))
    flat = torch.full((K,), policy_pick(S, o[0], 0, 0), dtype=torch.int32, device=S.device)
    o2, r2, d2, i2 = (_np(x) for x in S.buffer_step_envs(flat, mask=torch.ones(K, dtype=torch.bool, device=S.device)))
    assert (o2 == o2[:1]).all() and (r2 == r2[0]).all() and (d2 == d2[0]).all() and (i2 == i2[:1]).all()
    s2 = _snap(S)
    assert (s2 == s2[:1]).all()
    # the children equal the source stepped with the same flat index
    f = torch.zeros(n, dtype=torch.int32, device=P.device)
    f[src] = flat[0]
    op, rp, _, _ = P.buffer_step_envs(f, env_idx=[src])
    assert np.array_equal(_np(op[src]).view(np.uint8), o2[0].view(np.uint8)) and float(rp[src]) == r2[0]
    P.close(); S.close()


@pytest.mark.parametrize("continuous", [False, True], ids=["d", "c"])
def test_foreign_records_are_refused(continuous):
    n, B = 8, 3
    P = _batch(n, 1, continuous, buffer=B)
    plain, other_b, other_cfg = _batch(n, 1, continuous), _batch(n, 1, continuous, buffer=B + 1), _batch(n, 2, continuous, buffer=B)
    for X in (P, plain, other_b, other_cfg):
        X.reset()
    sz = P.buffer_snapshot_bytes
    assert plain.snapshot_bytes < sz < other_b.buffer_snapshot_bytes
    recs = []
    r = torch.zeros((1, sz), dtype=torch.uint8, device=P.device)
    r[0, :plain.snapshot_bytes] = plain.snapshot(env_idx=[0])[0]
    recs.append(r)
    recs.append(other_b.buffer_snapshot(env_idx=[0])[:, :sz].contiguous())
    recs.append(other_cfg.buffer_snapshot(env_idx=[0]))
    for k, rec in enumerate(recs):
        e = 2 + k
        before, snap0, items0 = _np(P._obs), _snap(P), _np(P.buffer_items())
        assert not P.state(e)["flags"] & BAD_SNAPSHOT
        P.buffer_restore(rec, env_idx=[e], rec_idx=[0])
        assert np.array_equal(_np(P._obs), before) and np.array_equal(_np(P.buffer_items()), items0), k
        assert P.state(e)["flags"] & BAD_SNAPSHOT, k
        s = _snap(P)
        assert np.array_equal(np.delete(s, e, 0), np.delete(snap0, e, 0)), k
        _, _, _, info = P.buffer_step_envs(torch.zeros(n, dtype=torch.int32, device=P.device), env_idx=[e])
        assert _np(info)[e, 1] & BAD_SNAPSHOT, k
    for X in (P, plain, other_b, other_cfg):
        X.close()


@pytest.mark.parametrize("name", NEEDS_ALIAS_D)
def test_alias_cases_continue_exactly(name):
    """the alias-mode cases' configurations: records taken mid-run continue in a fresh handle exactly as the source continues"""
    pct_b200 = _pb()
    c = CASES[name]
    n = 8
    st = np.stack([case_stream(c, c["seed"], c["env"] + e, 400) for e in range(n)])
    mk = lambda: pct_b200.PctBatch(n, c["setting"], container_size=c["container"], item_set=c["items"], internal_node_holder=c["nb"],
                                   leaf_node_holder=c["nl"], obs_dtype=torch.float64, item_stream=st, buffer=3)
    A, F = mk(), mk()
    A.reset(); F.reset()
    ta = torch.zeros((), dtype=torch.int64, device=A.device)
    _drive(A, ta, 40)
    F.buffer_restore(A.buffer_snapshot())
    tf = ta.clone()
    for (oa, ra, da, ia), (of, rf, df, i_f) in zip(_drive(A, ta, 40), _drive(F, tf, 40)):
        assert np.array_equal(oa, of) and np.array_equal(ra, rf) and np.array_equal(da, df) and np.array_equal(ia, i_f)
    for e in range(n):  # the support graphs: supports, loads and their alias flags, polygons (not the per-box stacks, nor the alias bits past
        ga, gf = A.support_graph(e), F.support_graph(e)  # n_edge that earlier episodes left)
        assert ga.keys() == gf.keys()
        for k in sorted(set(ga) - {"alias_stale", "own_stack"}):
            assert str(ga[k]) == str(gf[k]) if not isinstance(ga[k], list) else all(np.array_equal(x, y) for x, y in zip(ga[k], gf[k])), (e, k)
    A.close(); F.close()


# ---- 5. the lookahead example ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", [(1, False), (2, False), (1, True)], ids=["d1", "d2", "c1"])
def test_lookahead_example(setting, continuous):
    """tests/buffer_search.py commits, on every root, the state a direct step with the chosen flat index gives"""
    n, K, B = 16, 6, 3
    st = _streams(n, setting, continuous, 700, seed=31)
    root, direct = _batch(n, setting, continuous, st, buffer=B), _batch(n, setting, continuous, st, buffer=B)
    search = _batch(n * K, setting, continuous, np.repeat(st, K, axis=0), buffer=B)
    root.reset(); direct.reset(); search.reset()
    gen = torch.Generator(device=root.device)
    gen.manual_seed(3)
    for t in range(30):
        flats = buffer_search.candidate_flats(root._obs, root.nb, root.nl, B, K, gen)
        took = buffer_search.one_ply(root, search, flats)
        _, r, _, _ = direct.step(leaf_idx=took)
        assert np.array_equal(_np(root._obs).view(np.uint8), _np(direct._obs).view(np.uint8)), t
        assert np.array_equal(_snap(root), _snap(direct)) and torch.equal(root.buffer_items(), direct.buffer_items()), t
    for X in (root, direct, search):
        X.close()


# ---- 6. CUDA graphs ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", [(1, False), (2, False), (1, True)], ids=["d1", "d2", "c1"])
def test_graph_capture(setting, continuous):
    """a captured buffer_policy_random -> buffer_step_envs(mask) -> buffer_reset_envs(mask=done) loop with a snapshot / restore inside
    equals the eager loop"""
    n, B, T = 64, 3, 6
    st = _streams(n, setting, continuous, 600, seed=8)
    G, E = _batch(n, setting, continuous, st, buffer=B), _batch(n, setting, continuous, st, buffer=B)
    G.reset(); E.reset()

    def make(X):
        return dict(t=torch.zeros((), dtype=torch.int64, device=X.device), idx=torch.zeros(n, dtype=torch.int32, device=X.device),
                    m=(torch.arange(n, device=X.device) % 3 != 0), snap=torch.zeros((n // 4, X.buffer_snapshot_bytes), dtype=torch.uint8, device=X.device),
                    src=torch.arange(n // 4, device=X.device, dtype=torch.int32), dst=torch.arange(n // 2, n // 2 + n // 4, device=X.device, dtype=torch.int32),
                    obs=torch.zeros((T, n, X.obs_len), dtype=X.obs_dtype, device=X.device), rew=torch.zeros((T, n), dtype=torch.float32, device=X.device))

    def body(X, s):
        for t in range(T):
            X.random_policy_dev(PSEED, s["t"], out=s["idx"])
            _, r, d, _ = X.buffer_step_envs(s["idx"], mask=s["m"])
            X.buffer_reset_envs(mask=d)
            if t == 2:
                X.buffer_snapshot(env_idx=s["src"], out=s["snap"])
            if t == 4:
                X.buffer_restore(s["snap"], env_idx=s["dst"])
            s["obs"][t].copy_(X._obs)
            s["rew"][t].copy_(r)
            s["t"].add_(1)
    sg, se = make(G), make(E)
    torch.cuda.synchronize()
    strm = torch.cuda.Stream()
    strm.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=strm):
        body(G, sg)
    for rep in range(3):
        g.replay()
        body(E, se)
        torch.cuda.synchronize()
        assert torch.equal(sg["obs"], se["obs"]) and torch.equal(sg["rew"], se["rew"]), rep
        assert np.array_equal(_snap(G), _snap(E)), rep
    G.close(); E.close()


# ---- 7. errors -----------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("continuous", [False, True], ids=["d", "c"])
def test_errors(continuous):
    pct_b200 = _pb()
    L = pct_b200._lib.lib()
    n, B = 8, 3
    P = _batch(n, 1, continuous, buffer=B)
    h = P.h
    vp = lambda t: C.c_void_p(t.data_ptr())
    obs = torch.zeros((n, P.obs_len), dtype=torch.float64, device=P.device)
    idx = torch.zeros(n, dtype=torch.int32, device=P.device)
    mask = torch.ones(n, dtype=torch.uint8, device=P.device)
    sz = L.pct_buffer_snapshot_bytes(h)
    assert sz == P.buffer_snapshot_bytes > P.snapshot_bytes == L.pct_snapshot_bytes(h)
    buf = torch.zeros(2 * sz + 16, dtype=torch.uint8, device=P.device)
    rew, done = P._rew, P._done
    # before the first reset
    assert L.pct_buffer_step_envs(h, vp(idx), 1, None, vp(idx), vp(obs), vp(rew), vp(done), None, None) == STATE
    assert L.pct_buffer_reset_envs(h, vp(idx), 1, None, vp(obs), None, None) == STATE
    assert L.pct_buffer_snapshot(h, None, 1, vp(buf), None) == STATE
    assert L.pct_buffer_restore(h, None, None, 1, vp(buf), None, None) == STATE
    P.reset()
    ptr = lambda t: vp(t) if t is not None else None
    step = lambda e, k, m, li=idx, o=obs, r=rew, d=done: L.pct_buffer_step_envs(h, e, k, m, ptr(li), ptr(o), ptr(r), ptr(d), None, None)
    assert step(vp(idx), 1, vp(mask)) == INVALID  # both
    assert step(None, 1, None) == INVALID  # neither
    assert step(vp(idx), -1, None) == INVALID
    assert step(None, n - 1, vp(mask)) == INVALID
    for kw in (dict(li=None), dict(o=None), dict(r=None), dict(d=None)):
        assert step(vp(idx), 1, None, **kw) == INVALID, kw
    assert step(vp(idx), 0, None, li=None) == 0  # n == 0: a no-op
    rs = lambda e, k, m, o=obs: L.pct_buffer_reset_envs(h, e, k, m, ptr(o), None, None)
    assert rs(vp(idx), 1, vp(mask)) == INVALID and rs(None, 1, None) == INVALID and rs(vp(idx), -2, None) == INVALID
    assert rs(None, n + 1, vp(mask)) == INVALID and rs(vp(idx), 1, None, o=None) == INVALID
    assert L.pct_buffer_snapshot(h, None, 1, None, None) == INVALID
    assert L.pct_buffer_snapshot(h, None, -1, vp(buf), None) == INVALID
    assert L.pct_buffer_snapshot(h, None, 1, C.c_void_p(buf.data_ptr() + 8), None) == INVALID
    assert L.pct_buffer_restore(h, None, None, 1, None, None, None) == INVALID
    assert L.pct_buffer_restore(h, None, None, -1, vp(buf), None, None) == INVALID
    assert L.pct_buffer_restore(h, None, None, 1, C.c_void_p(buf.data_ptr() + 4), None, None) == INVALID
    with pytest.raises(pct_b200.PctError):
        P.buffer_step_envs(idx)  # no selection
    with pytest.raises(pct_b200.PctError):
        P.buffer_step_envs(idx[:3], env_idx=[0])
    with pytest.raises(pct_b200.PctError):
        P.buffer_reset_envs(env_idx=[0], mask=mask)
    with pytest.raises(pct_b200.PctError):
        P.buffer_restore(torch.zeros((1, sz - 16), dtype=torch.uint8, device=P.device))
    with pytest.raises(pct_b200.PctError):
        P.buffer_snapshot(out=torch.zeros((n, sz + 1), dtype=torch.uint8, device=P.device))
    # out-of-range record indices map to -1 on the device: skipped
    before = _snap(P)
    P.buffer_restore(P.buffer_snapshot(env_idx=[1]), env_idx=[3], rec_idx=[7])
    assert np.array_equal(_snap(P), before)
    torch.cuda.synchronize()
    P.close()
    Q = _batch(n, 1, continuous)  # a plain handle
    Q.reset()
    assert L.pct_buffer_snapshot_bytes(Q.h) == 0
    assert L.pct_buffer_step_envs(Q.h, vp(idx), 1, None, vp(idx), vp(obs), vp(rew), vp(done), None, None) == STATE
    assert L.pct_buffer_reset_envs(Q.h, vp(idx), 1, None, vp(obs), None, None) == STATE
    assert L.pct_buffer_snapshot(Q.h, None, 1, vp(buf), None) == STATE
    assert L.pct_buffer_restore(Q.h, None, None, 1, vp(buf), None, None) == STATE
    for f in (lambda: Q.buffer_step_envs(idx, env_idx=[0]), lambda: Q.buffer_reset_envs(env_idx=[0]), lambda: Q.buffer_snapshot(),
              lambda: Q.buffer_snapshot_bytes, lambda: Q.buffer_restore(torch.zeros((1, 16), dtype=torch.uint8, device=Q.device))):
        with pytest.raises(pct_b200.PctError):
            f()
    Q.close()
