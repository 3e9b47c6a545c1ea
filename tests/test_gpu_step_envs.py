"""GPU: stepping, resetting and re-expanding a chosen subset of envs (pct_step_envs, pct_reset_envs_only, pct_set_items_only;
PctBatch.step(env_idx= / mask=), reset(..., whole_batch=False), set_items(..., whole_batch=False)).

The parity claim: an env's trajectory does not depend on which other envs step with it.  Batch A is driven by a random schedule of
selections (list and mask forms, sizes 0, 1, ~1 %, ~50 % and all envs); its twin B, with the same item sources, takes full pct_steps.  The
action of env e at its k-th step is a keyed function of (e, k) and of its own observation (policy_pick), so after env e's t-th selected step
in A its observation row, reward, done and info record must equal B's env e after full step t, bit for bit.  On the way the schedule checks
that envs not selected are untouched: their observation rows, their reward / done / info entries (pre-filled with sentinel bytes) and their
snapshot records, while their action rows and leaf indices hold garbage.  After the schedule, full steps on both sides check that the LPT
buckets and the walk pools were left as a full step expects them.
"""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
from harness import CASES, ITEM_SET, NEEDS_ALIAS_D, case_stream, cont_case_stream, load_capacity_cases, make_stream, policy_pick  # noqa: E402
from pct_oracle import OracleContinuous, OracleDiscrete, make_continuous_stream  # noqa: E402
import many_supports as ms  # noqa: E402

pytestmark = pytest.mark.gpu
PSEED = 2024
DOMAINS = [(s, False) for s in (1, 2, 3)] + [(s, True) for s in (1, 2, 3)]
DOM_IDS = ["d%d" % s if not c else "c%d" % s for s, c in DOMAINS]
SENT_REW, SENT_DONE, SENT_INFO = -7.0, 0xAB, 0x5A5A5A5A
ERR_INVALID, ERR_STATE = -1, -4  # PCT_ERR_INVALID, PCT_ERR_STATE


def _pb():
    import pct_b200
    return pct_b200


def _np(t):
    return t.cpu().numpy().copy()


def _streams(n, setting, continuous, length, seed=11):
    if continuous:
        return np.stack([make_continuous_stream(seed, e, length, setting) for e in range(n)])
    return np.stack([make_stream(seed, e, length, setting) for e in range(n)])


def _batch(n, setting, continuous, stream=None, obs_dtype=torch.float64, **kw):
    pct_b200 = _pb()
    if continuous:
        if stream is not None:
            return pct_b200.PctBatch(n, setting, container_size=(1.0, 1.0, 1.0), continuous=True, obs_dtype=obs_dtype, item_stream=stream,
                                     size_minimum=0.1, **kw)
        return pct_b200.PctBatch(n, setting, container_size=(1.0, 1.0, 1.0), continuous=True, obs_dtype=obs_dtype,
                                 sample_from_distribution=True, seed=1234, **kw)
    if stream is not None:
        return pct_b200.PctBatch(n, setting, item_set=ITEM_SET, obs_dtype=obs_dtype, item_stream=stream, **kw)
    return pct_b200.PctBatch(n, setting, item_set=ITEM_SET, obs_dtype=obs_dtype, seed=1234, **kw)


def _snap(b):
    return _np(b.snapshot(out=torch.zeros((b.n_envs, b.snapshot_bytes), dtype=torch.uint8, device=b.device)))


class Policy(object):
    """the action of env e at its k-th step: policy_pick on its own observation; `rows`: action rows instead of leaf indices;
    `script[e]`: scripted action rows of env e's first steps (the many-support floors)"""

    def __init__(self, b, rows=False, script=None, pseed=PSEED, key=None):
        self.nb, self.nl, self.rows, self.script, self.pseed, self.key = b.nb, b.nl, rows, script, pseed, key

    def one(self, obs_e, e, k):
        if self.script is not None and k < len(self.script[e]):
            return 0, self.script[e][k]
        return policy_pick(obs_e.astype(np.float64), self.nb, self.nl, self.pseed, int(e if self.key is None else self.key), int(k))

    def tensors(self, b, obs, ks, envs, garbage=None):
        """full-size action tensor: rows / indices of `envs` (env e at step ks[e] on observation obs[e]), garbage elsewhere"""
        n = b.n_envs
        if self.rows:
            a = garbage.uniform(-50, 50, (n, 9)) if garbage is not None else np.zeros((n, 9))
            for e in envs:
                a[e] = self.one(obs[e], e, ks[e])[1]
            return dict(actions=torch.tensor(a, dtype=torch.float64, device=b.device))
        a = garbage.randint(-1000, 1000, n) if garbage is not None else np.zeros(n)
        for e in envs:
            a[e] = self.one(obs[e], e, ks[e])[0]
        return dict(leaf_idx=torch.tensor(a, dtype=torch.int32, device=b.device))


def _history(B, pol, T):
    """B's outputs after full step t = 0 (the reset) .. T"""
    obs = _np(B.reset())
    hist = [(obs, None, None, None)]
    n = B.n_envs
    for t in range(T):
        o, r, d, i = [_np(x) for x in B.step(**pol.tensors(B, hist[-1][0], [t] * n, range(n)))]
        hist.append((o, r, d, i))
    return hist


SIZES = ["0", "1", "1%", "50%", "all"]


def _pick(rng, live, n):
    s = SIZES[rng.randint(len(SIZES))]
    k = {"0": 0, "1": 1, "1%": max(1, n // 100), "50%": n // 2, "all": n}[s]
    return np.sort(rng.permutation(live)[:min(k, len(live))])


def _schedule(A, B, pol, T, seed=0, snap_every=7, extra=3, episodes=2):
    """drive A by selections until every env took T steps, against B's full steps; then `extra` full steps on both.  -> B's history, which
    A's selected steps equal record for record"""
    n = A.n_envs
    hist = _history(B, pol, T + extra)
    ep = np.stack([h[2] for h in hist[1:T + 1]]).astype(bool).sum(0)
    assert ep.min() >= episodes, "schedule too short: an env finished %d episodes" % ep.min()
    assert np.array_equal(_np(A.reset()), hist[0][0])
    rng = np.random.RandomState(seed)
    ks = np.zeros(n, dtype=int)
    calls = 0
    while ks.min() < T:
        sel = _pick(rng, np.nonzero(ks < T)[0], n)
        obs_now = np.stack([hist[ks[e]][0][e] for e in range(n)])  # every env's current observation, from B (= A's, checked below)
        acts = pol.tensors(A, obs_now, ks, sel, garbage=rng)
        use_mask = rng.rand() < 0.5
        A._rew.fill_(SENT_REW); A._done.fill_(SENT_DONE); A._info.fill_(SENT_INFO)
        before = A._obs.clone()
        snap0 = _snap(A) if snap_every and calls % snap_every == 0 else None
        if use_mask:
            m = torch.zeros(n, dtype=torch.bool, device=A.device)
            m[torch.as_tensor(sel, dtype=torch.long, device=A.device)] = True
            o, r, d, i = A.step(mask=m, **acts)
        else:
            o, r, d, i = A.step(env_idx=sel, **acts)
        o, r, d, i = _np(o), _np(r), _np(d), _np(i)
        un = np.ones(n, dtype=bool)
        un[sel] = False
        for e in sel:
            t = ks[e] + 1
            ho, hr, hd, hi = hist[t]
            where = "env %d step %d (call %d, %s of %d)" % (e, t, calls, "mask" if use_mask else "list", len(sel))
            assert np.array_equal(o[e], ho[e]), "observation of " + where
            assert r[e] == hr[e] and d[e] == hd[e], "reward / done of " + where
            assert np.array_equal(i[e], hi[e]), "info of " + where
        assert np.array_equal(o[un], _np(before)[un]), "an unselected env's observation rows were written (call %d)" % calls
        assert (r[un] == SENT_REW).all() and (d[un] == SENT_DONE).all() and (i[un] == SENT_INFO).all(), \
            "an unselected env's reward / done / info was written (call %d)" % calls
        if snap0 is not None:
            assert np.array_equal(_snap(A)[un], snap0[un]), "an unselected env's record changed (call %d)" % calls
        ks[sel] += 1
        calls += 1
    for t in range(T, T + extra):  # full steps: every env in exactly one LPT bucket, walk pools empty
        out = [_np(x) for x in A.step(**pol.tensors(A, hist[t][0], [t] * n, range(n)))]
        for x, y, nm in zip(out, hist[t + 1], ("obs", "reward", "done", "info")):
            assert np.array_equal(x, y), "%s of the full step %d after the schedule" % (nm, t + 1)
    return hist


# ---- 1. per-env schedule parity ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", DOMAINS, ids=DOM_IDS)
@pytest.mark.parametrize("source", ["random", "traj"])
def test_schedule_parity(setting, continuous, source):
    n, T = 64, 70
    s = _streams(n, setting, continuous, 300) if source == "traj" else None
    A, B = _batch(n, setting, continuous, s), _batch(n, setting, continuous, s)
    if source == "traj":
        A.set_trajectory_length(25)
        B.set_trajectory_length(25)
    _schedule(A, B, Policy(A, rows=(setting == 3)), T)
    A.close(); B.close()


@pytest.mark.parametrize("setting,continuous", [(1, False), (2, True)], ids=["d1", "c2"])
def test_schedule_parity_float32_rows(setting, continuous):
    n = 48
    A, B = _batch(n, setting, continuous, obs_dtype=torch.float32), _batch(n, setting, continuous, obs_dtype=torch.float32)
    _schedule(A, B, Policy(A, rows=True), 60, seed=3)
    A.close(); B.close()


@pytest.mark.parametrize("lnes,shuffle", [("EV", True), ("EP", True), ("CP", True), ("FC", True), ("EMS", True)])
def test_schedule_parity_lnes_shuffle(lnes, shuffle):
    n = 32
    s = _streams(n, 1, False, 300)
    A, B = _batch(n, 1, False, s, LNES=lnes, shuffle=shuffle), _batch(n, 1, False, s, LNES=lnes, shuffle=shuffle)
    _schedule(A, B, Policy(A), 70, seed=1)
    A.close(); B.close()


@pytest.mark.parametrize("name", NEEDS_ALIAS_D)
def test_schedule_parity_alias_cases(name):
    c = CASES[name]
    n = 8
    s = np.stack([case_stream(c, c["seed"], c["env"] + e, 400) for e in range(n)])
    pct_b200 = _pb()
    mk = lambda: pct_b200.PctBatch(n, c["setting"], container_size=c["container"], item_set=c["items"], internal_node_holder=c["nb"],
                                   leaf_node_holder=c["nl"], obs_dtype=torch.float64, item_stream=s, env_id_base=c["env"])
    A, B = mk(), mk()
    _schedule(A, B, Policy(A), max(60, c["steps"] + 10), seed=2, episodes=1)
    A.close(); B.close()


@pytest.mark.parametrize("cont", [False, True], ids=["discrete", "continuous"])
@pytest.mark.parametrize("setting", [1, 3])
def test_schedule_parity_many_supports(cont, setting):
    """the many-support floors (tests/many_supports.py): scripted build-up rows, then the policy, on both sides"""
    n = 32
    s = ms.streams(cont, setting, n)
    script = [ms.plan(cont, setting, e)[1] for e in range(n)]
    pct_b200 = _pb()
    mk = lambda: pct_b200.PctBatch(n, setting, container_size=ms.container(cont), continuous=cont, item_set=None if cont else ITEM_SET,
                                   obs_dtype=torch.float64, item_stream=s, size_minimum=ms.unit(cont))
    A, B = mk(), mk()
    T = max(len(r) for r in script) + 20
    _schedule(A, B, Policy(A, rows=True, script=script), T, seed=4, episodes=0)
    A.close(); B.close()


VARIANTS = [("PCT_B200_WALK", "fork"), ("PCT_B200_K3", "block"), ("PCT_B200_GROUPS", "2"), ("PCT_B200_OVERLAP", "0"),
            ("PCT_B200_OBS_DELTA", "0"), ("PCT_B200_ALIAS", "0")]


@pytest.mark.parametrize("var,val", VARIANTS, ids=["%s=%s" % v for v in VARIANTS])
@pytest.mark.parametrize("setting,continuous", [(1, False), (2, False), (1, True)], ids=["d1", "d2", "c1"])
def test_schedule_parity_launch_variants(var, val, setting, continuous, monkeypatch):
    monkeypatch.setenv(var, val)
    n = 48
    A, B = _batch(n, setting, continuous), _batch(n, setting, continuous)
    _schedule(A, B, Policy(A), 60, seed=5)
    A.close(); B.close()


# ---- 2. against the oracle -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", [(1, False), (3, False), (2, True)], ids=["d1", "d3", "c2"])
def test_schedule_against_oracle(setting, continuous):
    n, T = 16, 60
    s = _streams(n, setting, continuous, 400)
    A = _batch(n, setting, continuous, s)
    orc = [OracleContinuous(setting, stream=s[e]) if continuous else OracleDiscrete(setting, stream=s[e]) for e in range(n)]
    ref = [o.reset() for o in orc]
    obs = _np(A.reset())
    assert np.array_equal(obs, np.stack(ref))
    rng = np.random.RandomState(9)
    ks = np.zeros(n, dtype=int)
    while ks.min() < T:
        sel = _pick(rng, np.nonzero(ks < T)[0], n)
        picks = {e: policy_pick(ref[e], A.nb, A.nl, PSEED, int(e), int(ks[e])) for e in sel}
        idx = np.zeros(n, dtype=np.int32)
        for e in sel:
            idx[e] = picks[e][0]
        o, r, d, _ = [_np(x) for x in A.step(leaf_idx=torch.tensor(idx, device=A.device), env_idx=sel)]
        for e in sel:
            ref[e], rr, dd, _ = orc[e].step(picks[e][1])
            assert np.float32(rr) == r[e] and bool(dd) == bool(d[e]), (e, ks[e])
            if dd:
                ref[e] = orc[e].reset()
            assert np.array_equal(o[e], ref[e]), "env %d after its step %d" % (e, ks[e] + 1)
        ks[sel] += 1
    A.close()


# ---- 4. the _only calls --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", DOMAINS, ids=DOM_IDS)
def test_only_calls_match_whole_batch(setting, continuous):
    """reset_envs_only / set_items_only give the selected envs the rows, records and env records pct_reset_envs / pct_set_items give
    them, and write nothing of the other envs"""
    n = 64
    A, B = _batch(n, setting, continuous), _batch(n, setting, continuous)
    A.reset(); B.reset()
    pol = Policy(A)
    rng = np.random.RandomState(6)
    for t in range(12):
        acts = pol.tensors(A, _np(A._obs), [t] * n, range(n))
        A.step(**acts); B.step(**acts)
    ia = torch.zeros((n, 8), dtype=torch.int32, device=A.device)
    ib = torch.full((n, 8), SENT_INFO, dtype=torch.int32, device=B.device)
    for call in range(6):
        sel = np.sort(rng.permutation(n)[:rng.randint(1, n // 2)])
        before = _np(B._obs)
        snap_b0 = _snap(B)
        ib.fill_(SENT_INFO)
        if call % 3 == 2:
            items = (rng.uniform(0.1, 0.5, (len(sel), 3)) if continuous else rng.randint(1, 6, (len(sel), 3)))
            oa = _np(A.set_items(items, env_idx=sel, info=ia))
            ob = _np(B.set_items(items, env_idx=sel, info=ib, whole_batch=False))
        elif call % 3 == 1:
            m = torch.zeros(n, dtype=torch.bool, device=A.device)
            m[torch.as_tensor(sel, device=A.device)] = True
            oa = _np(A.reset(mask=m, info=ia))
            ob = _np(B.reset(mask=m, info=ib, whole_batch=False))
        else:
            oa = _np(A.reset(env_idx=sel, info=ia))
            ob = _np(B.reset(env_idx=sel, info=ib, whole_batch=False))
        un = np.ones(n, dtype=bool)
        un[sel] = False
        assert np.array_equal(oa[sel], ob[sel]), "rows of the selected envs (call %d)" % call
        assert np.array_equal(_np(ia)[sel], _np(ib)[sel]), "info of the selected envs (call %d)" % call
        assert np.array_equal(ob[un], before[un]) and (_np(ib)[un] == SENT_INFO).all(), "unselected envs written (call %d)" % call
        sa, sb = _snap(A), _snap(B)
        assert np.array_equal(sa[sel], sb[sel]), "env records of the selected envs (call %d)" % call
        assert np.array_equal(sb[un], snap_b0[un]), "env records of unselected envs changed (call %d)" % call
        # the envs stay twins: their next full steps agree
        acts = pol.tensors(A, oa, [100 + call] * n, range(n))
        for x, y in zip(A.step(**acts), B.step(**acts)):
            assert torch.equal(x, y), "full step after call %d" % call
    A.close(); B.close()


@pytest.mark.parametrize("setting,continuous", DOMAINS, ids=DOM_IDS)
def test_gym_loop_with_reset_only(setting, continuous):
    """step + reset(mask=done, whole_batch=False) (auto_reset=False) against the auto-reset twin over two episodes"""
    n = 64
    A, B = _batch(n, setting, continuous), _batch(n, setting, continuous, auto_reset=False)
    assert torch.equal(A.reset(), B.reset())
    eps = np.zeros(n, dtype=int)
    for t in range(400):
        idx = A.random_policy(PSEED, t)
        oa = [_np(x) for x in A.step(leaf_idx=idx)]
        ob = [_np(x) for x in B.step(leaf_idx=idx)]
        assert np.array_equal(oa[1], ob[1]) and np.array_equal(oa[2], ob[2]), t
        done = oa[2] != 0
        assert np.array_equal(oa[0][~done], ob[0][~done]), t
        B.reset(mask=B._done, whole_batch=False)
        assert torch.equal(A._obs, B._obs), "observation after reset(mask=done, whole_batch=False), step %d" % t
        eps += done
        if eps.min() >= 2:
            break
    assert eps.min() >= 2
    A.close(); B.close()


# ---- 5. capacities ---------------------------------------------------------------------------------------------------------------------
def _mild_streams(c, n):
    """streams of the case's configuration with larger items, whose episodes end long before any capacity (cf. tests/test_gpu_capacities.py)"""
    if c["domain"] == "continuous":
        return [cont_case_stream(dict(c, lo=0.1, hi=0.5), 500 + e, 0, len(c["stream"])) for e in range(n)]
    mild = [(a, b, h) for a in (5, 7) for b in (5, 8) for h in (4, 6)]
    return [case_stream(dict(c, items=mild), 500 + e, 0, len(c["stream"])) for e in range(n)]


def test_capacity_cases_through_selections():
    """env 0 follows each capacity case (the trajectory of tests/test_gpu_capacities.py: the case's stream, its policy seed, env key 0)
    next to three envs with mild items, through selections against full steps; every flag then rises at the same per-env step as in that
    lock-step with the oracle.  The walk pools are shared by the batch (WALK_CONT_PER_ENV per env), so the mild neighbours keep the case's
    walks within the pool, as a batch of one would"""
    cases = load_capacity_cases()
    pct_b200 = _pb()
    for name in sorted(cases):
        c = cases[name]
        s = np.stack([c["stream"]] + _mild_streams(c, 3))
        n = len(s)
        mk = lambda: pct_b200.PctBatch(n, c["setting"], container_size=c["container"], continuous=c["domain"] == "continuous",
                                       item_set=None if c["domain"] == "continuous" else c["items"], internal_node_holder=c["nb"],
                                       leaf_node_holder=c["nl"], obs_dtype=torch.float64, item_stream=s, size_minimum=c["size_minimum"],
                                       LNES=c["lnes"])
        A, B = mk(), mk()
        T = min(int(c["steps"]), len(c["stream"]) - 40)
        hist = _schedule(A, B, Policy(A, rows=True, pseed=c["pseed"], key=0), T, seed=8, snap_every=0, episodes=0)
        # env 0's flags, step by step (A's records equal these): the first one is the case's (t_star, flag), as in the lock-step with the
        # oracle (tests/test_gpu_capacities.py: flags of step t are the record after step t, hist[t + 1])
        flags = [int(hist[t + 1][3][0, 1]) for t in range(min(T, int(c["n_steps"])))]
        fired = [(t, f) for t, f in enumerate(flags) if f][:1]
        assert fired == ([(c["t_star"], c["flag"])] if c["flag"] else []), (name, fired)
        A.close(); B.close()


# ---- 5b. the previous step's done bytes as the mask ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", [(1, False), (2, False), (3, True)], ids=["d1", "d2", "c3"])
def test_step_mask_is_done(setting, continuous):
    """step(mask=done) with the done tensor of the previous step, the buffer the call itself rewrites: the call selects the envs that
    finished before it, including those that do not finish again (their done byte becomes 0 during the call).  Against a twin stepping the
    same envs by list"""
    n = 64
    A, B = _batch(n, setting, continuous), _batch(n, setting, continuous)
    assert torch.equal(A.reset(), B.reset())
    selected = again = 0
    for t in range(120):
        outs_a = A.step(leaf_idx=A.random_policy(PSEED, 3 * t))
        outs_b = B.step(leaf_idx=B.random_policy(PSEED, 3 * t))
        done = outs_a[2]
        for k in (1, 2):  # two chained masked steps: the second one selects the envs that finished in the first
            sel = np.nonzero(_np(outs_b[2]))[0]
            selected += len(sel)
            outs_a = A.step(leaf_idx=A.random_policy(PSEED, 3 * t + k), mask=done)
            outs_b = B.step(leaf_idx=B.random_policy(PSEED, 3 * t + k), env_idx=sel)
            assert outs_a[2] is done
            again += int(_np(outs_a[2])[sel].sum())
            for x, y, nm in zip(outs_a, outs_b, ("obs", "reward", "done", "info")):
                assert torch.equal(x, y), "%s after step(mask=done) %d.%d (%d envs selected)" % (nm, t, k, len(sel))
        assert torch.equal(_snap_t(A), _snap_t(B)), "env records after round %d" % t
    assert selected > 50 and again < selected, (selected, again)  # most selected envs did not finish again: the case in question
    A.close(); B.close()


def _snap_t(b):
    return b.snapshot(out=torch.zeros((b.n_envs, b.snapshot_bytes), dtype=torch.uint8, device=b.device))


# ---- 6. delta rows -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", [(1, False), (3, True)], ids=["d1", "c3"])
@pytest.mark.parametrize("buffers", ["same", "alternate", "foreign_then_tracked"])
def test_delta_rows(setting, continuous, buffers, monkeypatch):
    """the delta-row contract per env (default) against full row writes (PCT_B200_OBS_DELTA=0) over the same selections"""
    n = 32
    A = _batch(n, setting, continuous)
    monkeypatch.setenv("PCT_B200_OBS_DELTA", "0")
    F = _batch(n, setting, continuous)
    bufs = [A._obs, torch.zeros_like(A._obs)]
    fb = [F._obs, torch.zeros_like(F._obs)]
    A.reset(); F.reset()
    rng = np.random.RandomState(10)
    pol = Policy(A)
    ks = np.zeros(n, dtype=int)
    for call in range(80):
        sel = _pick(rng, np.arange(n), n)
        j = {"same": 0, "alternate": call % 2, "foreign_then_tracked": int(call % 10 == 5)}[buffers]
        cur = _np(fb[0])  # F always steps into its own buffer: the envs' current observations
        acts = pol.tensors(A, cur, ks, sel)
        oa = _np(A.step(out=bufs[j], env_idx=sel, **acts)[0])
        of = _np(F.step(env_idx=sel, **acts)[0])
        assert np.array_equal(oa[sel], of[sel]), "rows of the selected envs (call %d, buffer %d)" % (call, j)
        ks[sel] += 1
    A.close(); F.close()


# ---- 7. graph capture ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting", [1, 2])
def test_graph_capture(setting):
    """policy -> step(mask=m) -> reset(mask=done, whole_batch=False), captured once and replayed with a new mask each time, equals the
    eager loop.  done is cleared before the step: envs not stepped keep the done byte of an earlier step otherwise"""
    n = 64
    A, G = _batch(n, setting, False, auto_reset=False), _batch(n, setting, False, auto_reset=False)
    assert torch.equal(A.reset(), G.reset())
    ta = torch.zeros(1, dtype=torch.int64, device=A.device)
    tg = torch.zeros(1, dtype=torch.int64, device=G.device)
    ma = torch.zeros(n, dtype=torch.bool, device=A.device)
    mg = torch.zeros(n, dtype=torch.bool, device=G.device)

    def body(b, t_dev, m):
        idx = b.random_policy_dev(PSEED, t_dev)
        b._done.zero_()
        b.step(leaf_idx=idx, mask=m)
        b.reset(mask=b._done, whole_batch=False)
        t_dev += 1

    rng = np.random.RandomState(12)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        mg.copy_(torch.ones(n, dtype=torch.bool))
        body(G, tg, mg)  # warm-up outside the capture (kernel attributes, modules)
        body(A, ta, mg.clone())
    torch.cuda.current_stream().wait_stream(side)
    assert torch.equal(A._obs, G._obs)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        body(G, tg, mg)
    for it in range(60):
        m = torch.as_tensor(rng.rand(n) < [0.02, 0.5, 1.0][it % 3])
        ma.copy_(m); mg.copy_(m)
        body(A, ta, ma)
        graph.replay()
        for x, y, nm in ((A._obs, G._obs, "obs"), (A._rew, G._rew, "reward"), (A._done, G._done, "done"), (A._info, G._info, "info")):
            assert torch.equal(x, y), "%s after replay %d" % (nm, it)
    torch.cuda.synchronize()
    A.close(); G.close()


# ---- 8. errors --------------------------------------------------------------------------------------------------------------------------
def test_errors():
    pct_b200 = _pb()
    from pct_b200 import _lib
    L = _lib.lib()
    n = 8
    b = _batch(n, 1, False)
    dev = b.device
    idx = torch.zeros(n, dtype=torch.int32, device=dev)
    lst = torch.arange(2, dtype=torch.int32, device=dev)
    m = torch.ones(n, dtype=torch.uint8, device=dev)
    p = lambda t: C.c_void_p(t.data_ptr())
    args = lambda: (p(b._obs), p(b._rew), p(b._done), p(b._info), None)
    # before the first reset
    assert L.pct_step_envs(b.h, p(lst), 2, None, None, 0, p(idx), *args()) == ERR_STATE
    assert L.pct_reset_envs_only(b.h, p(lst), 2, None, p(b._obs), None, None) == ERR_STATE
    it = torch.ones((2, 3), dtype=torch.int32, device=dev)
    assert L.pct_set_items_only(b.h, p(lst), 2, p(it), None, p(b._obs), None, None) == ERR_STATE
    with pytest.raises(pct_b200.PctError):
        b.step(leaf_idx=idx, env_idx=[0])
    b.reset()
    launches = b.kernel_launches
    assert L.pct_step_envs(b.h, p(lst), 0, None, None, 0, p(idx), *args()) == 0 and b.kernel_launches == launches  # n == 0: nothing
    assert L.pct_reset_envs_only(b.h, p(lst), 0, None, p(b._obs), None, None) == 0 and b.kernel_launches == launches
    assert L.pct_step_envs(b.h, p(lst), 2, p(m), None, 0, p(idx), *args()) == ERR_INVALID  # both
    assert L.pct_step_envs(b.h, None, 2, None, None, 0, p(idx), *args()) == ERR_INVALID  # neither
    assert L.pct_step_envs(b.h, p(lst), -1, None, None, 0, p(idx), *args()) == ERR_INVALID
    assert L.pct_step_envs(b.h, None, n - 1, p(m), None, 0, p(idx), *args()) == ERR_INVALID  # mask of n != n_envs
    assert L.pct_step_envs(b.h, p(lst), 2, None, None, 0, None, *args()) == ERR_INVALID  # no action
    assert L.pct_reset_envs_only(b.h, p(lst), 2, p(m), p(b._obs), None, None) == ERR_INVALID
    assert L.pct_reset_envs_only(b.h, None, n + 1, p(m), p(b._obs), None, None) == ERR_INVALID
    assert L.pct_reset_envs_only(b.h, p(lst), -3, None, p(b._obs), None, None) == ERR_INVALID
    assert L.pct_set_items_only(b.h, p(lst), -1, p(it), None, p(b._obs), None, None) == ERR_INVALID
    # a selection enqueues as many kernels as a step
    assert L.pct_step_envs(b.h, p(lst), 2, None, None, 0, p(idx), *args()) == 0
    per_step = b.kernel_launches - launches
    b.step(leaf_idx=idx)
    assert b.kernel_launches - launches == 2 * per_step
    with pytest.raises(pct_b200.PctError):
        b.step(leaf_idx=idx, env_idx=[0], mask=torch.ones(n, dtype=torch.bool))
    with pytest.raises(pct_b200.PctError):
        b.step(leaf_idx=idx, mask=torch.ones(n + 1, dtype=torch.bool))
    with pytest.raises(pct_b200.PctError):
        b.step(leaf_idx=idx[:4], env_idx=[0])
    with pytest.raises(pct_b200.PctError):
        b.reset(env_idx=[0], mask=torch.ones(n, dtype=torch.bool), whole_batch=False)
    out = b.step(leaf_idx=idx, env_idx=[])  # empty list: nothing enqueued
    assert out[0] is b._obs
    # indices outside [0, n_envs) are skipped
    before = _np(b._obs)
    b._done.fill_(SENT_DONE)
    b.step(leaf_idx=idx, env_idx=[-1, n, n + 100])
    assert np.array_equal(_np(b._obs), before) and (_np(b._done) == SENT_DONE).all()
    torch.cuda.synchronize()
    b.close()
