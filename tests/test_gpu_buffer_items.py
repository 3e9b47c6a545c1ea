"""GPU: item preview and item override of buffered envs (pct_buffer_preview_items / pct_buffer_set_items; PctBatch.buffer_preview_items /
buffer_set_items; DESIGN.md section 21).

- Lock-step with the buffered env on the oracle (tests/buffer_items.py: ItemsOracle), overrides interleaved with steps at random: random env subsets,
  random slots, items of the configuration's source, the [100, 100, 100] sentinel, fractional discrete sizes, setting-3 densities.  After
  every call: every observation byte, buffer_items(), the records' flags and sums exactly, and the untouched records of unlisted envs.
- Stream twin on the device: overriding slot j with X equals a twin whose stream holds X at the draw position that filled slot j, from
  then on, with the keyed shuffle too.
- B = 1: buffer_set_items is set_items_only on a plain handle byte for byte, and buffer_preview_items(k) columns 1..k of preview_items.
- Envs not listed keep their rows, records, buffers and snapshot bytes; set_items(buffer_items()) leaves every snapshot byte as it was.
- A snapshot after an override, restored into another slot, continues bit-identically.
- The search example without mirrored streams (tests/buffer_items.py: one_ply_any_source) commits what the mirrored one commits.
- CUDA-graph capture and the error codes.
"""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
from buffer_items import ItemsOracle, one_ply_any_source  # noqa: E402
from buffer_oracle import config, refill  # noqa: E402
from harness import ITEM_SET, make_stream  # noqa: E402
from pct_oracle import make_continuous_stream  # noqa: E402
import buffer_search  # noqa: E402

pytestmark = pytest.mark.gpu
INVALID, STATE = -1, -4  # PCT_ERR_INVALID, PCT_ERR_STATE
SENT_INFO = 0x5A5A5A5A
PSEED = 61


def _np(t):
    return t.cpu().numpy().copy()


def _batch(c, streams, B, obs_dtype=torch.float64, **kw):
    import pct_b200
    cont = c["domain"] == "continuous"
    return pct_b200.PctBatch(len(streams), c["setting"], container_size=c["container"], continuous=cont,
                             item_set=None if cont else c.get("items"), internal_node_holder=c["nb"], leaf_node_holder=c["nl"], obs_dtype=obs_dtype,
                             item_stream=np.stack(streams), size_minimum=c["size_minimum"], LNES=c.get("lnes", "EMS"), buffer=B, **kw)


def _flat_slot(f, B, nl):
    return f // nl if 0 <= f < B * nl else 0


def _override_rows(rng, c, items, pool, sel):
    """rows (len(sel), B, 4): each listed env's current buffer with random slots replaced by an item of `pool` (the configuration's own
    source), the [100, 100, 100] sentinel or, in the discrete domain, a fractional size; setting 3 gets random densities"""
    B = items.shape[1]
    rows = items[sel].copy()
    for i in range(len(sel)):
        for j in rng.permutation(B)[:rng.randint(1, B + 1)]:
            u = rng.rand()
            if u < 0.12:
                rows[i, j, :3] = 100
            else:
                rows[i, j] = pool[rng.randint(len(pool))]
                if c["domain"] == "discrete" and u < 0.3:
                    rows[i, j, :3] += 0.6  # truncated back on the device and in the model
            rows[i, j, 3] = rng.uniform(0.05, 1.0) if c["setting"] == 3 else 1.0
    return rows


def _check_obs(got, m, npd, where):
    want = m.obs.astype(npd)
    if np.array_equal(got.view(np.uint8), want.view(np.uint8)):
        return
    g, w = got.reshape(-1, 9), want.reshape(-1, 9)
    bad = int(np.nonzero((g.view(np.uint8) != w.view(np.uint8)).reshape(len(g), -1).any(1))[0][0])
    raise AssertionError("%s: observation differs first at row %d: %s, oracle %s" % (where, bad, g[bad].tolist(), w[bad].tolist()))


# ---- (a) lock-step against the model, overrides interleaved --------------------------------------------------------------------------------
LOCK = [(nm, B, 64 if B == 16 else 50, "f64") for nm in ("d1", "d2", "d3", "c1", "c2", "c3") for B in (1, 3, 16)]
LOCK += [("big_s1", 3, 50, "f64"), ("pallet_s2", 3, 50, "f64"), ("mm_s3", 3, 50, "f64"), ("d3", 3, 50, "f32"), ("c1", 3, 50, "f32"),
         ("cp_big_s1", 3, 50, "f64")]


@pytest.mark.parametrize("name,B,nl,dt", LOCK, ids=["%s-B%d-nl%d-%s" % c for c in LOCK])
def test_lockstep_with_overrides(name, B, nl, dt):
    c, mk = config(name, nl)
    n, steps = (6, 24) if B == 16 else (10, 40)
    rng = np.random.RandomState(B * 1000 + len(name))
    obs_dtype = torch.float64 if dt == "f64" else torch.float32
    npd = np.float64 if dt == "f64" else np.float32
    streams = [mk(23, e, 600) for e in range(n)]
    pool = np.concatenate([mk(29, e, 40) for e in range(4)])
    P = _batch(c, streams, B, obs_dtype)
    P.reset()
    models = [ItemsOracle(c, s, B) for s in streams]
    for m in models:
        m.reset()
    live = np.array([m.sticky == 0 for m in models])  # an env whose model carries a capacity flag leaves the comparison
    o = _np(P._obs)
    for e in np.nonzero(live)[0]:
        _check_obs(o[e], models[e], npd, "env %d reset" % e)
    t_dev = torch.zeros((), dtype=torch.int64, device=P.device)
    info = torch.zeros((n, 8), dtype=torch.int32, device=P.device)
    n_set = 0
    for t in range(steps):
        if rng.rand() < 0.6:  # an override of a random subset, out-of-range indices among them
            sel = np.sort(rng.permutation(n)[:rng.randint(1, n + 1)])
            rows = _override_rows(rng, c, _np(P.buffer_items()), pool, sel)
            idx = list(sel)
            if rng.rand() < 0.3:
                idx, rows = idx + [n + 3, -1], np.concatenate([rows, rows[:2] if len(rows) >= 2 else np.concatenate([rows, rows])])
            info.fill_(SENT_INFO)
            P.buffer_set_items(torch.as_tensor(rows, device=P.device), env_idx=idx, info=info)
            o, items, inf, raw = _np(P._obs), _np(P.buffer_items()), P.decode_info(info), _np(info)
            for e in range(n):
                where = "env %d override at step %d" % (e, t)
                if e not in sel:
                    assert (raw[e] == SENT_INFO).all(), where + ": the record of an unlisted env was written"
                    continue
                m = models[e]
                _, rec = m.set_items(rows[list(sel).index(e)])
                n_set += 1
                if not live[e]:
                    continue
                if m.sticky:
                    live[e] = False
                    continue
                _check_obs(o[e], m, npd, where)
                assert np.array_equal(items[e], m.buf), where + ": buffered items"
                got = tuple(int(inf[k][e]) for k in ("counter", "flags", "n_leaf", "n_cand", "n_ems"))
                assert got == tuple(rec[k] for k in ("counter", "flags", "n_leaf", "n_cand", "n_ems")), (where, got, rec)
                assert (inf["ratio"][e], inf["ep_reward"][e], inf["ep_len"][e]) == (0, 0, 0), where + ": ratio / ep_reward / ep_len"
        flat = P.random_policy_dev(PSEED, t_dev).clone()
        f = _np(flat)
        _, r, d, inf = P.step(leaf_idx=flat)
        t_dev += 1
        o, r, d, inf, items = _np(P._obs), _np(r), _np(d).astype(bool), P.decode_info(inf), _np(P.buffer_items())
        for e in range(n):
            m = models[e]
            assert f[e] == m.policy(PSEED, e, t) or not live[e], "env %d step %d: the policy's flat index" % (e, t)
            if not live[e]:
                continue
            _, rr, dd, rec = m.step(int(f[e]))
            if m.sticky:
                live[e] = False
                continue
            where = "env %d step %d" % (e, t)
            _check_obs(o[e], m, npd, where)
            assert np.array_equal(items[e], m.buf) and d[e] == dd and r[e] == np.float32(rr), where
            assert (inf["flags"][e], inf["n_leaf"][e], inf["n_cand"][e]) == (rec["flags"], rec["n_leaf"], rec["n_cand"]), (where, rec)
    assert n_set >= steps // 2 and live.sum() >= n // 2, (n_set, live)
    P.close()


# ---- (b) the stream twin on the device ------------------------------------------------------------------------------------------------------
def _streams(n, setting, cont, L, seed):
    mk = make_continuous_stream if cont else make_stream
    return np.stack([mk(seed, e, L, setting) for e in range(n)])


def _plain_cfg(setting, cont, nl=50):
    return config(("c" if cont else "d") + str(setting), nl)[0]


TWIN = [(s, cont, B, sh) for s in (1, 2, 3) for cont in (False, True) for B in (1, 3, 16) for sh in (False, True) if not (cont and sh and B == 16)]


@pytest.mark.parametrize("setting,cont,B,shuffle", TWIN, ids=["%s%d-B%d%s" % ("c" if c else "d", s, B, "-shuf" if sh else "") for s, c, B, sh in TWIN])
def test_stream_twin(setting, cont, B, shuffle):
    """A: steps, then slot j of a random subset <- X, then more steps.  Z: a fresh batch whose stream holds X at the draw position that
    filled slot j (tracked on the host by the refill rule), stepped with A's flat indices: from the override on, every row, reward and
    done of Z is A's"""
    n, L, t0, T = 24, 600, 9, 14
    c = _plain_cfg(setting, cont, 64 if B == 16 else 50)
    st = _streams(n, setting, cont, L, 41)
    other = _streams(n, setting, cont, L, 43)
    A = _batch(c, list(st), B, shuffle=shuffle)
    A.reset()
    pos = np.zeros(n, dtype=np.int64)
    ids = np.arange(L, dtype=np.float64)[:, None].repeat(4, 1)
    posbuf = np.zeros((n, B, 4))
    for e in range(n):
        pos[e] = refill(posbuf[e], 0, ids, True, 0)
    t_dev = torch.zeros((), dtype=torch.int64, device=A.device)
    flats, hist = [], []
    for t in range(t0 + T):
        if t == t0:
            rng = np.random.RandomState(B + 10 * setting)
            sel = np.sort(rng.permutation(n)[:n // 2])
            items = _np(A.buffer_items())
            js = rng.randint(B, size=len(sel))
            X = other[sel, rng.randint(L, size=len(sel))]
            rows = items[sel].copy()
            rows[np.arange(len(sel)), js] = X
            A.buffer_set_items(torch.as_tensor(rows, device=A.device), env_idx=sel)
            twin = st.copy()
            for i, e in enumerate(sel):
                p = int(posbuf[e, js[i], 0])
                assert p < L - 1
                twin[e, p] = X[i]
            hist.append((_np(A._obs), None, None))
        flat = A.random_policy_dev(PSEED, t_dev).clone()
        t_dev += 1
        f = _np(flat)
        _, r, d, _ = A.step(leaf_idx=flat)
        d = _np(d).astype(bool)
        flats.append(flat.clone())
        if t >= t0:
            hist.append((_np(A._obs), _np(r), d))
        for e in range(n):
            pos[e] = refill(posbuf[e], pos[e], ids, d[e], _flat_slot(int(f[e]), B, c["nl"]))
    Z = _batch(c, list(twin), B, shuffle=shuffle)
    Z.reset()
    for t in range(t0 + T):
        if t == t0:
            assert np.array_equal(_np(Z._obs).view(np.uint8), hist[0][0].view(np.uint8)), "the override's rows"
        _, r, d, _ = Z.step(leaf_idx=flats[t])
        if t >= t0:
            o, rr, dd = hist[t - t0 + 1]
            assert np.array_equal(_np(Z._obs).view(np.uint8), o.view(np.uint8)), "step %d" % t
            assert np.array_equal(_np(r), rr) and np.array_equal(_np(d).astype(bool), dd), "step %d" % t
    A.close(); Z.close()


# ---- (c) B = 1 is the plain item calls -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,cont", [(1, False), (2, False), (3, False), (1, True), (3, True)], ids=["d1", "d2", "d3", "c1", "c3"])
def test_b1_is_the_plain_item_calls(setting, cont):
    import pct_b200
    n, L = 32, 500
    c = _plain_cfg(setting, cont)
    st = _streams(n, setting, cont, L, 51)
    pool = _streams(4, setting, cont, 40, 53).reshape(-1, 4)
    A = _batch(c, list(st), 1)
    Q = pct_b200.PctBatch(n, setting, container_size=c["container"], continuous=cont, item_set=None if cont else ITEM_SET, obs_dtype=torch.float64,
                          item_stream=st, size_minimum=c["size_minimum"])
    A.reset(); Q.reset()
    rng = np.random.RandomState(setting)
    t_dev = torch.zeros((), dtype=torch.int64, device=A.device)
    for t in range(20):
        for k in (1, 3):
            assert torch.equal(A.buffer_preview_items(k), Q.preview_items(k + 1)[:, 1:]), (t, k)
        if t % 3 == 1:
            sel = np.sort(rng.permutation(n)[:rng.randint(1, n)])
            it = pool[rng.randint(len(pool), size=len(sel))].copy()
            if setting == 3:
                it[:, 3] = rng.uniform(0.05, 1.0, size=len(sel))
            ia, iq = torch.full((n, 8), SENT_INFO, dtype=torch.int32, device=A.device), torch.full((n, 8), SENT_INFO, dtype=torch.int32, device=A.device)
            A.buffer_set_items(torch.as_tensor(it[:, None], device=A.device), env_idx=sel, info=ia)
            Q.set_items(torch.as_tensor(it[:, :3]), env_idx=sel, density=it[:, 3], info=iq, whole_batch=False)
            assert torch.equal(ia, iq), t
            assert np.array_equal(_np(A._obs).view(np.uint8), _np(Q._obs).view(np.uint8)), t
        flat = A.random_policy_dev(PSEED, t_dev).clone()
        t_dev += 1
        _, ra, da, ia = A.step(leaf_idx=flat)
        _, rq, dq, iq = Q.step(leaf_idx=flat)
        assert np.array_equal(_np(A._obs).view(np.uint8), _np(Q._obs).view(np.uint8)), t
        assert torch.equal(ra, rq) and torch.equal(da, dq) and torch.equal(ia, iq), t
    A.close(); Q.close()


# ---- (d) untouched state, identity, snapshot round trip ------------------------------------------------------------------------------------
def _snap(P, env_idx=None):
    n = P.n_envs if env_idx is None else len(env_idx)
    out = torch.zeros((n, P.buffer_snapshot_bytes), dtype=torch.uint8, device=P.device)
    return _np(P.buffer_snapshot(env_idx=env_idx, out=out))


def _walk(P, steps, seed=PSEED):
    t_dev = torch.zeros((), dtype=torch.int64, device=P.device)
    for _ in range(steps):
        P.step(leaf_idx=P.random_policy_dev(seed, t_dev).clone())
        t_dev += 1


@pytest.mark.parametrize("setting,cont,B", [(1, False, 3), (2, False, 16), (3, True, 3), (2, True, 16)], ids=["d1-B3", "d2-B16", "c3-B3", "c2-B16"])
def test_untouched_state_and_identity(setting, cont, B):
    n = 64
    c = _plain_cfg(setting, cont, 64 if B == 16 else 50)
    P = _batch(c, list(_streams(n, setting, cont, 500, 61)), B, shuffle=True)
    P.reset()
    _walk(P, 7)
    obs0, items0, snap0 = _np(P._obs), _np(P.buffer_items()), _snap(P)
    # the identity, on every env: rows, records' sums and every snapshot byte unchanged
    info = torch.zeros((n, 8), dtype=torch.int32, device=P.device)
    P.buffer_set_items(P.buffer_items(), info=info)
    assert np.array_equal(_np(P._obs).view(np.uint8), obs0.view(np.uint8))
    assert np.array_equal(_snap(P), snap0)
    st = [P.state(e) for e in range(n)]
    inf = P.decode_info(info)
    assert [int(v) for v in inf["n_ems"]] == [s["n_ems"] for s in st] and [int(v) for v in inf["n_leaf"]] == [s["n_leaf"] for s in st]
    assert [int(v) for v in inf["flags"]] == [s["flags"] for s in st] and [int(v) for v in inf["counter"]] == [s["n_boxes"] for s in st]
    # a change on a subset: unlisted envs keep rows of `out`, records, buffers and snapshot bytes
    sel = np.arange(3, n, 5)
    rows = items0[sel].copy()
    rows[:, 0] = items0[(sel + 1) % n, B - 1]
    out = torch.full((n, P.obs_len), 7.25, dtype=P.obs_dtype, device=P.device)
    info.fill_(SENT_INFO)
    P.buffer_set_items(torch.as_tensor(rows, device=P.device), env_idx=sel, out=out, info=info)
    o, raw, items, snap = _np(out), _np(info), _np(P.buffer_items()), _snap(P)
    rest = np.setdiff1d(np.arange(n), sel)
    assert (o[rest] == 7.25).all() and (raw[rest] == SENT_INFO).all()
    assert np.array_equal(items[rest], items0[rest]) and np.array_equal(snap[rest], snap0[rest])
    assert np.array_equal(_np(P._obs).view(np.uint8), obs0.view(np.uint8)), "the batch's own buffer was not the call's output"
    assert np.array_equal(items[sel], rows) and not (o[sel] == 7.25).all(axis=1).any()
    # the rows written for the listed envs are the ones a restore of their records writes
    back = torch.zeros_like(out)
    P.buffer_restore(torch.as_tensor(snap, device=P.device), out=back)
    assert np.array_equal(_np(back)[sel].view(np.uint8), o[sel].view(np.uint8))
    P.close()


@pytest.mark.parametrize("setting,cont", [(1, False), (3, True)], ids=["d1", "c3"])
def test_snapshot_after_override_round_trip(setting, cont):
    """every env on one stream: env 0 overridden, snapshotted, restored into env 5 (and env 0 of a second batch); they continue bit-identically
    under the same flat indices"""
    n, B = 8, 3
    c = _plain_cfg(setting, cont)
    st = np.repeat(_streams(1, setting, cont, 500, 71), n, axis=0)
    P, Y = _batch(c, list(st), B), _batch(c, list(st), B)
    P.reset(); Y.reset()
    _walk(P, 5)
    rows = _np(P.buffer_items(env_idx=[0]))
    rows[0, 1] = _streams(1, setting, cont, 40, 73)[0, 17]
    P.buffer_set_items(torch.as_tensor(rows, device=P.device), env_idx=[0])
    rec = P.buffer_snapshot(env_idx=[0])
    P.buffer_restore(rec, env_idx=[5])
    Y.buffer_restore(rec, env_idx=[0])
    for t in range(25):
        o = _np(P._obs)
        assert np.array_equal(o[0].view(np.uint8), o[5].view(np.uint8)) and np.array_equal(o[0].view(np.uint8), _np(Y._obs)[0].view(np.uint8)), t
        assert np.array_equal(_snap(P, [0])[0], _snap(P, [5])[0]) and np.array_equal(_snap(P, [0])[0], _snap(Y, [0])[0]), t
        valid = np.nonzero(o[0, P.nb * 9:(P.nb + B * P.nl) * 9].reshape(-1, 9)[:, 8] == 1)[0]
        f = int(valid[t % len(valid)]) if len(valid) and t != 12 else -1  # -1 at t = 12: the zero action ends the episode
        flat = torch.full((n,), f, dtype=torch.int32, device=P.device)
        P.step(leaf_idx=flat); Y.step(leaf_idx=flat)
    P.close(); Y.close()


# ---- (e) the search example without mirrored streams --------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,cont", [(1, False), (2, False), (3, False), (1, True)], ids=["d1", "d2", "d3", "c1"])
def test_search_without_mirrored_streams(setting, cont):
    """one_ply_any_source, whose search batch draws from an unrelated stream, commits on every root what one_ply with a mirrored search
    batch commits: rows, buffered items, rewards and done, over many plies.  Children whose episode ended take the root's next B draws
    (no trajectory length is set), and invalid candidate indices make such children"""
    n, K, B = 16, 6, 3
    c = _plain_cfg(setting, cont)
    st = _streams(n, setting, cont, 700, 31)
    R1, R2 = _batch(c, list(st), B), _batch(c, list(st), B)
    S1 = _batch(c, list(np.repeat(st, K, axis=0)), B)
    S2 = _batch(c, list(_streams(n * K, setting, cont, 90, 97)), B)
    for X in (R1, R2, S1, S2):
        X.reset()
    gen = torch.Generator(device=R1.device)
    gen.manual_seed(5)
    ended = 0
    for t in range(40):
        flats = buffer_search.candidate_flats(R1._obs, R1.nb, R1.nl, B, K, gen)
        a = buffer_search.one_ply(R1, S1, flats)
        ended += int(_np(S1._done).sum())
        b = one_ply_any_source(R2, S2, flats)
        assert torch.equal(a, b), t
        assert np.array_equal(_np(R1._obs).view(np.uint8), _np(R2._obs).view(np.uint8)), t
        assert torch.equal(R1.buffer_items(), R2.buffer_items()), t
    assert ended > 0, "no child ended its episode"
    for X in (R1, R2, S1, S2):
        X.close()


# ---- (f) CUDA graphs -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,cont", [(1, False), (1, True)], ids=["d1", "c1"])
def test_graph_capture(setting, cont):
    """a captured loop of preview -> set the refilled-slot's successor into slot 0 of half the envs -> buffered step equals the eager loop"""
    n, B, T = 64, 3, 5
    c = _plain_cfg(setting, cont)
    st = list(_streams(n, setting, cont, 500, 81))
    G, E = _batch(c, st, B), _batch(c, st, B)
    G.reset(); E.reset()

    def make(X):
        return dict(t=torch.zeros((), dtype=torch.int64, device=X.device), sel=torch.arange(0, n, 2, device=X.device, dtype=torch.int32),
                    pv=torch.zeros((n, 2, 4), dtype=torch.float64, device=X.device), items=torch.zeros((n, B, 4), dtype=torch.float64, device=X.device),
                    obs=torch.zeros((T, n, X.obs_len), dtype=X.obs_dtype, device=X.device))

    def body(X, s):
        for t in range(T):
            X.buffer_preview_items(2, out=s["pv"])
            X.buffer_items(out=s["items"])
            s["items"][:, 0].copy_(s["pv"][:, 1])
            X.buffer_set_items(s["items"][s["sel"].long()], env_idx=s["sel"])
            X.step(leaf_idx=X.random_policy_dev(PSEED, s["t"]))
            s["obs"][t].copy_(X._obs)
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
        assert torch.equal(sg["obs"], se["obs"]) and torch.equal(sg["pv"], se["pv"]), rep
        assert np.array_equal(_snap(G), _snap(E)), rep
    G.close(); E.close()


# ---- (g) errors ----------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cont", [False, True], ids=["d", "c"])
def test_errors(cont):
    import pct_b200
    L = pct_b200._lib.lib()
    n, B = 8, 3
    c = _plain_cfg(1, cont)
    P = _batch(c, list(_streams(n, 1, cont, 200, 91)), B)
    h = P.h
    vp = lambda t: C.c_void_p(t.data_ptr())
    obs = torch.zeros((n, P.obs_len), dtype=torch.float64, device=P.device)
    out = torch.zeros((n, 4, 4), dtype=torch.float64, device=P.device)
    items = torch.zeros((n, B, 4), dtype=torch.float64, device=P.device)
    # before pct_buffer_reset
    assert L.pct_buffer_preview_items(h, None, n, 1, vp(out), None) == STATE
    assert L.pct_buffer_set_items(h, None, n, vp(items), vp(obs), None, None) == STATE
    with pytest.raises(pct_b200.PctError):
        P.buffer_preview_items()
    P.reset()
    assert L.pct_buffer_preview_items(h, None, -1, 1, vp(out), None) == INVALID
    assert L.pct_buffer_preview_items(h, None, n, 0, vp(out), None) == INVALID
    assert L.pct_buffer_preview_items(h, None, n, 1, None, None) == INVALID
    assert L.pct_buffer_preview_items(h, None, 1 << 29, 2, vp(out), None) == INVALID  # n * k * 4 past INT32_MAX
    assert L.pct_buffer_preview_items(h, None, 0, 1, None, None) == 0  # n == 0: a no-op
    assert L.pct_buffer_set_items(h, None, -1, vp(items), vp(obs), None, None) == INVALID
    assert L.pct_buffer_set_items(h, None, n, None, vp(obs), None, None) == INVALID
    assert L.pct_buffer_set_items(h, None, n, vp(items), None, None, None) == INVALID
    assert L.pct_buffer_set_items(h, None, (1 << 31) // 12 + 1, vp(items), vp(obs), None, None) == INVALID  # n * B * 4 past INT32_MAX
    assert L.pct_buffer_set_items(h, None, 0, None, None, None, None) == 0
    with pytest.raises(pct_b200.PctError):
        P.buffer_set_items(torch.zeros((n, B + 1, 4), dtype=torch.float64))
    with pytest.raises(pct_b200.PctError):
        P.buffer_set_items(torch.zeros((2, B, 4), dtype=torch.float64), env_idx=[0])
    with pytest.raises(pct_b200.PctError):
        P.buffer_preview_items(k=0)
    # out-of-range rows: zeros in the preview, skipped by the override
    before = _snap(P)
    idx = torch.tensor([-1, n, 2], dtype=torch.int32, device=P.device)
    pv = P.buffer_preview_items(2, env_idx=idx)
    assert (pv[:2] == 0).all() and torch.equal(pv[2], P.buffer_preview_items(2)[2])
    P.buffer_set_items(torch.full((2, B, 4), 3.0, dtype=torch.float64), env_idx=[-1, n])
    assert np.array_equal(_snap(P), before)
    torch.cuda.synchronize()
    P.close()
    Q = pct_b200.PctBatch(n, 1, container_size=c["container"], continuous=cont, item_set=None if cont else ITEM_SET,
                          item_stream=_streams(n, 1, cont, 200, 91), size_minimum=c["size_minimum"], obs_dtype=torch.float64)  # a plain handle
    Q.reset()
    assert L.pct_buffer_preview_items(Q.h, None, n, 1, vp(out), None) == STATE
    assert L.pct_buffer_set_items(Q.h, None, n, vp(items), vp(obs), None, None) == STATE
    with pytest.raises(pct_b200.PctError):
        Q.buffer_set_items(items)
    Q.close()
