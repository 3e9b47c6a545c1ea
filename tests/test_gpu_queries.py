"""GPU: batched placement queries and height maps (pct_query_placements(_f64) / pct_height_maps, PctBatch.query_placements / height_maps).

Answers are checked bit for bit against the oracle's Space.drop_box_virtual / Space.plain and against the single-query path, on
batches stepped in lock-step with the oracle by the random leaf policy.  Queries must leave every env exactly as it was.
"""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
from harness import CASES, ITEM_SET, OracleDiscrete, case_stream, make_stream, policy_pick  # noqa: E402
from pct_oracle import OracleContinuous, make_continuous_stream  # noqa: E402
from query_compose import composed_rows  # noqa: E402

pytestmark = pytest.mark.gpu
PSEED = 4321
DOMAINS = [(s, False) for s in (1, 2, 3)] + [(s, True) for s in (1, 2, 3)]
DOM_IDS = ["d%d" % s if not c else "c%d" % s for s, c in DOMAINS]
PERMS = ((0, 1, 2), (1, 0, 2), (1, 2, 0), (2, 1, 0), (0, 2, 1), (2, 0, 1))
BIG40 = dict(setting=1, container=(40, 36, 30), items=[(i, j, k) for i in (3, 7, 12) for j in (4, 9) for k in (3, 8, 11)], nb=80, nl=50)


def _pb():
    import pct_b200
    return pct_b200


class Lockstep(object):
    """a PctBatch driven by per-env item streams and the oracle envs with the same streams, stepped together by the random leaf policy"""

    def __init__(self, n, setting, continuous, case=None, seed=11, length=600):
        pct_b200 = _pb()
        self.n, self.continuous, self.t = n, continuous, 0
        if continuous:
            self.container, items, self.nb, self.nl = (1.0, 1.0, 1.0), None, 80, 50
            streams = np.stack([make_continuous_stream(seed, e, length, setting) for e in range(n)])
            self.b = pct_b200.PctBatch(n, setting, container_size=self.container, continuous=True, obs_dtype=torch.float64, item_stream=streams,
                                       size_minimum=0.1)
            self.o = [OracleContinuous(setting, stream=streams[e]) for e in range(n)]
        else:
            c = case or dict(setting=setting, container=(10, 10, 10), items=ITEM_SET, nb=80, nl=50)
            self.container, items, self.nb, self.nl = tuple(c["container"]), c["items"], c["nb"], c["nl"]
            streams = np.stack([(case_stream(c, seed, e, length) if case else make_stream(seed, e, length, setting)) for e in range(n)])
            self.b = pct_b200.PctBatch(n, setting, container_size=self.container, item_set=items, internal_node_holder=self.nb,
                                       leaf_node_holder=self.nl, obs_dtype=torch.float64, item_stream=streams)
            self.o = [OracleDiscrete(setting, container_size=self.container, internal_node_holder=self.nb, leaf_node_holder=self.nl,
                                     stream=streams[e]) for e in range(n)]
        self.items = items
        self.obs = self.b.reset().cpu().numpy().copy()
        ref = np.stack([o.reset() for o in self.o])
        assert np.array_equal(self.obs, ref), "reset observations differ from the oracle"

    def step(self):
        idx = self.b.random_policy(PSEED, self.t)
        obs, _, done, _ = self.b.step(leaf_idx=idx)
        for e, o in enumerate(self.o):
            _, row = policy_pick(self.obs[e], self.nb, self.nl, PSEED, e, self.t)
            _, _, d, _ = o.step(row)
            if d:
                o.reset()
        self.t += 1
        self.obs = obs.cpu().numpy().copy()
        return done.cpu().numpy().astype(bool)

    def leaves(self, e):
        rows = self.obs[e].reshape(-1, 9)[self.nb:self.nb + self.nl]
        return rows[rows[:, 8] == 1]

    def close(self):
        self.b.close()


def _orient(nb, row, continuous):
    """LeafNode2Action: the oriented sizes of a leaf row (the item entries matching its x and y extents, z the remaining one)"""
    rest = list(nb)
    out = []
    for ext in (row[3] - row[0], row[4] - row[1]):
        i = int(np.argmin([abs(v - ext) for v in rest]))
        out.append(rest.pop(i))
    return out + rest


def _queries(ls, e, rng, k=96):
    """k placements for env e: its leaf rows, zero sizes, over-tall items, and random positions over [-1, W] x [-1, L] with rotated item sizes"""
    o = ls.o[e]
    nb = o.next_box
    W, L, H = ls.container
    q = []
    for row in ls.leaves(e)[:40]:
        q.append(_orient(nb, row, ls.continuous) + [row[0], row[1]])
    if ls.continuous:
        for row in ls.leaves(e)[:6]:  # the 1e-6 tolerances of the bounds tests
            d = _orient(nb, row, True)
            q.append(d + [row[0] - 5e-7, row[1]])
            q.append(d + [W - d[0] + 5e-7, row[1]])
            q.append(d + [row[0], L - d[1] + 2e-6])
        size = lambda: [round(v, 3) for v in rng.uniform(0.05, 0.6, 3)]
        pos = lambda: [round(rng.uniform(-0.1, W + 0.05), 3), round(rng.uniform(-0.1, L + 0.05), 3)]
    else:
        size = lambda: [ls.items[rng.integers(len(ls.items))][i] for i in PERMS[rng.integers(6)]]
        pos = lambda: [int(rng.integers(-1, W + 1)), int(rng.integers(-1, L + 1))]
    for _ in range(3):
        s = size()
        q.append([0, s[1], s[2]] + pos())
        q.append([s[0], 0, s[2]] + pos())
    for _ in range(4):
        s = size()
        q.append([s[0], s[1], H + (0.25 if ls.continuous else 1)] + pos())
    while len(q) < k:
        q.append(size() + pos())
    return q[:k]


def _answer(b, q, **kw):
    f, h = b.query_placements(torch.as_tensor(np.asarray(q)), **kw)
    return f.cpu().numpy(), h.cpu().numpy()


# ---- 1. against the oracle ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", DOMAINS, ids=DOM_IDS)
def test_queries_equal_the_oracle(setting, continuous):
    ls = Lockstep(96, setting, continuous)
    rng = np.random.default_rng(setting + 10 * continuous)
    before_done = checked = 0
    for t in range(70):
        if t % 5 == 0:
            q = [_queries(ls, e, rng) for e in range(ls.n)]
            f, h = _answer(ls.b, q)
            assert f.dtype == np.bool_ and h.dtype == (np.float64 if continuous else np.int32)
            for e in range(ls.n):
                for j, x in enumerate(q[e]):
                    ok, mh = ls.o[e].drop_box_virtual(x[:3], x[3], x[4])
                    assert (bool(f[e, j]), h[e, j]) == (ok, mh), "env %d query %d %s at step %d: got %s, oracle %s" % (e, j, x, t, (f[e, j], h[e, j]), (ok, mh))
            checked += 1
            assert f.any() and not f.all()
        done = ls.step()
        if t % 5 == 0:
            before_done += int(done.sum())
    assert before_done > 0, "no sampled state was the step before a done"
    ls.close()


# ---- 2. against the single query ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", DOMAINS, ids=DOM_IDS)
def test_queries_equal_the_single_query(setting, continuous):
    ls = Lockstep(64, setting, continuous, seed=23)
    rng = np.random.default_rng(7)
    for _ in range(25):
        ls.step()
    q = np.asarray([_queries(ls, e, rng) for e in range(ls.n)])
    den = rng.uniform(0.2, 3.0, size=q.shape[:2]) if setting == 3 else None
    f, h = _answer(ls.b, q, density=den)
    for e in range(0, ls.n, 3):
        for j in range(0, q.shape[1], 5):
            d = float(den[e, j]) if den is not None else ls.o[e].next_den
            x = q[e, j]
            ok, mh = ls.b.query_placement(e, x[:3], x[3], x[4], density=d)
            assert (bool(f[e, j]), h[e, j]) == (ok, mh), (e, j, x)
    ls.close()


# ---- 3. leaf rows ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", DOMAINS, ids=DOM_IDS)
def test_leaf_rows_are_feasible(setting, continuous):
    """Every valid leaf row is feasible.  Its rest height is at most the leaf's z (an EMS corner can lie above the height map under the
    footprint: the box drops), and it is the z at which the step places the box of the chosen leaf."""
    ls = Lockstep(128, setting, continuous, seed=31)
    for t in range(40):
        nbx = [ls.o[e].packed for e in range(ls.n)]
        leaves = [ls.leaves(e) for e in range(ls.n)]
        k = max(len(x) for x in leaves)
        q = np.zeros((ls.n, k, 5))
        q[:, :, 3] = -1  # padding: an infeasible position
        for e in range(ls.n):
            for j, row in enumerate(leaves[e]):
                q[e, j] = _orient(ls.o[e].next_box, row, continuous) + [row[0], row[1]]
        f, h = _answer(ls.b, q)
        pick = [policy_pick(ls.obs[e], ls.nb, ls.nl, PSEED, e, t)[0] for e in range(ls.n)]
        done = ls.step()
        for e in range(ls.n):
            m = len(leaves[e])
            assert f[e, :m].all(), "env %d step %d: a leaf row is infeasible" % (e, t)
            assert (h[e, :m] <= leaves[e][:, 2] + (1e-9 if continuous else 0)).all()
            if m and not done[e]:
                placed = ls.obs[e].reshape(-1, 9)[len(nbx[e])]
                assert placed[2] == h[e, pick[e]], "env %d step %d: placed at z %s, query said %s" % (e, t, placed[2], h[e, pick[e]])
    ls.close()


# ---- 4. height maps -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["default", "big_s1", "big40"])
def test_height_maps_equal_the_oracle(which):
    case = {"default": None, "big_s1": CASES["big_s1"], "big40": BIG40}[which]
    ls = Lockstep(64, 1, False, case=case, seed=41, length=1500)
    W, L = ls.container[:2]
    for t in range(120):
        if t % 10 == 0:
            hm = ls.b.height_maps().cpu().numpy()
            assert hm.shape == (ls.n, W, L) and hm.dtype == np.int32
            for e in range(ls.n):
                assert np.array_equal(hm[e], ls.o[e].plain()), "env %d step %d" % (e, t)
            sub = ls.b.height_maps(env_idx=[5, 0, 63]).cpu().numpy()
            assert np.array_equal(sub, hm[[5, 0, 63]])
        ls.step()
    assert hm.any()
    if which == "big40":  # a bin the single discrete query refuses; the batched one answers it
        q = [_queries(ls, e, np.random.default_rng(e)) for e in range(ls.n)]
        f, h = _answer(ls.b, q)
        for e in range(0, ls.n, 4):
            for j, x in enumerate(q[e]):
                assert (bool(f[e, j]), h[e, j]) == ls.o[e].drop_box_virtual(x[:3], x[3], x[4])
        with pytest.raises(_pb().PctError, match="sides <= 32"):
            ls.b.query_placement(0, (3, 4, 3), 0, 0)
    ls.close()


# ---- 5. read-only ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting,continuous", DOMAINS, ids=DOM_IDS)
def test_queries_leave_the_envs_unchanged(setting, continuous):
    a = Lockstep(64, setting, continuous, seed=53)
    b = Lockstep(64, setting, continuous, seed=53)
    rng = np.random.default_rng(3)
    for _ in range(30):
        a.step()
        b.step()
    s0 = a.b.snapshot().cpu().numpy()
    obs0 = a.b._obs.clone()
    q = np.asarray([_queries(a, e, rng, k=300) for e in range(a.n)])
    _answer(a.b, q)
    _answer(a.b, q[::-1].copy(), env_idx=np.arange(a.n)[::-1].copy())
    if not continuous:
        a.b.height_maps()
    torch.cuda.synchronize()
    assert np.array_equal(a.b.snapshot().cpu().numpy(), s0), "a query changed an env record"
    assert torch.equal(a.b._obs, obs0)
    for t in range(2):
        idx = a.b.random_policy(9, t).clone()
        ra = [x.cpu().numpy().copy() for x in a.b.step(leaf_idx=idx)]
        rb = [x.cpu().numpy().copy() for x in b.b.step(leaf_idx=idx)]
        for u, v, nm in zip(ra, rb, ("obs", "reward", "done", "info")):
            assert np.array_equal(u, v), "step %d after the queries: %s" % (t, nm)
    a.close()
    b.close()


# ---- 6. graph capture ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("continuous", [False, True], ids=["discrete", "continuous"])
def test_queries_in_a_cuda_graph(continuous):
    a = Lockstep(128, 1, continuous, seed=61)
    b = Lockstep(128, 1, continuous, seed=61)
    rng = np.random.default_rng(5)
    for _ in range(10):
        a.step()
        b.step()
    qd = torch.float64 if continuous else torch.int32
    q = torch.as_tensor(np.asarray([_queries(a, e, rng, k=130) for e in range(a.n)]), dtype=qd, device=a.b.device)
    n, k = q.shape[:2]
    f = torch.zeros((n, k), dtype=torch.bool, device=a.b.device)
    h = torch.zeros((n, k), dtype=qd, device=a.b.device)
    hm = torch.zeros((n, 10, 10), dtype=torch.int32, device=a.b.device)
    idx = torch.zeros(n, dtype=torch.int32, device=a.b.device)
    obs = torch.zeros_like(a.b._obs)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        a.b.query_placements(q, out=(f, h))
        if not continuous:
            a.b.height_maps(out=hm)
        a.b.random_policy(7, 3, out=idx)
        res = a.b.step(leaf_idx=idx, out=obs)
    for rep in range(3):
        graph.replay()
        torch.cuda.synchronize()
        ef, eh = b.b.query_placements(q)
        assert torch.equal(f, ef) and torch.equal(h, eh), "replay %d: queries" % rep
        if not continuous:
            assert torch.equal(hm, b.b.height_maps()), "replay %d: height maps" % rep
        er = b.b.step(leaf_idx=b.b.random_policy(7, 3))
        for u, v, nm in zip(res, er, ("obs", "reward", "done", "info")):
            assert torch.equal(u, v), "replay %d: %s" % (rep, nm)
    a.close()
    b.close()


# ---- 7. DBL / HM composed in torch on the two calls ------------------------------------------------------------------------------------
def _next_boxes(b):
    from pct_b200 import _lib
    d = _lib.StateDump()
    out = np.zeros((b.n_envs, 3), dtype=np.int64)
    for e in range(b.n_envs):
        assert b.L.pct_get_state(b.h, e, C.byref(d)) == 0
        out[e] = d.next_box[:3]
    return torch.from_numpy(out).to(b.device)


@pytest.mark.parametrize("name", ["DBL", "HM"])
@pytest.mark.parametrize("setting", [1, 2, 3])
def test_composed_heuristics_equal_the_builtin(name, setting):
    b = _pb().PctBatch(256, setting, item_set=ITEM_SET, seed=77)
    b.reset()
    episodes = np.zeros(256, dtype=np.int64)
    t = 0
    while (episodes < 2).any():
        mine = composed_rows(b, name, _next_boxes(b))
        ref = b.heuristic_actions(name)
        if not torch.equal(mine, ref):
            bad = int(torch.nonzero((mine != ref).any(1))[0])
            raise AssertionError("step %d env %d: composed %s, built-in %s" % (t, bad, mine[bad].tolist(), ref[bad].tolist()))
        _, _, done, _ = b.step(actions=ref)
        episodes += done.cpu().numpy().astype(np.int64)
        t += 1
        assert t < 1000
    b.close()


# ---- 8. errors and edges ------------------------------------------------------------------------------------------------------------------
def test_errors_and_edges():
    pct_b200 = _pb()
    PctError = pct_b200.PctError
    d = pct_b200.PctBatch(8, 1, item_set=ITEM_SET, seed=1)
    c = pct_b200.PctBatch(8, 1, container_size=(1.0, 1.0, 1.0), continuous=True, sample_from_distribution=True, seed=1)
    qi = torch.ones((8, 4, 5), dtype=torch.int32)
    with pytest.raises(PctError, match="before pct_reset"):
        d.query_placements(qi)
    with pytest.raises(PctError, match="before pct_reset"):
        d.height_maps()
    d.reset()
    c.reset()
    with pytest.raises(PctError, match="no height map"):
        c.height_maps()
    L = d.L
    assert L.pct_query_placements(c.h, None, 1, 1, None, None, None, None, None) == -1
    assert L.pct_query_placements_f64(d.h, None, 1, 1, None, None, None, None, None) == -1
    assert L.pct_height_maps(c.h, None, 1, None, None) == -1
    assert L.pct_query_placements(d.h, None, -1, 1, None, None, None, None, None) == -1
    assert L.pct_query_placements(d.h, None, 1, -1, None, None, None, None, None) == -1
    assert L.pct_query_placements(d.h, None, 65536, 65536, None, None, None, None, None) == -1
    assert "overflows" in L.pct_last_error(d.h).decode()
    assert L.pct_height_maps(d.h, None, -1, None, None) == -1
    for bad in (torch.ones((8, 4), dtype=torch.int32), torch.ones((8, 4, 4), dtype=torch.int32)):
        with pytest.raises(PctError, match="shape"):
            d.query_placements(bad)
    with pytest.raises(PctError, match="density"):
        d.query_placements(qi, density=torch.ones(8, 3))
    with pytest.raises(PctError, match="env_idx"):
        d.query_placements(qi, env_idx=[0, 1])
    with pytest.raises(PctError, match="out"):
        d.query_placements(qi, out=(torch.zeros((8, 4), dtype=torch.uint8, device=d.device), torch.zeros((8, 4), dtype=torch.int32, device=d.device)))
    with pytest.raises(PctError, match="out"):
        d.height_maps(out=torch.zeros((8, 10, 9), dtype=torch.int32, device=d.device))
    # n == 0 / k == 0: no-ops
    launches = d.kernel_launches
    f, h = d.query_placements(torch.zeros((0, 4, 5), dtype=torch.int32))
    assert f.shape == (0, 4) and h.shape == (0, 4)
    f, h = d.query_placements(torch.zeros((8, 0, 5), dtype=torch.int32))
    assert f.shape == (8, 0)
    assert d.height_maps(env_idx=[]).shape == (0, 10, 10)
    assert L.pct_query_placements(d.h, None, 0, 0, None, None, None, None, None) == 0
    assert L.pct_height_maps(d.h, None, 0, None, None) == 0
    assert d.kernel_launches == launches
    # out-of-range rows: infeasible / 0 and zero maps; the other rows are answered as usual
    for _ in range(6):
        d.step(leaf_idx=d.random_policy(3, _))
    q = torch.tensor([[[2, 2, 2, 0, 0], [1, 1, 1, 3, 4], [3, 2, 1, 8, 0]]] * 4, dtype=torch.int32)
    want_f, want_h = d.query_placements(q[:2], env_idx=[0, 5])
    f = torch.ones((4, 3), dtype=torch.bool, device=d.device)
    h = torch.full((4, 3), 77, dtype=torch.int32, device=d.device)
    d.query_placements(q, env_idx=[-1, 0, 8, 5], out=(f, h))
    assert not f[[0, 2]].any() and not h[[0, 2]].any()
    assert torch.equal(f[[1, 3]], want_f) and torch.equal(h[[1, 3]], want_h)
    cq = torch.tensor([[[0.2, 0.3, 0.2, 0.0, 0.0]]] * 2, dtype=torch.float64)
    cf, ch = c.query_placements(cq, env_idx=[9, 1])
    assert not cf[0].any() and ch[0, 0] == 0 and bool(cf[1, 0])
    hm = d.height_maps(env_idx=[100, 2])
    assert not hm[0].any() and torch.equal(hm[1], d.height_maps()[2])
    torch.cuda.synchronize()
    d.close()
    c.close()
