"""GPU: the support graph every env carries between steps (supports, loads, stored polygons and split directions, alias entries;
canonical form: harness.compare_graphs) against per-env oracles, for every env after the reset and after every step, in lock-step under
injected item streams and the shared policy.  The other GPU parity tests compare what the policy sees; this compares the state the apply
kernel's stability descent writes and every later walk reads.  Each test prints how much it compared."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
from harness import (CASES, CONT_CASES, ITEM_SET, capacity_oracle, capacity_trace, case_stream, compare_graphs, cont_case_stream,  # noqa: E402
                     load_capacity_cases, make_stream, policy_pick)
from pct_oracle import OracleContinuous, OracleDiscrete, make_continuous_stream  # noqa: E402

pytestmark = pytest.mark.gpu
DIVERGING = [(False, 1, 126, 39), (False, 3, 92, 103), (True, 1, 597, 103)]  # (continuous, setting, env id, parting step); items 1234, policy 4321


class Lock(object):
    """a batch and one oracle per env in lock-step; every call compares observations and then every env's graph"""

    def __init__(self, cont, setting, streams, container=None, nb=80, nl=50, size_minimum=None, auto_reset=True, alias=True, pseed=5, gid=None,
                 make_oracle=None):
        import pct_b200
        self.n, self.nb, self.nl, self.pseed, self.auto, self.t = len(streams), nb, nl, pseed, auto_reset, 0
        self.gid = gid if gid is not None else list(range(self.n))
        container = container or ((1.0, 1.0, 1.0) if cont else (10, 10, 10))
        if size_minimum is None:
            size_minimum = 0.1 if cont else float(np.min(np.asarray(streams)[:, :, :3]))
        self.kw = dict(container_size=container, continuous=cont, internal_node_holder=nb, leaf_node_holder=nl, obs_dtype=torch.float64,
                       size_minimum=size_minimum, auto_reset=auto_reset)
        self.setting, self.streams = setting, np.stack(streams)
        self.gpu = pct_b200.PctBatch(self.n, setting, item_stream=self.streams, **self.kw)
        mk = make_oracle or (lambda s: (OracleContinuous if cont else OracleDiscrete)(setting, container_size=container, internal_node_holder=nb,
                                                                                     leaf_node_holder=nl, size_minimum=size_minimum, stream=s))
        self.orcs = [mk(s) for s in streams]
        for o in self.orcs:
            o.set_alias_mode(alias)
        self.tot = dict(pairs=0, loads=0, vertices=0, splits=0, own=0, failed_with_loads=0)

    def compare(self, what, gpu=None, envs=None):
        for e in (range(self.n) if envs is None else envs):
            r = self.orcs[e].support_graph()
            for k, v in compare_graphs((gpu or self.gpu).support_graph(e), r, "%s env %d:" % (what, e)).items():
                self.tot[k] += v
            self.tot["pairs"] += 1
            self.tot["failed_with_loads"] += int(r["failed_box"][0])

    def reset(self):
        self.o_ref = np.stack([o.reset() for o in self.orcs])
        o = self.gpu.reset().cpu().numpy()
        assert np.array_equal(o, self.o_ref), "reset"
        self.compare("reset")

    def step(self, compare=True):
        t = self.t
        picks = [policy_pick(self.o_ref[e], self.nb, self.nl, self.pseed, self.gid[e], t) for e in range(self.n)]
        res = [o.step(p[1]) for o, p in zip(self.orcs, picks)]
        ob, _, d, info = self.gpu.step(leaf_idx=torch.from_numpy(np.array([p[0] for p in picks], dtype=np.int32)).cuda())
        d_ref = np.array([r[2] for r in res])
        assert np.array_equal(d.cpu().numpy().astype(bool), d_ref), "step %d done" % t
        # the only flag a valid trajectory may raise: the box beyond a full holder (IndexError in the reference, error 1 in the oracle)
        assert np.array_equal(self.gpu.decode_info(info)["flags"], [int(r[3].get("error") == 1) for r in res]), "step %d flags" % t
        if not self.auto:  # the terminal observation and the graph the failed placement left behind
            assert np.array_equal(ob.cpu().numpy(), np.stack([r[0] for r in res])), "step %d" % t
            if compare:
                self.compare("step %d" % t)
            if d_ref.any():
                ob = self.gpu.reset(mask=torch.from_numpy(d_ref).cuda())
        self.o_ref = np.stack([o.reset() if r[2] else r[0] for o, r in zip(self.orcs, res)])
        bad = np.argwhere(ob.cpu().numpy() != self.o_ref)
        assert len(bad) == 0, "step %d: observation of env %d" % (t, bad[0][0])
        if compare:
            self.compare("after step %d" % t)
        self.t += 1

    def run(self, steps):
        for _ in range(steps):
            self.step()
        return self

    def done(self, what, loads=1, vertices=1):
        print("%s: compared %s" % (what, self.tot))
        assert self.tot["pairs"] > 0 and self.tot["loads"] >= loads and self.tot["vertices"] >= vertices, self.tot
        self.gpu.close()


def _streams(cont, setting, n, seed, length=300):
    return [(make_continuous_stream if cont else make_stream)(seed, e, length, setting) for e in range(n)]


@pytest.mark.parametrize("auto_reset", [True, False], ids=["auto_reset", "gym"])
@pytest.mark.parametrize("cont", [False, True], ids=["discrete", "continuous"])
@pytest.mark.parametrize("setting", [1, 2, 3])
def test_graph_lockstep(setting, cont, auto_reset):
    k = Lock(cont, setting, _streams(cont, setting, 16, 31 + setting), auto_reset=auto_reset)
    k.reset()
    k.run(100)
    k.done("setting %d" % setting, *((2000, 500) if setting != 2 else (0, 0)))
    assert (k.tot["own"] > 0) == (setting != 2)


@pytest.mark.parametrize("name", ["big_s1", "big_s3", "dense16_s1", "flat_s1", "holders_s1", "c:box2_s1", "c:box2_s3", "c:holders_s1"])
def test_graph_on_other_configurations(name):
    """dense16_s1 fills its 80-box holder: the 81st real placement must leave the load list of box 0 alone"""
    cont = name.startswith("c:")
    c = (CONT_CASES if cont else CASES)[name[2:] if cont else name]
    mk = cont_case_stream if cont else case_stream
    k = Lock(cont, c["setting"], [mk(c, 91, e, 400) for e in range(8)], container=c["container"], nb=c["nb"], nl=c["nl"],
             size_minimum=c["low"] if cont else min(min(i) for i in c["items"]), auto_reset=False, pseed=91)
    k.reset()
    k.run(c["steps"] + 30)
    k.done(name, 1000, 300)


@pytest.mark.parametrize("name", ["d_box80_s1", "c_box80_s1"])
def test_graph_with_a_full_holder(name):
    """the capacity cases that fill the box holder (where n_edge and n_poly are largest), up to, not past, their flagged step"""
    c = load_capacity_cases()[name]
    tr = capacity_trace(c)
    steps = tr["t_star"] if tr["t_star"] >= 0 else tr["n_steps"]
    cont = c["domain"] == "continuous"
    k = Lock(cont, c["setting"], [c["stream"]], container=c["container"], nb=c["nb"], nl=c["nl"], size_minimum=c["size_minimum"], auto_reset=False,
             pseed=c["pseed"], gid=[0], make_oracle=lambda s: capacity_oracle(c))
    k.reset()
    k.run(steps)
    g = k.gpu.support_graph(0)
    print("%s: n_box %d n_edge %d n_poly %d after %d steps" % (name, g["n_box"], g["n_edge"], g["n_poly"], steps))
    assert g["n_box"] >= 60
    k.done(name, 1000, 300)


@pytest.mark.parametrize("cont", [False, True], ids=["discrete", "continuous"])
@pytest.mark.parametrize("setting", [1, 3])
def test_graph_of_a_box_on_sixteen_supports(setting, cont):
    """a 4 x 4 floor of unit boxes (0.1-cubes), then a 4 x 4 (0.4 x 0.4) item on all of them, its centre on the common corner of the middle
    four: 16 loads written by one descent through the lstsq split and the per-env scratch"""
    u = 0.1 if cont else 1
    seq = np.array([[u, u, u, 0.5]] * 16 + [[4 * u, 4 * u, u, 0.7]] + [[2 * u, 2 * u, u, 0.9]] * 6)
    if setting != 3:
        seq[:, 3] = 1.0
    k = Lock(cont, setting, [seq], auto_reset=False, size_minimum=u)
    k.reset()
    acts = [(round(x * u, 1), round(y * u, 1)) for x in range(4) for y in range(4)] + [(0, 0)]
    for i, (lx, ly) in enumerate(acts):
        s = seq[i]
        row = np.array([lx, ly, 0, lx + s[0], ly + s[1], 0, 0, 0, 1], dtype=np.float64)
        row[2] = u if i == 16 else 0
        o_ref, _, d_ref, _ = k.orcs[0].step(row)
        ob, _, d, info = k.gpu.step(actions=torch.from_numpy(row[None]).cuda())
        assert not d_ref and not bool(d.cpu().numpy()[0]) and not k.gpu.decode_info(info)["flags"].any(), i
        assert np.array_equal(ob.cpu().numpy()[0], o_ref), i
        k.compare("placement %d" % i)
    g = k.gpu.support_graph(0)
    assert len(g["supports"][16]) == 16 and all(g["load_upper"][b] == [16] for b in range(16)) and k.orcs[0].n_lstsq > 0
    k.done("16 supports", 16, 4)


@pytest.mark.parametrize("cont,setting,env_id,step", DIVERGING)
@pytest.mark.parametrize("alias", [None, "0"], ids=["alias", "snapshot"])
def test_graph_through_the_parting_steps(cont, setting, env_id, step, alias, monkeypatch):
    """each apply kernel against the oracle of its own semantics, through and past the step at which the two semantics part"""
    if alias is None:
        monkeypatch.delenv("PCT_B200_ALIAS", raising=False)
    else:
        monkeypatch.setenv("PCT_B200_ALIAS", alias)
    s = (make_continuous_stream if cont else make_stream)(1234, env_id, 600, setting)
    k = Lock(cont, setting, [s], auto_reset=False, alias=alias is None, pseed=4321, gid=[env_id], size_minimum=0.1 if cont else 1)
    k.reset()
    k.run(step + 20)
    assert k.gpu.support_graph(0)["alias"] == (alias is None)
    k.done("parting trajectory", 300, 100)


@pytest.mark.parametrize("var,val", [("PCT_B200_WALK", "fork"), ("PCT_B200_LPT", "0"), ("PCT_B200_K3", "block")])
@pytest.mark.parametrize("cont", [False, True], ids=["discrete", "continuous"])
def test_launch_variants_leave_the_graph_alone(cont, var, val, monkeypatch):
    monkeypatch.setenv(var, val)
    k = Lock(cont, 1, _streams(cont, 1, 16, 47))
    k.reset()
    k.run(60)
    k.done("%s=%s" % (var, val), 1000, 300)


@pytest.mark.parametrize("cont", [False, True], ids=["discrete", "continuous"])
@pytest.mark.parametrize("setting", [1, 3])
def test_state_moving_calls(setting, cont):
    """snapshot -> restore into another slot (over richer stale state) and into another handle, reset of chosen envs, set_items and the
    read-only queries: after each the graphs are the oracle's, and 20 more lock-step steps follow"""
    import pct_b200
    n = 8
    streams = _streams(cont, setting, n, 61 + setting)
    k = Lock(cont, setting, streams, auto_reset=False)
    k.reset()
    k.run(25)
    # read-only calls run the stability routine on the same records
    k.gpu.preview_items(3)
    if cont:
        q = torch.tensor([[[0.2, 0.2, 0.2, 0.0, 0.0], [0.1, 0.3, 0.1, 0.3, 0.3]]] * n, dtype=torch.float64, device="cuda")
    else:
        q = torch.tensor([[[2, 2, 2, 0, 0], [1, 3, 1, 3, 3]]] * n, dtype=torch.int32, device="cuda")
        k.gpu.height_maps()
    k.gpu.query_placements(q)
    k.gpu.heuristic_actions("LSAH")
    k.compare("after the read-only calls")
    # set_items with each env's own current item: every env is re-expanded, the graph stays
    k.gpu.set_items(torch.tensor(np.array([o.next_box for o in k.orcs]), dtype=torch.float64 if cont else torch.int32, device="cuda"))
    k.compare("after set_items")
    k.run(3)
    # snapshot of every env; env 0's record goes over the (different, possibly richer) state of slot 1 and into a fresh handle
    snap = k.gpu.snapshot()
    other = pct_b200.PctBatch(n, setting, item_stream=k.streams, **k.kw)
    other.reset()
    other.restore(snap)
    k.compare("restored into another handle", gpu=other)
    other.close()
    k.gpu.restore(snap, env_idx=[1], rec_idx=[0])
    want = k.orcs[0].support_graph()
    compare_graphs(k.gpu.support_graph(1), want, "slot 1 <- record of env 0:")
    k.gpu.restore(snap, env_idx=[1], rec_idx=[1])
    k.compare("restored back")
    # reset of chosen envs: by index list, then by mask; the others untouched
    k.gpu.reset(env_idx=[2, 5])
    for e in (2, 5):
        k.o_ref[e] = k.orcs[e].reset()
    k.compare("after reset(env_idx)")
    m = np.zeros(n, dtype=bool)
    m[[0, 7]] = True
    ob = k.gpu.reset(mask=torch.from_numpy(m).cuda())
    for e in (0, 7):
        k.o_ref[e] = k.orcs[e].reset()
    assert np.array_equal(ob.cpu().numpy(), k.o_ref)
    k.compare("after reset(mask)")
    assert all(k.gpu.support_graph(e)["n_edge"] == 0 for e in (0, 7))
    k.run(20)
    k.done("state-moving calls", 1000, 300)


@pytest.mark.parametrize("cont", [False, True], ids=["discrete", "continuous"])
def test_structure_of_every_graph_at_full_size(cont):
    """4096 envs, 120 steps of the random policy, then every env decoded: the decoder accepts a record only if its CSR offsets are
    monotone and end at n_edge, every edge below n_edge is in exactly one load list, each list is acyclic, in insertion order and ends
    at last_in, every support is an earlier box and (alias mode) e_upper agrees with the CSR; here also: finite loads, object entries
    equal to the upper box's own stack."""
    import pct_b200
    n = 4096
    kw = dict(container_size=(1.0, 1.0, 1.0), continuous=True, sample_from_distribution=True) if cont else dict(item_set=ITEM_SET)
    gpu = pct_b200.PctBatch(n, 1, seed=1234, **kw)
    gpu.reset()
    for t in range(120):
        _, _, _, info = gpu.step(leaf_idx=gpu.random_policy(4321, t))
    assert not gpu.decode_info(info)["flags"].any()
    edges = boxes = stale = 0
    for e in range(n):
        g = gpu.support_graph(e)  # raises PctError with the finding if a list is broken
        edges += g["n_edge"]
        boxes += g["n_box"]
        stale += g["alias_stale"]
        for u in range(g["n_box"]):
            assert np.isfinite(g["loads"][u]).all(), (e, u)
            for i, (up, al) in enumerate(zip(g["load_upper"][u], g["load_alias"][u])):
                if al and up < g["n_box"]:
                    assert np.array_equal(g["loads"][u][i].view(np.uint64), g["own_stack"][up].view(np.uint64)), (e, u, i)
    print("decoded %d envs: %d boxes, %d edges, %d stale alias bits" % (n, boxes, edges, stale))
    assert edges > 4 * n
    gpu.close()
