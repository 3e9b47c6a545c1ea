"""CPU: the support graph an env carries from step to step (supports, loads, stored polygons, alias entries: harness.compare_graphs
defines the canonical form) compared after EVERY real placement between the oracle's objects and the pools the device stability routine
writes, through the host build of the device sources (tests/host_emul/stab_host.cpp) and the decoder the C ABI runs on device records
(csrc/pct_support_graph.h).  Observations compare what the policy sees; this compares the state that decides later feasibility."""
import ctypes as C

import numpy as np
import pytest

from harness import CASES, CONT_CASES, case_stream, compare_graphs, cont_case_stream, make_stream, policy_pick
from pct_oracle import OracleContinuous, OracleDiscrete, make_continuous_stream
from test_host_emul_stability import DIVERGING, DIVERGING_C, _placement, lib  # noqa: F401  (lib: the host build, a fixture)


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


class Host(object):
    """one env of the host build, discrete or continuous, behind the three calls the drivers need"""

    def __init__(self, L, cont, setting, container, nb, alias):
        self.L, self.cont, self.p = L, cont, "shc_" if cont else "sh_"
        self.h = (L.shc_create(setting, *[float(c) for c in container]) if cont else L.sh_create(setting, *[int(c) for c in container]))
        getattr(L, self.p + "set_holder").argtypes = [C.c_void_p, C.c_int]
        getattr(L, self.p + "set_holder")(self.h, nb)
        getattr(L, self.p + "set_alias")(self.h, int(alias))
        self.reset()

    def reset(self):
        getattr(self.L, self.p + "reset")(self.h)

    def place(self, row, next_box, den):
        if self.cont:
            return self.L.shc_place_row(self.h, _dp(np.ascontiguousarray(row[:6], dtype=np.float64)), _dp(np.array(next_box, dtype=np.float64)), den)
        (x, y, z), lx, ly = _placement(row, next_box)
        return self.L.sh_place(self.h, x, y, z, lx, ly, den)

    def graph(self):
        from pct_b200 import _lib
        d, err = _lib.SupportGraph(), C.create_string_buffer(256)
        ok = getattr(self.L, self.p + "support_graph")(self.h, C.byref(d), err, 256)
        assert ok, "decoder: " + err.value.decode()
        return _lib.graph_to_dict(d)

    def field(self, which):
        return getattr(self.L, self.p + "pool_field")(self.h, which)

    def close(self):
        getattr(self.L, self.p + "destroy")(self.h)


def _run(L, env, cont, setting, container, nb, nl, seed, env_id, steps, alias, fail_from=None):
    """lock-step of the oracle env and the host build under the shared policy, graphs compared after the reset and after every real
    placement (a failed one included, before the reset that follows it).  fail_from: once the bin holds that many boxes the policy picks the
    highest candidate the oracle found unstable instead, so that the real placement fails.  -> totals"""
    host = Host(L, cont, setting, container, nb, alias)
    env.set_alias_mode(alias)
    o = env.reset()
    tot = dict(pairs=0, loads=0, vertices=0, splits=0, own=0, failed=0, failed_with_loads=0, stale=0)
    compare_graphs(host.graph(), env.support_graph(), "after reset:")
    for t in range(steps):
        _, row = policy_pick(o, nb, nl, seed, env_id, t)
        if fail_from is not None and len(env.packed) >= fail_from:
            cand, feas = env.candidates()
            bad = [p for p, f in zip(cand, feas) if f == 0 and p[2] > 0]
            if bad:
                row = np.array(list(max(bad, key=lambda p: p[2])[:5]) + [container[2], 0, 0, 1], dtype=np.float64)
        nbx, den = env.next_box, env.next_den
        o, _, done, _ = env.step(row)
        placed = host.place(row, nbx, den)
        assert placed == (not done), "step %d real placement: host build %d, oracle done=%s" % (t, placed, done)
        g, r = host.graph(), env.support_graph()
        for k, v in compare_graphs(g, r, "step %d:" % t).items():
            tot[k] += v
        tot["pairs"] += 1
        tot["failed"] += int(done)
        tot["failed_with_loads"] += int(r["failed_box"][0])
        tot["stale"] = max(tot["stale"], g["alias_stale"])
        if done:
            o = env.reset()
            host.reset()
    host.close()
    return tot


def _oracle(cont, setting, seed, env_id, n=700, case=None):
    if case is not None and cont:
        return OracleContinuous(setting, container_size=case["container"], internal_node_holder=case["nb"], leaf_node_holder=case["nl"],
                                size_minimum=case["low"], stream=cont_case_stream(case, seed, env_id, n))
    if case is not None:
        return OracleDiscrete(setting, container_size=case["container"], internal_node_holder=case["nb"], leaf_node_holder=case["nl"],
                              size_minimum=min(min(i) for i in case["items"]), stream=case_stream(case, seed, env_id, n))
    if cont:
        return OracleContinuous(setting, stream=make_continuous_stream(seed, env_id, n, setting))
    return OracleDiscrete(setting, stream=make_stream(seed, env_id, n, setting))


def _invariants(g):
    """structural invariants of an oracle export (the device side's are enforced by its decoder)"""
    assert sum(len(x) for x in g["load_upper"]) == g["n_edge"]
    for u in range(g["n_box"]):
        assert all(0 <= s < u for s in g["supports"][u]), (u, g["supports"][u])
        assert all(u < up <= g["n_box"] for up in g["load_upper"][u]), (u, g["load_upper"][u])
        assert len(set(g["load_upper"][u])) == len(g["load_upper"][u])
        assert np.isfinite(g["loads"][u]).all()  # a mass may be 0 (the supports beside a direct one) or negative (a component of the lstsq split)
        assert (len(g["polygon"][u]) >= 3) == (len(g["supports"][u]) >= 1)
        for s in g["supports"][u]:  # every support lists the box among its loads, and only supports do
            assert u in g["load_upper"][s]
        assert np.isfinite(g["own_stack"][u]).all()
    n_sup = sum(len(x) for x in g["supports"])
    assert g["n_edge"] == n_sup + (g["failed_box"][1] if g["failed_box"][0] else 0)


@pytest.mark.parametrize("cont", [False, True], ids=["discrete", "continuous"])
@pytest.mark.parametrize("setting", [1, 2, 3])
def test_oracle_export_is_well_formed(setting, cont):
    n_edge = 0
    for env_id in range(3):
        env = _oracle(cont, setting, 300 + setting, env_id)
        o = env.reset()
        for t in range(150):
            _, row = policy_pick(o, 80, 50, 300 + setting, env_id, t)
            o, _, done, _ = env.step(row)
            g = env.support_graph()
            _invariants(g)
            n_edge = max(n_edge, g["n_edge"])
            if done:
                o = env.reset()
                assert env.support_graph()["n_edge"] == 0
    assert (n_edge > 20) == (setting != 2)


@pytest.mark.parametrize("alias", [False, True], ids=["snapshot", "alias"])
@pytest.mark.parametrize("cont", [False, True], ids=["discrete", "continuous"])
@pytest.mark.parametrize("setting", [1, 2, 3])
def test_host_build_graph_equals_the_oracle_graph(lib, setting, cont, alias):
    tot = None
    for env_id in range(4):
        seed = (77 if cont else 300) + setting
        t = _run(lib, _oracle(cont, setting, seed, env_id), cont, setting, (1.0, 1.0, 1.0) if cont else (10, 10, 10), 80, 50, seed, env_id, 300, alias)
        tot = t if tot is None else {k: tot[k] + v for k, v in t.items()}
    print("compared", tot)
    assert tot["pairs"] == 1200
    if setting != 2:
        assert tot["loads"] > 5000 and tot["vertices"] > 2000 and tot["splits"] > 100 and (tot["own"] > 2000) == alias
    else:
        assert tot["loads"] == tot["vertices"] == 0


@pytest.mark.parametrize("alias", [False, True], ids=["snapshot", "alias"])
@pytest.mark.parametrize("name", ["big_s1", "big_s3", "dense16_s1", "flat_s1", "holders_s1", "c:box2_s1", "c:box2_s3", "c:holders_s1"])
def test_graph_on_other_configurations(lib, name, alias):
    cont = name.startswith("c:")
    c = (CONT_CASES if cont else CASES)[name[2:] if cont else name]
    tot = _run(lib, _oracle(cont, c["setting"], 91, 2, 600, case=c), cont, c["setting"], c["container"], c["nb"], c["nl"], 91, 2, 300, alias)
    print("compared", tot)
    assert tot["loads"] > 1000 and tot["vertices"] > 300


@pytest.mark.parametrize("alias", [False, True], ids=["snapshot", "alias"])
@pytest.mark.parametrize("cont,setting,env_id,step", [(False,) + d for d in DIVERGING] + [(True,) + d for d in DIVERGING_C])
def test_graph_through_the_parting_steps(lib, cont, setting, env_id, step, alias):
    """each build against the oracle of its own semantics, through and past the step at which the two semantics part"""
    tot = _run(lib, _oracle(cont, setting, 1234, env_id, 600), cont, setting, (1.0, 1.0, 1.0) if cont else (10, 10, 10), 80, 50, 4321, env_id,
               step + 25, alias)
    assert tot["loads"] > 300


@pytest.mark.parametrize("alias", [False, True], ids=["snapshot", "alias"])
@pytest.mark.parametrize("cont", [False, True], ids=["discrete", "continuous"])
def test_graph_after_a_failed_real_placement(lib, cont, alias):
    """A real placement whose descent fails: both sides keep what it wrote before it failed (in alias mode: what alias_sync_loads leaves
    behind) until the reset.  Once a bin holds 14 boxes the policy picks the highest placement the oracle found unstable; most of those fail at their
    own support polygon and write nothing, the ones that fail further down leave loads of a box that was never placed."""
    tot = None
    for setting in (1, 3):
        for env_id in range(6):
            seed = (77 if cont else 300) + setting
            t = _run(lib, _oracle(cont, setting, seed, env_id), cont, setting, (1.0, 1.0, 1.0) if cont else (10, 10, 10), 80, 50, seed, env_id, 250,
                     alias, fail_from=14)
            tot = t if tot is None else {k: tot[k] + v for k, v in t.items()}
    print("compared", tot)
    assert tot["failed"] >= 50 and tot["failed_with_loads"] >= 2


def _first_graph_difference(host, env, t):
    try:
        compare_graphs(host.graph(), env.support_graph(), "step %d:" % t)
        return None
    except AssertionError as ex:
        return str(ex)


def test_graph_parts_no_later_than_the_observations(lib):
    """Sensitivity: the snapshot build next to the ALIAS oracle.  DESIGN.md section 3 (b): under the snapshot semantics a box below briefly
    carries more mass, so the stored graph leaves the alias oracle's before (or when) an observation does.  Prints, per trajectory, the
    step at which the graph parts and the step at which the observations of the two semantics part."""
    earlier, report = 0, []
    for cont, traj in ((False, DIVERGING), (True, DIVERGING_C)):
        for setting, env_id, step in traj:
            a, b = _oracle(cont, setting, 1234, env_id, 600), _oracle(cont, setting, 1234, env_id, 600)  # alias oracle, snapshot oracle
            a.set_alias_mode(True)
            b.set_alias_mode(False)
            host = Host(lib, cont, setting, (1.0, 1.0, 1.0) if cont else (10, 10, 10), 80, False)
            oa, ob = a.reset(), b.reset()
            t_graph = t_obs = None
            for t in range(step + 1):
                _, row = policy_pick(ob, 80, 50, 4321, env_id, t)
                nbx, den = b.next_box, b.next_den
                oa, _, da, _ = a.step(row)
                ob, _, db, _ = b.step(row)
                host.place(row, nbx, den)
                if t_graph is None and _first_graph_difference(host, a, t):
                    t_graph = t
                if da != db or not np.array_equal(oa, ob):
                    t_obs = t
                    break
                if da:
                    oa, ob = a.reset(), b.reset()
                    host.reset()
            host.close()
            report.append(("continuous" if cont else "discrete", setting, env_id, t_graph, t_obs))
            assert t_obs == step
            assert t_graph is not None and t_graph <= t_obs, report[-1]
            earlier += int(t_graph < t_obs)
    print("domain, setting, env, step the graph parts, step the observations part:", report)
    assert earlier >= 1, report


# ---- the decoder and the comparison on a damaged record: each names box and field --------------------------------------------------
def _loaded_host(lib, alias=True):
    env = _oracle(False, 1, 301, 0)
    env.set_alias_mode(alias)
    host = Host(lib, False, 1, (10, 10, 10), 80, alias)
    o = env.reset()
    for t in range(18):
        _, row = policy_pick(o, 80, 50, 301, 0, t)
        nbx, den = env.next_box, env.next_den
        o, _, done, _ = env.step(row)
        assert host.place(row, nbx, den) and not done
    assert host.graph()["n_edge"] > 8
    compare_graphs(host.graph(), env.support_graph())
    return host, env


def test_a_flipped_load_mass_is_named(lib):
    host, env = _loaded_host(lib)
    g = host.graph()
    raw = (C.c_uint64 * (4 * 256)).from_address(host.field(0))  # e_st: 256 x (cx, cy, cz, m)
    q = g["n_edge"] // 2
    raw[4 * q + 3] ^= 1  # last bit of the mass of edge q
    with pytest.raises(AssertionError, match=r"box \d+ load mass: row \d+ \(from box \d+\)"):
        compare_graphs(host.graph(), env.support_graph(), "env 0")
    raw[4 * q + 3] ^= 1
    compare_graphs(host.graph(), env.support_graph())
    host.close()


def test_a_flipped_list_link_is_named(lib):
    host, env = _loaded_host(lib)
    nxt = (C.c_uint8 * 256).from_address(host.field(1))
    q = next(i for i in range(host.graph()["n_edge"]) if nxt[i] != 255)  # an edge with a successor in its box's list
    keep = nxt[q]
    for bad, what in ((q, "filed twice"), (255, "is in no load list|ends at edge"), (254, "beyond n_edge")):
        nxt[q] = bad
        d, err = __import__("pct_b200")._lib.SupportGraph(), C.create_string_buffer(256)
        assert lib.sh_support_graph(host.h, C.byref(d), err, 256) == 0
        assert __import__("re").search(r"(box|edge) \d+.*(%s)" % what, err.value.decode()), err.value
    nxt[q] = keep
    compare_graphs(host.graph(), env.support_graph())
    host.close()


def test_a_flipped_alias_bit_is_named(lib):
    host, env = _loaded_host(lib, alias=True)
    bits = (C.c_uint32 * 8).from_address(host.field(2))
    bits[0] ^= 1 << 3
    with pytest.raises(AssertionError, match=r"box \d+ load is_alias"):
        compare_graphs(host.graph(), env.support_graph(), "env 0")
    host.close()
