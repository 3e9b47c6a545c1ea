"""GPU: action rows the leaf list never proposes (tests/rows_rule.py) on the apply kernels, the only code that decodes a row
(LeafNode2Action) and runs a real Space.drop_box: resting height over an arbitrary footprint, the apply kernel's own bounds and height
tests, and the real stability descent with its failure exits.

  * the records of the unmodified reference (tests/golden/rows_*.npz) replayed on PctBatch (auto_reset=False, float64 and float32 rows)
    and on the single-env facades (rows, and (rot, lx, ly) triples where the row is a plain rotation at a non-negative position):
    observations, reward, done, counter (and the facades' ratio) must be the record's; PCT_FLAG_BAD_ACTION on exactly the steps where
    the reference raised, no other flag.  float32 continuous rows are compared as tests/test_f32_rows.py compares them.
  * the real verdict against the read-only one: query_placements' feasibility and rest height for K placements per env, then each
    placement stepped as a row in its own slot restored from a snapshot; both against the oracle.
  * leaf indices at the edges: -1, n_leaf, leaf_node_holder and 2**31 - 1 select the all-zero row (a negative index does not wrap)."""
import glob
import itertools
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
from rows_rule import make_oracle  # noqa: E402

pytestmark = pytest.mark.gpu
G = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "rows_*.npz")))
TOL = 1e-6
BAD_ACTION = 2


def _batch(g, n=1):
    import pct_b200
    cont = str(g["domain"]) == "c"
    return pct_b200.PctBatch(n, int(g["setting"]), container_size=tuple(g["container"].tolist()), continuous=cont, internal_node_holder=int(g["nb"]),
                             leaf_node_holder=int(g["nl"]), obs_dtype=torch.float64, item_stream=np.stack([g["stream"]] * n),
                             size_minimum=float(g["size_minimum"]), auto_reset=False)


def _same(o, ref, f32, what):
    if not f32:
        assert np.array_equal(o, ref), "%s: observation differs at %s" % (what, np.argwhere(o != ref)[:4].tolist())
        return
    a, b = o.reshape(-1, 9), ref.reshape(-1, 9)
    assert np.array_equal(a[:, 6:9], b[:, 6:9]), "%s: valid / feasibility flags differ" % what
    assert np.abs(o - ref).max() <= TOL, "%s: coordinates differ by %g" % (what, np.abs(o - ref).max())


@pytest.mark.parametrize("dtype", ["f64", "f32"])
@pytest.mark.parametrize("path", G, ids=[os.path.basename(p)[5:-4] for p in G])
def test_batch_follows_the_reference_on_rows_of_its_own(path, dtype):
    g = np.load(path)
    cont = str(g["domain"]) == "c"
    if g["rows"].dtype == np.float32 and dtype == "f64":
        pytest.skip("recorded with float32 rows")
    f32 = cont and (dtype == "f32")
    if f32 and g["rows"].dtype != np.float32:
        pytest.skip("float64 continuous records are replayed with float64 rows; float32 rows have records of their own")
    env = _batch(g)
    obs, k = g["obs"], 0
    o = env.reset().cpu().numpy()[0]
    assert np.array_equal(o, obs[k]); k += 1
    flagged = 0
    for t in range(len(g["rows"])):
        w = "%s step %d (%s)" % (g["name"], t, g["kind"][t])
        a = torch.from_numpy(g["rows"][t][None].astype(np.float32 if dtype == "f32" else np.float64)).cuda()
        ob, r, d, info = env.step(actions=a)
        rec = env.decode_info(info)
        raised = bool(g["err"][t])
        assert int(rec["flags"][0]) == (BAD_ACTION if raised else 0), "%s: flags %d, reference raised %r" % (w, rec["flags"][0], str(g["err"][t]))
        assert bool(d.cpu().numpy()[0]) == bool(g["done"][t]), w
        flagged += raised
        if not raised:
            _same(ob.cpu().numpy()[0], obs[k], f32, w); k += 1
            assert rec["counter"][0] == g["counter"][t], w
            assert abs(float(r.cpu().numpy()[0]) - g["reward"][t]) <= 1e-6, w
            if bool(g["done"][t]):  # pct_step_info carries the ratio as float32
                assert abs(float(rec["ratio"][0]) - g["ratio"][t]) <= 1e-6, "%s: ratio %r, reference %r" % (w, rec["ratio"][0], g["ratio"][t])
        if bool(g["done"][t]):
            o = env.reset().cpu().numpy()[0]
            assert np.array_equal(o, obs[k]), "%s: reset" % w; k += 1
    assert k == len(obs)
    print("%s (%s rows): %d steps, %d flagged" % (g["name"], dtype, len(g["rows"]), flagged))
    env.close()


def _triple(row, nb):
    """(rot, lx, ly) for a row that is a plain rotation of the item at a non-negative integer position, else None"""
    if not np.all(row[:6] == np.round(row[:6])) or row[0] < 0 or row[1] < 0 or not row[:6].any():
        return None
    x, y = int(row[3] - row[0]), int(row[4] - row[1])
    if (x, y) == (nb[0], nb[1]):
        return (0, int(row[0]), int(row[1]))
    if (x, y) == (nb[1], nb[0]):
        return (1, int(row[0]), int(row[1]))
    return None


@pytest.mark.parametrize("path", G, ids=[os.path.basename(p)[5:-4] for p in G])
def test_facades_follow_the_reference_on_rows_of_its_own(path):
    import pct_b200
    g = np.load(path)
    cont = str(g["domain"]) == "c"
    cls = pct_b200.PackingContinuous if cont else pct_b200.PackingDiscrete
    kw = dict(sample_from_distribution=False) if cont else dict(item_set=[(1, 1, 1)])
    env = cls(int(g["setting"]), container_size=tuple(g["container"].tolist()), internal_node_holder=int(g["nb"]), leaf_node_holder=int(g["nl"]),
              item_stream=g["stream"][None], size_minimum=float(g["size_minimum"]), **kw)
    f32 = g["rows"].dtype == np.float32
    obs, k, triples = g["obs"], 0, 0
    o = env.reset()
    assert np.array_equal(o, obs[k]); k += 1
    for t in range(len(g["rows"])):
        w = "%s step %d (%s)" % (g["name"], t, g["kind"][t])
        row = g["rows"][t]
        a = row
        if not cont and t % 2:
            tr = _triple(row.astype(np.float64), env.next_box)
            if tr is not None:
                a, triples = list(tr), triples + 1
        o, r, d, info = env.step(a)
        raised = bool(g["err"][t])
        assert info.get("flags", 0) == (BAD_ACTION if raised else 0), w
        assert d == bool(g["done"][t]), w
        if not raised:
            _same(o, obs[k], f32, w); k += 1
            assert info["counter"] == g["counter"][t] and abs(r - g["reward"][t]) <= 1e-12, w
            if d:
                assert abs(info["ratio"] - g["ratio"][t]) <= (1e-6 if f32 else 1e-12), w
        if d:
            o = env.reset()
            assert np.array_equal(o, obs[k]), "%s: reset" % w; k += 1
    assert k == len(obs)
    print("%s: %d steps on the facade, %d as (rot, lx, ly) triples" % (g["name"], len(g["rows"]), triples))
    env.close()


def _placements(orc, cont, container, K, rng):
    """K placements [x, y, z, lx, ly] of the current item: every orientation at the leaf positions, box corners and arbitrary points"""
    sides = orc.next_box
    W, L, _ = container
    perms = [(sides[p[0]], sides[p[1]], sides[p[2]]) for p in itertools.permutations(range(3))]
    pts = [(e[0], e[1]) for e in orc.ems()] + [(b[3] + b[0], b[4]) for b in orc.packed] + [(b[3], b[4] + b[1]) for b in orc.packed]
    q = []
    while len(q) < K:
        x, y, z = perms[len(q) % len(perms)]
        if rng.random() < 0.5 and pts:
            lx, ly = pts[rng.integers(len(pts))]
        elif cont:
            lx, ly = round(rng.random() * max(W - x, 0), 3), round(rng.random() * max(L - y, 0), 3)
        else:
            lx, ly = int(rng.integers(0, max(W - x, 0) + 1)), int(rng.integers(0, max(L - y, 0) + 1))
        q.append([x, y, z, lx, ly])
    return np.array(q, dtype=np.float64)


@pytest.mark.parametrize("setting", [1, 3])
@pytest.mark.parametrize("name", ["d_cube", "c_cube"])
def test_real_verdict_agrees_with_the_read_only_one(name, setting):
    """16 envs at several depths of a recorded trajectory; K placements each through query_placements, then each placement stepped as a
    row in a slot restored from the env's snapshot (fan-out to K slots of a second handle).  The step succeeds exactly when the query
    says feasible, the placed box rests at the query's height, and both are the oracle's drop_box_virtual / real step on a copy of the env
    (the item stream from the draw that started the episode, then the episode's rows).  A real / virtual parting is allowed only where the
    oracle's snapshot-mode copy shows it is the alias parting."""
    import pct_b200
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "rows_%s_s%d.npz" % (name, setting)))
    cont = str(g["domain"]) == "c"
    container = tuple(g["container"].tolist())
    K, n = 32, 16
    rng = np.random.default_rng(77 + setting)
    # 16 states: the oracle replays the record's rows up to depth t_e (a fresh episode after every done)
    depths = sorted(set(int(v) for v in np.linspace(3, len(g["rows"]) - 1, n)))
    src = _batch(g, 1)
    fan = _batch(g, K)
    fan.reset()
    compared = failed = partings = flagged = 0
    o = src.reset()
    orc = make_oracle(g)
    orc.reset()
    cfg = {k: g[k] for k in ("domain", "setting", "container", "nb", "nl", "size_minimum", "stream")}
    t, draw0, draws, episode = 0, 0, 1, []  # draws: items the env has drawn (one per reset, one per placement); episode: rows since its reset

    def copy_at_state(alias=True):
        """an oracle in the state of `orc`: the stream from the draw that started this episode, then the episode's rows"""
        c = make_oracle(dict(cfg, stream=cfg["stream"][draw0:]), alias)
        c.reset()
        for r in episode:
            c.step(r)
        return c

    for depth in depths:
        while t < depth:
            row = g["rows"][t].astype(np.float64)
            _, _, d, _ = orc.step(row)
            ob, _, dd, _ = src.step(actions=torch.from_numpy(row[None]).cuda())
            assert bool(dd.cpu().numpy()[0]) == d
            if d:
                orc.reset()
                src.reset()
                draw0, episode = draws, []
            else:
                episode.append(row)
            draws += 1
            t += 1
        q = _placements(orc, cont, container, K, rng)
        feas, rest = src.query_placements(torch.from_numpy(q[None]).to(torch.float64 if cont else torch.int32))
        feas, rest = feas.cpu().numpy()[0], rest.cpu().numpy()[0].astype(np.float64)
        snap = src.snapshot()
        fan.restore(snap, env_idx=list(range(K)), rec_idx=[0] * K)
        rows = np.zeros((K, 9))
        rows[:, 0], rows[:, 1], rows[:, 3], rows[:, 4], rows[:, 5] = q[:, 3], q[:, 4], q[:, 3] + q[:, 0], q[:, 4] + q[:, 1], container[2]
        ob, _, d, info = fan.step(actions=torch.from_numpy(rows).cuda())
        d = d.cpu().numpy().astype(bool)
        flags = fan.decode_info(info)["flags"]
        for i in range(K):
            w = "%s s%d depth %d placement %s" % (name, setting, depth, q[i].tolist())
            ok_v, mh_v = orc.drop_box_virtual(q[i, :3], q[i, 3], q[i, 4])
            assert feas[i] == ok_v and (not ok_v or rest[i] == mh_v), "%s: query (%s, %r), oracle virtual (%s, %r)" % (w, feas[i], rest[i], ok_v, mh_v)
            _, _, d_real, info_real = copy_at_state().step(rows[i])  # the oracle's real step on a copy of the env
            assert d[i] == d_real, "%s: device step done %s, oracle real step done %s" % (w, d[i], d_real)
            # a footprint at or past max(W, L) has an empty slice of the height map: the reference raises there (include/pct_b200.h)
            assert flags[i] == (BAD_ACTION if info_real.get("error") == 2 else 0), "%s: flags %d" % (w, flags[i])
            flagged += int(flags[i] != 0)
            if not d[i]:
                z = fan.state(i)["boxes"][-1][2]
                assert z == rest[i], "%s: placed at z %r, query rest height %r" % (w, z, rest[i])
            if (not d[i]) != bool(feas[i]):
                # real and virtual verdicts part: allowed only as the alias parting (DESIGN.md section 3 (b)), which the snapshot semantics do not have
                _, _, d_snap, _ = copy_at_state(alias=False).step(rows[i])
                assert (not d_snap) == bool(feas[i]), "%s: real and virtual verdicts part in both alias modes" % w
                partings += 1
            failed += int(d[i] and rest[i] > 0)
            compared += 1
    print("%s s%d: %d placements compared, %d failed placements over boxes, %d alias partings of real and virtual verdicts, %d flagged" % (
        name, setting, compared, failed, partings, flagged))
    assert compared >= n * K // 2
    src.close()
    fan.close()


@pytest.mark.parametrize("name", ["d_cube_s1", "c_cube_s3"])
def test_leaf_indices_at_the_edges_select_the_zero_row(name):
    """-1, n_leaf, leaf_node_holder and 2**31 - 1 against the oracle stepped with the all-zero row (include/pct_b200.h, d_leaf_idx)"""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "rows_%s.npz" % name))
    env = _batch(g, 4)
    orcs = [make_oracle(g) for _ in range(4)]
    o_ref = np.stack([orc.reset() for orc in orcs])
    assert np.array_equal(env.reset().cpu().numpy(), o_ref)
    nb, nl = int(g["nb"]), int(g["nl"])
    for t in range(40):
        edge = t % 3 == 2
        nl_now = [int((o_ref[e].reshape(-1, 9)[nb:nb + nl, 8] == 1).sum()) for e in range(4)]
        idx = np.array([-1, nl_now[1], nl, 2 ** 31 - 1], dtype=np.int32) if edge else np.zeros(4, dtype=np.int32)
        res = [orcs[e].step(np.zeros(9) if edge or nl_now[e] == 0 else o_ref[e].reshape(-1, 9)[nb].copy()) for e in range(4)]
        ob, _, d, info = env.step(leaf_idx=torch.from_numpy(idx).cuda())
        done = np.array([r[2] for r in res])
        assert np.array_equal(d.cpu().numpy().astype(bool), done), t
        assert np.array_equal(ob.cpu().numpy(), np.stack([r[0] for r in res])), "step %d: indices %s" % (t, idx.tolist())
        assert not env.decode_info(info)["flags"].any(), t
        o_ref = np.stack([orcs[e].reset() if done[e] else res[e][0] for e in range(4)])
        if done.any():
            ob = env.reset(mask=torch.from_numpy(done).cuda())
        assert np.array_equal(ob.cpu().numpy(), o_ref), "after step %d" % t
    steps = 40
    print("%s: %d steps with edge leaf indices every third step" % (name, steps))
    env.close()


@pytest.mark.parametrize("alias", [None, "0"], ids=["alias", "snapshot"])
@pytest.mark.parametrize("auto_reset", [True, False], ids=["auto_reset", "gym"])
@pytest.mark.parametrize("setting", [1, 2, 3])
@pytest.mark.parametrize("cont", [False, True], ids=["discrete", "continuous"])
def test_rule_lockstep_with_graphs(cont, setting, auto_reset, alias, monkeypatch):
    """64 envs against one oracle each, stepped by the rule of tests/rows_rule.py on injected streams for 160 steps: observations, rewards,
    done and flags after every step, and the support graphs of a quarter of the envs (harness.compare_graphs), in gym mode also the graph a
    failed real descent leaves behind.  Each apply kernel (PCT_B200_ALIAS unset: object aliasing; 0: snapshot) against the oracle of its own
    semantics.  Setting 2 has no stability check, so its alias modes are the same kernel: run once."""
    import pct_b200
    from harness import compare_graphs, make_stream
    from pct_oracle import OracleContinuous, OracleDiscrete, make_continuous_stream
    from rows_rule import is_leaf, oracle_counts_step, pick
    if setting == 2 and alias is not None:
        pytest.skip("setting 2 has no stability check: the alias modes do not differ")
    if alias is None:
        monkeypatch.delenv("PCT_B200_ALIAS", raising=False)
    else:
        monkeypatch.setenv("PCT_B200_ALIAS", alias)
    n, steps, nb, nl, seed = 64, 160, 80, 50, 9300 + setting
    container = (1.0, 1.0, 1.0) if cont else (10, 10, 10)
    streams = np.stack([(make_continuous_stream if cont else make_stream)(seed, e, steps + 8, setting) for e in range(n)])
    gpu = pct_b200.PctBatch(n, setting, container_size=container, continuous=cont, obs_dtype=torch.float64, item_stream=streams,
                            size_minimum=0.1 if cont else 1.0, auto_reset=auto_reset)
    orcs = [(OracleContinuous if cont else OracleDiscrete)(setting, container_size=container, size_minimum=0.1 if cont else 1.0, stream=s)
            for s in streams]
    for o in orcs:
        o.set_alias_mode(alias is None)
    watched = range(0, n, 4)
    tot = dict(pairs=0, loads=0, vertices=0, splits=0, own=0, failed_with_loads=0, offleaf_multi=0, lstsq=0, flagged=0, offleaf=0)

    def graphs(what):
        for e in watched:
            for k, v in compare_graphs(gpu.support_graph(e), orcs[e].support_graph(), "%s env %d:" % (what, e)).items():
                tot[k] += v
            tot["pairs"] += 1

    o_ref = np.stack([o.reset() for o in orcs])
    assert np.array_equal(gpu.reset().cpu().numpy(), o_ref)
    graphs("reset")
    for t in range(steps):
        picks = [pick(o_ref[e], nb, nl, container, cont, seed, e, t) for e in range(n)]
        res = []
        for e in range(n):
            lb = orcs[e].n_lstsq
            r = orcs[e].step(picks[e][0])
            res.append(r)
            if setting != 2 and (r[2] or not is_leaf(picks[e][0], o_ref[e], nb, nl)):
                for k, v in oracle_counts_step(orcs[e], picks[e][0], o_ref[e], r, nb, nl, lb).items():
                    tot[k] += v
            tot["offleaf"] += int(not is_leaf(picks[e][0], o_ref[e], nb, nl))
        rows = torch.from_numpy(np.stack([p[0] for p in picks])).cuda()
        ob, rew, d, info = gpu.step(actions=rows)
        done = np.array([r[2] for r in res])
        assert np.array_equal(d.cpu().numpy().astype(bool), done), "step %d done" % t
        want = [BAD_ACTION if r[3].get("error") == 2 else int(r[3].get("error") == 1) for r in res]
        assert np.array_equal(gpu.decode_info(info)["flags"], want), "step %d flags" % t
        tot["flagged"] += int(np.count_nonzero(want))
        r_ref = np.array([r[1] for r in res], dtype=np.float32)
        assert np.abs(rew.cpu().numpy() - r_ref).max() <= 1e-6, "step %d rewards" % t
        if not auto_reset:  # the terminal observation and the graph a failed placement left behind
            assert np.array_equal(ob.cpu().numpy(), np.stack([r[0] for r in res])), "step %d" % t
            graphs("step %d" % t)
            if done.any():
                ob = gpu.reset(mask=torch.from_numpy(done).cuda())
        o_ref = np.stack([orcs[e].reset() if done[e] else res[e][0] for e in range(n)])
        bad = np.argwhere(ob.cpu().numpy() != o_ref)
        assert len(bad) == 0, "step %d: observation of env %d" % (t, bad[0][0])
        graphs("after step %d" % t)
    print("rule lock-step %s s%d %s %s: %s" % ("continuous" if cont else "discrete", setting, "auto_reset" if auto_reset else "gym",
                                                "alias" if alias is None else "snapshot", tot))
    assert tot["offleaf"] > n * steps // 10, tot
    if not cont:
        assert tot["flagged"] > 0, tot  # rows on which the reference raises
    if setting != 2:
        assert tot["failed_with_loads"] >= 10 and tot["offleaf_multi"] >= 20 and tot["loads"] > 0, tot
    gpu.close()
