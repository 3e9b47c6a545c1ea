"""GPU: the heuristic baselines of buffered envs (buffer_heuristic_actions, buffer_step_rows; DESIGN.md section 22).

Lock-step against the buffered oracle model (tests/buffer_heuristics.py: the plain oracle baseline composed over the slots): after every step
the chosen slots and rows, every byte of the observation, the buffered items and the records.  At B = 1 against a plain handle byte for byte,
the row step against the model with caller-built rows, run_heuristic / evaluate_batched with a buffer against the oracle, CUDA-graph capture,
and the error codes of the three C calls."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
from buffer_heuristics import RowBufferedOracle  # noqa: E402
from buffer_oracle import config  # noqa: E402
from harness import CONT_BINS, CONT_ITEM_SET, cont_item_set  # noqa: E402

pytestmark = pytest.mark.gpu
SEED = 17
BAD = 2  # PCT_FLAG_BAD_ACTION: the "no placement" row of a discrete baseline ends the episode with it
INV, ST = -1, -4  # PCT_ERR_INVALID, PCT_ERR_STATE


def _np(t):
    return t.cpu().numpy().copy()


def _items(name, c):
    if c["domain"] == "discrete":
        return [tuple(i) for i in c["items"]]
    return cont_item_set(CONT_BINS[name]) if name in CONT_BINS else CONT_ITEM_SET


def _batch(cfg, c, streams, B, **kw):
    import pct_b200
    cont = c["domain"] == "continuous"
    return pct_b200.PctBatch(len(streams), c["setting"], container_size=c["container"], continuous=cont, item_set=_items(cfg, c),
                             internal_node_holder=c["nb"], leaf_node_holder=c["nl"], obs_dtype=torch.float64, item_stream=np.stack(streams),
                             size_minimum=c["size_minimum"], LNES=c.get("lnes", "EMS"), buffer=B, **kw)


def lockstep(cfg, heur, B, n=3, steps=30, nl=None):
    """n envs of configuration cfg with B slots, driven by buffer_heuristic_actions + buffer_step_rows, against RowBufferedOracle models"""
    c, mk = config(cfg, **({"nl": nl} if nl else {}))
    items = _items(cfg, c)
    streams = [mk(SEED, e, 400) for e in range(n)]
    P = _batch(cfg, c, streams, B)
    models = [RowBufferedOracle(c, s, B) for s in streams]
    o = _np(P.reset())
    for e, m in enumerate(models):
        m.reset()
        assert o[e].tobytes() == m.obs.tobytes(), "%s env %d: reset observation" % (cfg, e)
    dones = 0
    for t in range(steps):
        slots, rows = P.buffer_heuristic_actions(heur, seed=SEED, t=t)
        s, rw = _np(slots), _np(rows)
        want = [m.heuristic(heur, items, SEED, e, t) for e, m in enumerate(models)]
        for e in range(n):
            where = "%s %s B=%d env %d step %d" % (cfg, heur, B, e, t)
            assert s[e] == want[e][0], "%s: slot %d, model %d (scores %s, ranks %s)" % (where, s[e], want[e][0], want[e][3], want[e][4])
            assert np.array_equal(rw[e], want[e][1].astype(rw.dtype)), "%s: row %s, model %s" % (where, rw[e].tolist(), want[e][1].tolist())
        ob, r, d, info = P.buffer_step_rows(slots, rows)
        o, r, d, rec = _np(ob), _np(r), _np(d).astype(bool), P.decode_info(info)
        it = _np(P.buffer_items())
        for e, m in enumerate(models):
            where = "%s %s B=%d env %d step %d" % (cfg, heur, B, e, t)
            _, rr, dd, mr = m.step_row(int(s[e]), want[e][1])
            assert d[e] == dd and rec["counter"][e] == mr["counter"], where + ": done / counter"
            assert np.float32(rr) == r[e], where + ": reward"
            assert rec["flags"][e] & ~BAD == mr["flags"], "%s: flags %d, model %d" % (where, rec["flags"][e], mr["flags"])
            if want[e][2] is None and c["domain"] == "discrete":
                assert dd and rec["flags"][e] & BAD, where + ": no placement ends the episode with the bad-action flag"
            assert rec["n_leaf"][e] == mr["n_leaf"] and rec["n_cand"][e] == mr["n_cand"], where + ": record sums"
            assert o[e].tobytes() == m.obs.tobytes(), where + ": observation"
            assert it[e].tobytes() == m.buf.tobytes(), where + ": buffered items"
            dones += int(dd)
    P.close()
    return dones


DISC7 = ("LSAH", "OnlineBPH", "BR", "MACS", "DBL", "HM", "RANDOM")


DISC_CASES = [("d1", 1), ("d1", 3), ("d1", 16), ("d2", 3), ("d3", 3), ("big_s1", 3)]
CONT_CASES = [("c1", 1), ("c1", 3), ("c1", 16), ("c2", 3), ("c3", 3), ("pallet_s1", 3), ("mm_s2", 3)]


@pytest.mark.parametrize("cfg,B", DISC_CASES)
@pytest.mark.parametrize("heur", DISC7)
def test_lockstep_discrete(heur, cfg, B):
    lockstep(cfg, heur, B, n=2, steps=16 if B < 16 else 8)


@pytest.mark.parametrize("heur", ["HM", "MACS", "RANDOM"])
@pytest.mark.parametrize("B", [1, 3])
def test_lockstep_side255_big_path(heur, B):
    """HM / MACS / RANDOM on a side-255 bin: the BIG instantiation (height map and bitmap in dynamic shared memory)"""
    lockstep("side255", heur, B, n=1, steps=1 if heur == "MACS" else 2)


@pytest.mark.parametrize("cfg,B", CONT_CASES)
@pytest.mark.parametrize("heur", ["LSAH", "OnlineBPH", "BR"])
def test_lockstep_continuous(heur, cfg, B):
    lockstep(cfg, heur, B, n=2, steps=16 if B < 16 else 8)


@pytest.mark.parametrize("cont", [False, True])
@pytest.mark.parametrize("heur", ["LSAH", "OnlineBPH", "BR", "RANDOM"])
def test_b1_equals_a_plain_handle(heur, cont):
    """B = 1: buffer_heuristic_actions + buffer_step_rows give a plain handle's heuristic_actions + step(actions=rows), byte for byte, over
    whole episodes (the buffered observation at B = 1 is the plain one)"""
    if cont and heur == "RANDOM":
        pytest.skip("continuous: LSAH / OnlineBPH / BR only")
    c, mk = config("c1" if cont else "d2")
    streams = [mk(SEED, e, 600) for e in range(64)]
    Pb = _batch("c1" if cont else "d2", c, streams, 1)
    Pp = _batch("c1" if cont else "d2", c, streams, None)
    ob, op = _np(Pb.reset()), _np(Pp.reset())
    assert ob.tobytes() == op.tobytes()
    ends = 0
    for t in range(120):
        s, rb = Pb.buffer_heuristic_actions(heur, seed=SEED, t=t)
        rp = Pp.heuristic_actions(heur, seed=SEED, t=t)
        assert not s.any() and torch.equal(rb, rp), "step %d: rows" % t
        xb, yb, db, ib = Pb.buffer_step_rows(s, rb)
        xp, yp, dp, ip = Pp.step(actions=rp)
        assert _np(xb).tobytes() == _np(xp).tobytes() and torch.equal(yb, yp) and torch.equal(db, dp) and torch.equal(ib, ip), "step %d" % t
        ends += int(db.sum())
    assert ends > 0
    Pb.close()
    Pp.close()


@pytest.mark.parametrize("cfg", ["d1", "c2"])
@pytest.mark.parametrize("f32", [False, True])
def test_step_rows_caller_rows(cfg, f32):
    """buffer_step_rows with caller-built rows against the model's set_next + step: leaf rows of any slot (float32 or float64), rows of
    another slot's item (a bad action), all-zero rows and slots outside [0, B)"""
    c, mk = config(cfg)
    B, n = 3, 6
    streams = [mk(SEED + 1, e, 400) for e in range(n)]
    P = _batch(cfg, c, streams, B)
    models = [RowBufferedOracle(c, s, B) for s in streams]
    P.reset()
    for m in models:
        m.reset()
    rng = np.random.default_rng(3)
    for t in range(30):
        slots, rows = np.zeros(n, dtype=np.int32), np.zeros((n, 9))
        for e, m in enumerate(models):
            kind = rng.integers(0, 6)
            j = int(rng.integers(0, B))
            live = np.nonzero(m.n_leaf)[0]
            if kind <= 2 and len(live):  # a leaf of a slot that has one
                j = int(live[rng.integers(0, len(live))])
                rows[e] = m.blocks[j, rng.integers(0, m.n_leaf[j])]
            elif kind == 3 and len(live):  # another slot's leaf row
                k = int(live[rng.integers(0, len(live))])
                rows[e] = m.blocks[k, 0]
            elif kind == 4:
                j = [-1, B, 1000][rng.integers(0, 3)]
                rows[e] = m.blocks[0, 0]
            slots[e] = j
        if f32:
            rows = rows.astype(np.float32).astype(np.float64) if c["domain"] == "discrete" else rows
        rt = torch.tensor(rows, dtype=torch.float32 if (f32 and c["domain"] == "discrete") else torch.float64, device=P.device)
        ob, r, d, info = P.buffer_step_rows(torch.tensor(slots, device=P.device), rt)
        o, d, rec = _np(ob), _np(d).astype(bool), P.decode_info(info)
        for e, m in enumerate(models):
            where = "%s env %d step %d slot %d" % (cfg, e, t, slots[e])
            _, _, dd, mr = m.step_row(int(slots[e]), rows[e])
            assert d[e] == dd and rec["counter"][e] == mr["counter"], where
            assert rec["flags"][e] & ~BAD == mr["flags"], where
            assert o[e].tobytes() == m.obs.tobytes(), where + ": observation"
    P.close()


def _dataset(rng, n, lo=15, hi=30):
    return [np.array([[rng.integers(1, 6), rng.integers(1, 6), rng.integers(1, 6)] for _ in range(rng.integers(lo, hi))], dtype=np.float64)
            for _ in range(n)]


@pytest.mark.parametrize("heur", ["LSAH", "DBL", "HM", "OnlineBPH"])
@pytest.mark.parametrize("B", [1, 3])
def test_run_heuristic_buffered_dataset(heur, B):
    """run_heuristic(..., buffer=B) on a small dataset: per-episode ratio, length and packed boxes equal a CPU model run of the same
    episodes; at B = 1 the results equal run_heuristic without a buffer"""
    from pct_b200.evaluation import _streams
    from pct_b200.heuristics import run_heuristic
    from harness import ITEM_SET
    trajs = _dataset(np.random.default_rng(5), 10)
    episodes, n = 9, 4
    _, rec = run_heuristic(heur, 1, episodes, item_set=ITEM_SET, data=trajs, n_envs=n, seed=SEED, return_episodes=True, buffer=B)
    if B == 1:
        _, plain = run_heuristic(heur, 1, episodes, item_set=ITEM_SET, data=trajs, n_envs=n, seed=SEED, return_episodes=True)
        assert np.array_equal(rec["ratio"], plain["ratio"]) and np.array_equal(rec["length"], plain["length"]) and rec["packed"] == plain["packed"]
    stream, traj_len, quota = _streams(trajs, episodes, n, pad=B)
    c, _ = config("d1")
    for e in range(n):
        m = RowBufferedOracle(c, stream[e], B, traj=traj_len)
        m.reset()
        ep, t = 0, 0
        while ep < quota[e]:
            packed = m.orc.packed
            slot, row, _, _, _ = m.heuristic(heur, ITEM_SET, SEED, e, t)
            _, _, d, mr = m.step_row(slot, row)
            t += 1
            if d:
                k = e + ep * n
                assert rec["length"][k] == mr["counter"] and rec["ratio"][k] == mr["ratio"], "episode %d" % k
                assert [list(map(int, b)) for b in rec["packed"][k]] == [list(map(int, b)) for b in packed], "episode %d: packed" % k
                ep += 1


@pytest.mark.parametrize("B", [1, 3])
def test_evaluate_batched_buffered(B):
    """evaluate_batched(..., buffer=B) with a fixed flat-index policy (the last leaf of the last slot that has one) equals the model"""
    from pct_b200.evaluation import _streams, evaluate_batched
    from harness import ITEM_SET
    trajs = _dataset(np.random.default_rng(9), 8)
    episodes, n = 7, 3
    nl = 50

    def policy(obs, batch):
        lv = obs[:, 80 * 9:(80 + B * nl) * 9].reshape(obs.shape[0], B, nl, 9)[..., 8] == 1
        cnt = lv.sum(2)
        j = torch.where(cnt > 0, torch.arange(B, device=obs.device).expand_as(cnt), torch.full_like(cnt, -1)).max(1).values
        jj = j.clamp(min=0)
        l = (cnt.gather(1, jj[:, None])[:, 0] - 1).clamp(min=0)
        return (jj * nl + l).to(torch.int32)

    out = evaluate_batched(trajs, 1, policy=policy, item_set=ITEM_SET, episodes=episodes, n_envs=n, buffer=B)
    stream, traj_len, quota = _streams(trajs, episodes, n, pad=B)
    c, _ = config("d1")
    for e in range(n):
        m = RowBufferedOracle(c, stream[e], B, traj=traj_len)
        m.reset()
        ep = 0
        while ep < quota[e]:
            live = [j for j in range(B) if m.n_leaf[j] > 0]
            j = live[-1] if live else 0
            flat = j * nl + max(int(m.n_leaf[j]) - 1, 0)
            _, _, d, mr = m.step(flat)
            if d:
                k = e + ep * n
                assert out["length"][k] == mr["counter"] and out["ratio"][k] == mr["ratio"], "episode %d" % k
                ep += 1


def test_graph_capture():
    """the heuristic call and the row step capture into one CUDA graph; its replays continue the eager trajectory of a twin"""
    c, mk = config("d1")
    streams = [mk(SEED, e, 400) for e in range(32)]
    Pe, Pg = _batch("d1", c, streams, 3), _batch("d1", c, streams, 3)
    Pe.reset()
    Pg.reset()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            sl, rw = Pg.buffer_heuristic_actions("LSAH")
            og, _, dg, ig = Pg.buffer_step_rows(sl, rw)
    torch.cuda.synchronize()
    for t in range(20):
        g.replay()
        sl2, rw2 = Pe.buffer_heuristic_actions("LSAH")
        oe, _, de, ie = Pe.buffer_step_rows(sl2, rw2)
        torch.cuda.synchronize()
        assert torch.equal(og, oe) and torch.equal(dg, de) and torch.equal(ig, ie), "replay %d" % t
    Pe.close()
    Pg.close()


def test_errors():
    import pct_b200
    from pct_b200 import _lib
    L = _lib.lib()
    c, mk = config("d1")
    streams = [mk(SEED, e, 100) for e in range(4)]
    P = _batch("d1", c, streams, 3)
    dev = P.device
    sl = torch.zeros(4, dtype=torch.int32, device=dev)
    rw = torch.zeros((4, 9), dtype=torch.float32, device=dev)
    rd = torch.zeros((4, 9), dtype=torch.float64, device=dev)
    obs = torch.zeros((4, P.obs_len), dtype=torch.float64, device=dev)
    rew = torch.zeros(4, dtype=torch.float32, device=dev)
    done = torch.zeros(4, dtype=torch.uint8, device=dev)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    rc = lambda f, *a: int(f(P.h, *a))  # noqa: E731
    assert rc(L.pct_buffer_heuristic_actions, 0, p(sl), p(rw), 0, 0, None) == ST  # before pct_buffer_reset
    assert rc(L.pct_buffer_step_rows, p(sl), p(rw), 0, p(obs), p(rew), p(done), None, None) == ST
    P.reset()
    assert rc(L.pct_buffer_heuristic_actions, 7, p(sl), p(rw), 0, 0, None) == INV
    assert rc(L.pct_buffer_heuristic_actions, -1, p(sl), p(rw), 0, 0, None) == INV
    assert rc(L.pct_buffer_heuristic_actions, 0, None, p(rw), 0, 0, None) == INV
    assert rc(L.pct_buffer_heuristic_actions, 0, p(sl), None, 0, 0, None) == INV
    assert rc(L.pct_buffer_heuristic_actions_f64, 0, p(sl), p(rd), None) == INV  # the continuous call on a discrete handle
    assert rc(L.pct_buffer_step_rows, None, p(rw), 0, p(obs), p(rew), p(done), None, None) == INV
    assert rc(L.pct_buffer_step_rows, p(sl), None, 0, p(obs), p(rew), p(done), None, None) == INV
    assert rc(L.pct_buffer_heuristic_actions, 0, p(sl), p(rw), 0, 0, None) == 0
    assert rc(L.pct_heuristic_actions, 0, p(rw), 0, 0, None) == ST  # the plain call keeps refusing a buffered handle
    P.close()
    # BR without an item set; an unbuffered handle
    Q = pct_b200.PctBatch(2, 1, item_stream=np.stack(streams[:2]), obs_dtype=torch.float64, buffer=2, size_minimum=1)
    Q.reset()
    assert int(L.pct_buffer_heuristic_actions(Q.h, 2, p(sl), p(rw), 0, 0, None)) == ST
    assert int(L.pct_buffer_heuristic_actions(Q.h, 0, p(sl), p(rw), 0, 0, None)) == 0
    Q.close()
    U = _batch("d1", c, streams, None)
    U.reset()
    assert int(L.pct_buffer_heuristic_actions(U.h, 0, p(sl), p(rw), 0, 0, None)) == ST
    assert int(L.pct_buffer_step_rows(U.h, p(sl), p(rw), 0, p(obs), p(rew), p(done), None, None)) == ST
    U.close()
    # continuous: only LSAH / OnlineBPH / BR, and not the discrete call
    cc, mkc = config("c1")
    V = _batch("c1", cc, [mkc(SEED, e, 100) for e in range(4)], 2)
    V.reset()
    for code in (3, 4, 5, 6):
        assert int(L.pct_buffer_heuristic_actions_f64(V.h, code, p(sl), p(rd), None)) == INV
    assert int(L.pct_buffer_heuristic_actions(V.h, 0, p(sl), p(rw), 0, 0, None)) == INV
    assert int(L.pct_buffer_heuristic_actions_f64(V.h, 1, p(sl), p(rd), None)) == 0
    V.close()
    with pytest.raises(pct_b200.PctError):
        _batch("d1", c, streams, None).buffer_heuristic_actions("LSAH")
