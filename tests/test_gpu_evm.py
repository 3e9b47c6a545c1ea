"""GPU: LNES='EVM' (EventPoint over the maintained EMS list and ZMAP) in lock-step with the CPU model of tests/evm_oracle.py, which
tests/test_evm_cpu.py holds against records of the reference.  Every comparison is exact: observation bytes, rewards, dones and flags."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
import buffer_oracle  # noqa: E402
from evm_cases import EVM_CASES  # noqa: E402
from evm_oracle import EvmOracle, FLAG_CAND_OVERFLOW  # noqa: E402
from harness import FLAG_EMS, case_stream, policy_pick  # noqa: E402

pytestmark = pytest.mark.gpu
SEED = 23


def _batch(c, streams, **kw):
    import pct_b200
    return pct_b200.PctBatch(len(streams), c["setting"], container_size=c["container"], item_set=c["items"], internal_node_holder=c["nb"],
                             leaf_node_holder=c["nl"], obs_dtype=torch.float64, item_stream=np.stack(streams), LNES="EVM", **kw)


def _models(c, streams, shuffle=False):
    ms = [EvmOracle(c["setting"], c["container"], c["nb"], c["nl"], stream=s) for s in streams]
    if shuffle:
        for e, m in enumerate(ms):
            m.set_shuffle(SEED, e)
    return ms


def _streams(c, n, steps):
    return [case_stream(c, c["seed"], e, steps + 64) for e in range(n)]


@pytest.mark.parametrize("shuffle", [False, True], ids=["list", "shuffle"])
@pytest.mark.parametrize("by", ["leaf", "rows"])
@pytest.mark.parametrize("name", sorted(EVM_CASES))
def test_step_lockstep(name, by, shuffle):
    """pct_step by leaf index and by caller rows; an env leaves the lock-step on the step its model flags, and the device flags exactly there"""
    c = EVM_CASES[name]
    n, steps = 8, c["steps"]
    streams = _streams(c, n, steps)
    ms = _models(c, streams, shuffle)
    P = _batch(c, streams, seed=SEED, shuffle=shuffle)
    o_ref = np.stack([m.reset() for m in ms])
    o = P.reset().cpu().numpy()
    live = np.ones(n, dtype=bool)
    flagged = 0
    for t in range(steps):
        fl = np.array([P.state(e)["flags"] for e in range(n)])
        for e in np.nonzero(live)[0]:
            if ms[e].flags:
                assert fl[e] & FLAG_CAND_OVERFLOW, (name, t, e)
                live[e] = False
                flagged += 1
                continue
            if fl[e] & FLAG_EMS:  # the EMS list's own capacity, as under LNES='EMS'
                assert len(ms[e].ems()) > 128 or ms[e].o.n_ems_intermediate() > 256, (name, t, e)
                live[e] = False
                continue
            assert fl[e] == 0, (name, t, e, fl[e])
            assert np.array_equal(o_ref[e], o[e]), (name, t, e, np.argwhere(o_ref[e] != o[e])[:3].tolist())
        if not live.any():
            break
        picks = [policy_pick(o_ref[e], c["nb"], c["nl"], SEED, e, t) for e in range(n)]
        rows = np.stack([p[1] for p in picks])
        for e in np.nonzero(live)[0]:
            ob, r, d, _ = ms[e].step(rows[e])
            o_ref[e] = ms[e].reset() if d else ob
        if by == "leaf":
            ob, r, d, info = P.step(leaf_idx=torch.tensor([p[0] for p in picks], dtype=torch.int64, device=P.device))
        else:
            ob, r, d, info = P.step(actions=torch.from_numpy(rows).to(P.device))
        o = ob.cpu().numpy()
    if c["setting"] == 2 and c["container"] != (10, 10, 10):
        assert flagged > 0  # these bins cross the per-level set limit within the record's steps (tests/golden/evm_golden.npz)


def test_selected_envs_and_items():
    """pct_step_envs, pct_reset_envs_only and pct_set_items_only against the model; expand_items row l equals set_items row l"""
    c = EVM_CASES["s2_10"]
    n, steps = 8, 30
    streams = _streams(c, n, steps + 10)
    ms = _models(c, streams)
    P = _batch(c, streams)
    o_ref = np.stack([m.reset() for m in ms])
    o = P.reset().cpu().numpy()
    rng = np.random.RandomState(3)
    for t in range(steps):
        assert np.array_equal(o_ref, o), t
        sel = np.sort(rng.choice(n, 3, replace=False))
        picks = [policy_pick(o_ref[e], c["nb"], c["nl"], SEED, e, t) for e in range(n)]
        if t % 7 == 3:
            for e in sel:
                o_ref[e] = ms[e].reset()
            o = P.reset(env_idx=torch.tensor(sel, device=P.device), whole_batch=False).cpu().numpy()
            continue
        if t % 5 == 4:
            items = np.array([[1 + (e + t) % 5, 2, 1 + t % 3] for e in sel], dtype=np.int32)
            want = P.expand_items(torch.from_numpy(items[:, None, :]).to(P.device), env_idx=torch.tensor(sel, device=P.device))[0].cpu().numpy()
            for i, e in enumerate(sel):
                o_ref[e] = ms[e].set_next(np.array([*items[i], 1.0]))
            o = P.set_items(torch.from_numpy(items).to(P.device), env_idx=torch.tensor(sel, device=P.device), whole_batch=False).cpu().numpy()
            for i, e in enumerate(sel):
                assert np.array_equal(want[i, 0].reshape(-1), o[e].reshape(-1, 9)[c["nb"]:c["nb"] + c["nl"]].reshape(-1)), (t, e)
            continue
        for e in sel:
            ob, _, d, _ = ms[e].step(picks[e][1])
            o_ref[e] = ms[e].reset() if d else ob
        ob, _, _, _ = P.step(leaf_idx=torch.tensor([p[0] for p in picks], dtype=torch.int64, device=P.device),
                             env_idx=torch.tensor(sel, device=P.device))
        o = ob.cpu().numpy()
    assert all(P.state(e)["flags"] == 0 for e in range(n))


def test_snapshot_restore_and_graph():
    """a snapshot taken mid-episode and restored into a fresh handle continues byte for byte; steps captured in a CUDA graph replay exactly"""
    c = EVM_CASES["s1_14x12"]
    n = 16
    streams = _streams(c, n, 80)
    A = _batch(c, streams)
    A.reset()
    for t in range(12):
        A.step(leaf_idx=A.random_policy(5, t))
    snap = A.snapshot()
    B = _batch(c, streams)
    B.reset()
    B.restore(snap)
    st = torch.cuda.Stream()
    idx = [A.random_policy(5, 100 + t).clone() for t in range(6)]
    outs_a = [A.step(leaf_idx=i)[0].clone() for i in idx]
    B.step(leaf_idx=idx[0])  # warm-up outside the capture
    B.restore(snap)
    static_idx = idx[0].clone()
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g, stream=st):
        ob_g, _, _, _ = B.step(leaf_idx=static_idx)
    B.restore(snap)
    for t in range(6):
        static_idx.copy_(idx[t])
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(ob_g, outs_a[t]), t


@pytest.mark.parametrize("B", [3, 16])
def test_buffered_lockstep(B, monkeypatch):
    """a buffered batch against the buffered oracle model (tests/buffer_oracle.py) with the EVM model as its env"""
    from test_gpu_buffer_oracle import lockstep

    def make(c, stream):
        return EvmOracle(c["setting"], c["container"], c["nb"], c["nl"], c["size_minimum"], stream) if c.get("lnes") == "EVM" \
            else buffer_oracle.OracleDiscrete(c["setting"], container_size=c["container"], internal_node_holder=c["nb"], leaf_node_holder=c["nl"],
                                              size_minimum=c["size_minimum"], stream=stream, lnes=c.get("lnes", "EMS"))
    monkeypatch.setattr(buffer_oracle, "make_oracle", make)
    e = EVM_CASES["s1_10"]
    c = dict(domain="discrete", setting=1, container=e["container"], nb=80, nl=50, size_minimum=1, lnes="EVM", items=e["items"])
    streams = [case_stream(e, 31, k, 400) for k in range(4)]
    fired = lockstep(c, streams, B, 25, graphs=0)
    assert not any(fired)


def test_twin_of_ems():
    """EVM and EMS batches stepped by the same heuristic rows keep the same boxes, EMS lists and draw positions; only the leaves differ"""
    c = EVM_CASES["s3_10"]
    n = 32
    streams = _streams(c, n, 120)
    import pct_b200
    A = _batch(c, streams)
    E = pct_b200.PctBatch(n, c["setting"], container_size=c["container"], item_set=c["items"], obs_dtype=torch.float64, item_stream=np.stack(streams))
    oa, oe = A.reset().cpu().numpy(), E.reset().cpu().numpy()
    for t in range(40):
        rows = E.heuristic_actions("LSAH", seed=1, t=t).clone()
        A.step(actions=rows)
        E.step(actions=rows)
        for e in range(0, n, 5):
            sa, se = A.state(e), E.state(e)
            assert np.array_equal(sa["boxes"], se["boxes"]) and np.array_equal(sa["ems"], se["ems"]) and sa["draw_pos"] == se["draw_pos"], (t, e)
    assert not np.array_equal(oa, oe)
