"""GPU: the ALIAS variant of the real placement (the default since round 2; PCT_B200_ALIAS=0 selects the snapshot kernels of round 1:
pct_apply_kernel<STAB, ALIAS = true> -> stability_check<true, GeomD, true>, the reference's Python-object semantics of the load entries,
DESIGN.md section 3 (b)) against the oracle's alias mode — on the BASELINE-stream trajectories where the two semantics part
(scratch/alias_rate.py) and on ordinary batches; the snapshot kernels must keep following the snapshot oracle on the same trajectories.
The routine's logic is also verified on its HOST build (tests/test_host_emul_stability.py).
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
from harness import ITEM_SET, make_stream, policy_pick  # noqa: E402
from pct_oracle import OracleDiscrete  # noqa: E402

pytestmark = pytest.mark.gpu
DIVERGING = [(1, 126, 39), (1, 835, 167), (3, 92, 103)]  # (setting, global env id, step of the first difference); items 1234, policy 4321


def _lockstep(setting, env_id, steps, alias, monkeypatch):
    import pct_b200
    monkeypatch.setenv("PCT_B200_ALIAS", "1" if alias else "0")
    gpu = pct_b200.PctBatch(1, setting, item_set=ITEM_SET, seed=1234, env_id_base=env_id, obs_dtype=torch.float64)
    orc = OracleDiscrete(setting, stream=make_stream(1234, env_id, 600, setting))
    orc.set_alias_mode(alias)
    o_ref, o = orc.reset(), gpu.reset().cpu().numpy()[0]
    for t in range(steps):
        assert np.array_equal(o_ref, o), "step %d (alias=%s)" % (t, alias)
        _, row = policy_pick(o_ref, 80, 50, 4321, env_id, t)
        o_ref, _, d_ref, _ = orc.step(row)
        if d_ref:
            o_ref = orc.reset()
        obs, _, d, info = gpu.step(leaf_idx=gpu.random_policy(4321, t))
        assert bool(d.cpu().numpy()[0]) == d_ref, "done at step %d (alias=%s)" % (t, alias)
        assert not gpu.decode_info(info)["flags"].any()
        o = obs.cpu().numpy()[0]
    gpu.close()


@pytest.mark.parametrize("setting,env_id,step", DIVERGING)
@pytest.mark.parametrize("alias", [True, False], ids=["alias", "snapshot"])
def test_real_placement_semantics_on_the_parting_trajectories(setting, env_id, step, alias, monkeypatch):
    _lockstep(setting, env_id, step + 30, alias, monkeypatch)


def test_snapshot_build_parts_from_the_alias_oracle(monkeypatch):
    """sensitivity: the default kernels do NOT follow the alias oracle through the parting step"""
    import pct_b200
    setting, env_id, step = DIVERGING[0]
    monkeypatch.setenv("PCT_B200_ALIAS", "0")
    gpu = pct_b200.PctBatch(1, setting, item_set=ITEM_SET, seed=1234, env_id_base=env_id, obs_dtype=torch.float64)
    orc = OracleDiscrete(setting, stream=make_stream(1234, env_id, 600, setting))
    orc.set_alias_mode(True)
    o_ref, o = orc.reset(), gpu.reset().cpu().numpy()[0]
    parted = False
    for t in range(step + 2):
        if not np.array_equal(o_ref, o):
            parted = True
            break
        _, row = policy_pick(o_ref, 80, 50, 4321, env_id, t)
        o_ref, _, d_ref, _ = orc.step(row)
        if d_ref:
            o_ref = orc.reset()
        obs, _, d, _ = gpu.step(leaf_idx=gpu.random_policy(4321, t))
        o = obs.cpu().numpy()[0]
    assert parted
    gpu.close()


@pytest.mark.parametrize("setting", [1, 3])
def test_alias_variant_on_a_batch(setting, monkeypatch):
    """32 envs x 150 steps in alias mode against per-env alias oracles (the ordinary lock-step of tests/test_gpu_discrete_parity.py)"""
    import pct_b200
    monkeypatch.setenv("PCT_B200_ALIAS", "1")
    n, seed = 32, 1234
    gpu = pct_b200.PctBatch(n, setting, item_set=ITEM_SET, seed=seed, obs_dtype=torch.float64)
    orcs = [OracleDiscrete(setting, stream=make_stream(seed, e, 600, setting)) for e in range(n)]
    for o_ in orcs:
        o_.set_alias_mode(True)
    o_ref = np.stack([o_.reset() for o_ in orcs])
    o = gpu.reset().cpu().numpy()
    for t in range(150):
        assert np.array_equal(o_ref, o), "step %d envs %s" % (t, np.unique(np.argwhere(o_ref != o)[:, 0])[:5])
        nxt = []
        for e in range(n):
            _, row = policy_pick(o_ref[e], 80, 50, 4321, e, t)
            ob, _, d_ref, _ = orcs[e].step(row)
            nxt.append(orcs[e].reset() if d_ref else ob)
        o_ref = np.stack(nxt)
        obs, _, _, info = gpu.step(leaf_idx=gpu.random_policy(4321, t))
        assert not gpu.decode_info(info)["flags"].any()
        o = obs.cpu().numpy()
    gpu.close()


# ---- continuous domain (pctc_apply_kernel<true, ALIAS = true>) -------------------------------------------------------------------------
DIVERGING_C = [(1, 1, 169), (1, 548, 152), (1, 597, 103), (1, 638, 163), (3, 635, 215)]  # scratch/alias_rate.py, sample_from_distribution streams


@pytest.mark.parametrize("setting,env_id,step", DIVERGING_C)
@pytest.mark.parametrize("alias", [True, False], ids=["alias", "snapshot"])
def test_real_placement_semantics_on_the_parting_trajectories_continuous(setting, env_id, step, alias, monkeypatch):
    import pct_b200
    from pct_oracle import OracleContinuous, make_continuous_stream
    monkeypatch.setenv("PCT_B200_ALIAS", "1" if alias else "0")
    gpu = pct_b200.PctBatch(1, setting, container_size=(1.0, 1.0, 1.0), continuous=True, sample_from_distribution=True, seed=1234,
                            env_id_base=env_id, obs_dtype=torch.float64)
    orc = OracleContinuous(setting, stream=make_continuous_stream(1234, env_id, 600, setting))
    orc.set_alias_mode(alias)
    o_ref, o = orc.reset(), gpu.reset().cpu().numpy()[0]
    for t in range(step + 25):
        assert np.array_equal(o_ref, o), "step %d (alias=%s)" % (t, alias)
        _, row = policy_pick(o_ref, 80, 50, 4321, env_id, t)
        o_ref, _, d_ref, _ = orc.step(row)
        if d_ref:
            o_ref = orc.reset()
        obs, _, d, info = gpu.step(leaf_idx=gpu.random_policy(4321, t))
        assert bool(d.cpu().numpy()[0]) == d_ref, "done at step %d (alias=%s)" % (t, alias)
        assert not gpu.decode_info(info)["flags"].any()
        o = obs.cpu().numpy()[0]
    gpu.close()


@pytest.mark.parametrize("setting,env_id,step", DIVERGING)
def test_terminal_observation_of_the_facade_under_the_object_semantics(setting, env_id, step, monkeypatch):
    """gym.Env semantics (no auto-reset): the observation returned WITH done=True is computed on the state the failed real placement left
    behind, where objects and snapshots differ — the ALIAS apply kernel synchronises the stored loads (alias_sync_loads) so that the
    ordinary feasibility kernel reproduces the alias oracle's terminal observation"""
    import pct_b200
    monkeypatch.setenv("PCT_B200_ALIAS", "1")
    stream = make_stream(1234, env_id, 600, setting)
    env = pct_b200.PackingDiscrete(setting=setting, container_size=[10, 10, 10], item_set=ITEM_SET, item_stream=stream[None])
    orc = OracleDiscrete(setting, stream=stream)
    orc.set_alias_mode(True)
    o_ref, o = orc.reset(), env.reset()
    terminals = 0
    for t in range(step + 10):
        assert np.array_equal(o_ref, o), "step %d" % t
        _, row = policy_pick(o_ref, 80, 50, 4321, env_id, t)
        o_ref, _, d_ref, _ = orc.step(row)
        o, _, d, _ = env.step(row)
        assert d == d_ref
        if d:
            assert np.array_equal(o_ref, o), "terminal observation after step %d" % t
            terminals += 1
            o_ref, o = orc.reset(), env.reset()
    assert terminals >= 1
    env.close()
