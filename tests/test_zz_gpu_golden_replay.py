"""GPU vs the reference's own records, with no oracle in between: every trajectory under tests/golden/ that was recorded
from the UNMODIFIED reference env (default configuration: discrete_s*_t*.npz, discrete_{EV,EP,CP,FC}_s*.npz,
continuous_s*_t0.npz; other containers / item sets / holder sizes: case_*.npz, ccase_*.npz) is replayed on the drop-in
single-env facades (PackingDiscrete / PackingContinuous = a GPU batch of one, gym.Env semantics) with the recorded leaf
rows; every float64 observation — terminal ones and the ones after reset() included —, reward, done, counter and ratio
must equal the record.

No record is excluded.
"""
import glob
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
from harness import CASES, CONT_CASES, ITEM_SET  # noqa: E402

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
DISCRETE = sorted(glob.glob(os.path.join(G, "discrete_*.npz"))) + sorted(glob.glob(os.path.join(G, "case_*.npz")))
CONTINUOUS = sorted(glob.glob(os.path.join(G, "continuous_s*.npz"))) + sorted(glob.glob(os.path.join(G, "ccase_*.npz")))
# no record is left out: the kernels implement the reference's object-alias semantics of the load entries by default since round 2, so
# ccase_alias_s1.npz (DESIGN.md section 3 (b)) is replayed like every other record


def _replay(env, g, exact_scalars):
    obs, k = g["obs"], 0
    o = env.reset()
    assert o.dtype == np.float64 and np.array_equal(o, obs[k]), "reset observation"
    k += 1
    for t in range(len(g["rows"])):
        o, r, d, info = env.step(g["rows"][t])
        assert np.array_equal(o, obs[k]), "observation after step %d (done=%s): %s" % (t, d, np.argwhere(o != obs[k])[:6].ravel())
        k += 1
        assert d == bool(g["done"][t]) and info["counter"] == g["counter"][t] and "flags" not in info, (t, info)
        assert r == g["reward"][t] if exact_scalars else abs(r - g["reward"][t]) < 1e-12
        if d:
            assert info["ratio"] == g["ratio"][t] if exact_scalars else abs(info["ratio"] - g["ratio"][t]) < 1e-12
            o = env.reset()
            assert np.array_equal(o, obs[k]), "observation after the reset following step %d" % t
            k += 1
    assert k == len(obs)


def test_files_present():
    assert len(DISCRETE) >= 14 + len(CASES) and len(CONTINUOUS) == 3 + len(CONT_CASES)


@pytest.mark.parametrize("path", DISCRETE, ids=[os.path.basename(p) for p in DISCRETE])
def test_gpu_replays_reference_record_discrete(path):
    import pct_b200
    g = np.load(path)
    if "name" in g.files:
        c = CASES[str(g["name"])]
    else:
        c = dict(setting=int(g["setting"]), container=(10, 10, 10), items=ITEM_SET, nb=80, nl=50, lnes=str(g["lnes"]) if "lnes" in g.files else "EMS")
    env = pct_b200.PackingDiscrete(setting=c["setting"], container_size=list(c["container"]), item_set=c["items"], internal_node_holder=c["nb"],
                                   leaf_node_holder=c["nl"], LNES=c["lnes"], item_stream=g["stream"][None])
    _replay(env, g, True)
    env.close()


@pytest.mark.parametrize("path", CONTINUOUS, ids=[os.path.basename(p) for p in CONTINUOUS])
def test_gpu_replays_reference_record_continuous(path):
    import pct_b200
    g = np.load(path)
    if "name" in g.files:
        c = CONT_CASES[str(g["name"])]
    else:
        c = dict(setting=int(g["setting"]), container=(1.0, 1.0, 1.0), nb=80, nl=50, low=0.1)
    env = pct_b200.PackingContinuous(setting=c["setting"], container_size=list(c["container"]), item_set=None, sample_from_distribution=False,
                                     internal_node_holder=c["nb"], leaf_node_holder=c["nl"], item_stream=g["stream"][None], size_minimum=c["low"])
    _replay(env, g, False)  # the facade sums get_ratio with numpy, the reference with reduce(): last-bit differences allowed on the scalars
    env.close()


# ---- dataset evaluation on the continuous env (records of the reference's own loop: tests/golden/eval_cont_s*.npz) ----------
EVAL_C = sorted(glob.glob(os.path.join(G, "eval_cont_s*.npz")))


def _eval_golden(path):
    g = np.load(path)
    off = np.concatenate([[0], np.cumsum(g["packed_len"])])
    packed = [g["packed_flat"][off[i]:off[i + 1]].tolist() for i in range(len(g["ratio"]))]
    return int(g["setting"]), g["data"], g["ratio"], g["counter"], packed


@pytest.mark.parametrize("path", EVAL_C, ids=[os.path.basename(p) for p in EVAL_C])
@pytest.mark.parametrize("n_envs", [1, 5])
def test_batched_evaluation_matches_reference_continuous(path, n_envs):
    from harness import eval_policy_torch
    from pct_b200.evaluation import evaluate_batched
    setting, data, ratio, counter, packed = _eval_golden(path)
    out = evaluate_batched(list(data), setting, policy=eval_policy_torch, container_size=(1.0, 1.0, 1.0), continuous=True, sample_left_bound=0.1,
                           n_envs=n_envs)
    assert out["length"].tolist() == counter.tolist()
    assert out["packed"] == packed
    assert out["ratio"].tolist() == ratio.tolist()


def test_single_env_facade_replays_reference_evaluation_continuous(tmp_path):
    """the single-env loop of evaluation_tools.evaluate on the drop-in PackingContinuous(load_test_data=True)"""
    import pct_b200
    from harness import sequential_eval
    setting, data, ratio, counter, packed = _eval_golden(EVAL_C[0])
    ds = os.path.join(str(tmp_path), "set.pt")
    torch.save([t.tolist() for t in data], ds)
    env = pct_b200.PackingContinuous(setting=setting, container_size=[1, 1, 1], item_set=None, data_name=ds, load_test_data=True,
                                     internal_node_holder=80, leaf_node_holder=50, shuffle=False, sample_from_distribution=True,
                                     sample_left_bound=0.1, sample_right_bound=0.5)
    rec = sequential_eval(lambda ep: (env, env.reset()), 5)
    assert [r[1] for r in rec] == counter[:5].tolist()
    assert [r[2] for r in rec] == packed[:5]
    assert np.allclose([r[0] for r in rec], ratio[:5], rtol=0, atol=1e-12)
    env.close()
