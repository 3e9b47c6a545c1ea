"""GPU: the many-support scenarios of tests/many_supports.py in lock-step with the oracle — stability walks that visit nodes on 9 .. 32 supports,
whose hull, contact rectangles and least-squares split live in the env's one HBM scratch behind a per-env lock, with many walks of one env in
flight at once in different warps and SMs.  One env and a batch of 1024, both domains, settings 1 and 3.  Every step: observations (float64, bit
for bit), rewards, dones, counters, and flags, which must be zero (the scenarios stay inside every capacity on the oracle).  After the build-up
and at the end: the support graph of every env (harness.compare_graphs).  Launch variants, each set before the handle is created: the default
sequential walks, the fork-join walks, round 1's block-per-env feasibility kernel (discrete), 32 continuations per warp in both walk pools (up
to 32 walks of one env contending for its lock in one warp), and the snapshot semantics of the loads.

tests/test_many_supports_cpu.py counts what these scenarios cover and replays them through the host build of the same stability source."""
import functools

import numpy as np
import pytest

torch = pytest.importorskip("torch")
import many_supports as M  # noqa: E402
from harness import compare_graphs  # noqa: E402

pytestmark = pytest.mark.gpu

N_BATCH = 1024
VARIANTS = {"default": {}, "fork": {"PCT_B200_WALK": "fork"}, "k3_block": {"PCT_B200_K3": "block"},
            "lanes32": {"PCT_B200_WALK_LANES": "32", "PCT_B200_WALK_LANES_TALL": "32"}, "snapshot": {"PCT_B200_ALIAS": "0"}}
CASES = [(cont, setting) for cont in (False, True) for setting in (1, 3)]


@functools.lru_cache(maxsize=None)
def _oracle(cont, setting, n, alias):
    return M.trajectories(cont, setting, n, alias=alias)


def _lockstep(monkeypatch, cont, setting, n, variant):
    import pct_b200
    for k in {k for v in VARIANTS.values() for k in v}:
        monkeypatch.delenv(k, raising=False)
    for k, v in VARIANTS[variant].items():
        monkeypatch.setenv(k, v)
    alias = variant != "snapshot"
    recs = _oracle(cont, setting, n, alias)
    gpu = pct_b200.PctBatch(n, setting, container_size=M.container(cont), continuous=cont, internal_node_holder=M.NB, leaf_node_holder=M.NL,
                            obs_dtype=torch.float64, item_stream=M.streams(cont, setting, n), size_minimum=M.unit(cont))
    name = "%s setting %d, %d envs, %s" % ("continuous" if cont else "discrete", setting, n, variant)

    def same_obs(o, i, where):
        bad = [e for e, dg in enumerate(M.digest_rows(o.cpu().numpy())) if dg != recs[e]["obs"][i]]
        assert not bad, "%s, %s: observations of envs %s differ" % (name, where, bad[:8])

    same_obs(gpu.reset(), 0, "reset")
    rows = torch.from_numpy(np.stack([r["rows"] for r in recs], axis=1)).cuda()  # (steps, n, 9)
    compared = dict(loads=0, vertices=0)
    for t in range(M.STEPS):
        ob, rew, done, info = gpu.step(actions=rows[t])
        where = "step %d" % t
        inf = gpu.decode_info(info)
        assert not inf["flags"].any(), "%s, %s: flags %s in envs %s" % (name, where, np.unique(inf["flags"]), np.nonzero(inf["flags"])[0][:8])
        same_obs(ob, t + 1, where)
        for field, got, want in (("reward", rew.cpu().numpy(), np.array([r["reward"][t] for r in recs], dtype=np.float32)),
                                 ("done", done.cpu().numpy().astype(bool), np.array([r["done"][t] for r in recs])),
                                 ("counter", inf["counter"], np.array([r["counter"][t] for r in recs]))):
            bad = np.nonzero(got != want)[0]
            assert len(bad) == 0, "%s, %s: %s of env %d is %s, oracle %s" % (name, where, field, bad[0], got[bad[0]], want[bad[0]])
        if t in M.CHECKPOINTS:
            for e in range(n):
                for k, v in compare_graphs(gpu.support_graph(e), recs[e]["graphs"][t], "%s, after %s, env %d:" % (name, where, e)).items():
                    compared[k] = compared.get(k, 0) + v
    gpu.close()
    print("%s: %d steps in lock-step, graphs compared %s" % (name, M.STEPS, compared))
    assert compared["loads"] > 20 * n and compared["vertices"] > 4 * n


@pytest.mark.parametrize("cont,setting", CASES, ids=["d1", "d3", "c1", "c3"])
def test_one_env(monkeypatch, cont, setting):
    _lockstep(monkeypatch, cont, setting, 1, "default")


@pytest.mark.parametrize("cont,setting,variant", [(c, s, v) for c, s in CASES for v in VARIANTS if not (c and v == "k3_block")],  # k3_block: discrete only
                         ids=["%s%d-%s" % ("c" if c else "d", s, v) for c, s in CASES for v in VARIANTS if not (c and v == "k3_block")])
def test_batch(monkeypatch, cont, setting, variant):
    _lockstep(monkeypatch, cont, setting, N_BATCH, variant)
