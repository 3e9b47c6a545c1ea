"""GPU, BASELINE config 4 at full size: 4096 PackingContinuous envs (sample_from_distribution U(0.1, 0.5), unit container, device
item generator) stepped with the synthetic policy — every one of the final float64 observations, the per-env episode counts and the
reward sums must equal the threaded CPU oracle's (oracle/pct_oracle_batch_continuous.c).  Trajectories are chaotic, so equality of
the final state certifies every intermediate step.  Settings 1 (stability) and 2 (six orientations).
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
from pct_oracle import OracleBatchContinuous  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("setting,n", [(1, 4096), (2, 4096), (3, 1024)])
def test_full_size_final_observations_continuous(setting, n):
    import pct_b200
    steps, iseed, pseed = 100, 1234, 4321
    gpu = pct_b200.PctBatch(n, setting, container_size=(1.0, 1.0, 1.0), continuous=True, sample_from_distribution=True, seed=iseed,
                            obs_dtype=torch.float64)
    cpu = OracleBatchContinuous(n, setting, iseed, pseed)
    gpu.reset()
    rsum = torch.zeros(n, dtype=torch.float64, device="cuda")
    nd = torch.zeros(n, dtype=torch.int64, device="cuda")
    flags = torch.zeros(n, dtype=torch.int32, device="cuda")
    for t in range(steps):
        obs, r, d, info = gpu.step(leaf_idx=gpu.random_policy(pseed, t))
        rsum += r.double(); nd += d.long(); flags |= info[:, 1]
    cpu.run(steps)
    o_ref, r_ref, nd_ref = cpu.get()
    assert int(flags.max()) == 0
    assert np.array_equal(nd.cpu().numpy(), nd_ref)
    bad = np.unique(np.argwhere(obs.cpu().numpy() != o_ref)[:, 0])
    assert len(bad) == 0, "envs with a different final observation: %s" % bad[:10]
    assert np.allclose(rsum.cpu().numpy(), r_ref, rtol=0, atol=1e-4)  # GPU rewards are float32 (VecPyTorch contract)
