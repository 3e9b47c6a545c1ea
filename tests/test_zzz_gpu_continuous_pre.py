"""GPU: the pre-rounded (default since round 2) resting-height loop of the continuous feasibility kernel (PCT_B200_CONT_PRE=1,
csrc/pct_continuous.cu rest_height_pre) must be bit-identical to the default: same lock-step parity against the CPU oracle
as tests/test_gpu_continuous_parity.py, and identical streams with the switch on and off.

Round 2 made the pre-rounded loop the default.
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("setting", [1, 2, 3])
def test_pre_rounded_mode_lockstep_vs_oracle(setting, monkeypatch):
    from test_gpu_continuous_parity import _run
    monkeypatch.setenv("PCT_B200_CONT_PRE", "1")
    _run(setting, 24, 100, "idx", seed=33)


@pytest.mark.parametrize("setting", [1, 2])
def test_pre_rounded_mode_equals_default(setting, monkeypatch):
    import pct_b200
    outs = []
    for mode in ("0", "1"):
        monkeypatch.setenv("PCT_B200_CONT_PRE", mode)
        b = pct_b200.PctBatch(512, setting, container_size=(1.0, 1.0, 1.0), continuous=True, sample_from_distribution=True, seed=17,
                              obs_dtype=torch.float64)
        obs = b.reset()
        acc = [obs.clone()]
        for t in range(60):
            obs, r, d, info = b.step(leaf_idx=b.random_policy(5, t))
            acc.append(obs.clone())
        assert not b.decode_info(info)["flags"].any()
        outs.append(torch.stack(acc).cpu().numpy())
        b.close()
    assert np.array_equal(outs[0], outs[1])
