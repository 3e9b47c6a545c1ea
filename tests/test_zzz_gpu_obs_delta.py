"""GPU: the delta observation writes (default since round 2) of the discrete feasibility kernel (PCT_B200_OBS_DELTA, default 1: when the caller hands back the
same observation buffer, only the rows that can differ from its contents are written) must leave exactly the observation the default
path writes — on the library-owned buffer, with alternating caller buffers (every switch falls back to a full write), inside a captured
CUDA graph, and through the zero-copy host path.

The delta rows are the default; this file also pins the full-rewrite mode.
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
from harness import ITEM_SET  # noqa: E402

pytestmark = pytest.mark.gpu


def _trace(setting, n, steps, delta, monkeypatch, alternate=False, obs_dtype=None):
    import pct_b200
    monkeypatch.setenv("PCT_B200_OBS_DELTA", "1" if delta else "0")
    b = pct_b200.PctBatch(n, setting, item_set=ITEM_SET, seed=41, obs_dtype=obs_dtype or torch.float32)
    bufs = [torch.full((n, b.obs_len), 7.0, dtype=b.obs_dtype, device=b.device) for _ in range(2)] if alternate else None
    out = [b.reset(out=bufs[0] if alternate else None).clone()]
    for t in range(steps):
        tgt = None if not alternate else bufs[0 if (t // 3) % 2 else 1]  # switch buffers every third step
        obs, r, d, info = b.step(leaf_idx=b.random_policy(3, t), out=tgt)
        out.append(obs.clone())
    assert not b.decode_info(info)["flags"].any()
    res = torch.stack(out).cpu().numpy()
    b.close()
    return res


@pytest.mark.parametrize("setting", [1, 2, 3])
def test_delta_equals_full_on_the_library_buffer(setting, monkeypatch):
    ref = _trace(setting, 700, 90, False, monkeypatch)
    got = _trace(setting, 700, 90, True, monkeypatch)
    assert np.array_equal(ref, got)


@pytest.mark.parametrize("setting", [1, 2])
def test_delta_equals_full_continuous(setting, monkeypatch):
    """the continuous emit kernel's delta rows (round 2): library buffer and alternating caller buffers, float32 and float64"""
    import pct_b200
    res = []
    for delta in ("0", "1"):
        monkeypatch.setenv("PCT_B200_OBS_DELTA", delta)
        n = 200
        b = pct_b200.PctBatch(n, setting, container_size=(1.0, 1.0, 1.0), continuous=True, sample_from_distribution=True, seed=12,
                              obs_dtype=torch.float64 if setting == 2 else torch.float32)
        bufs = [torch.full((n, b.obs_len), 7.0, dtype=b.obs_dtype, device=b.device) for _ in range(2)]
        out = [b.reset().clone()]
        for t in range(60):
            tgt = None if t < 30 else bufs[0 if (t // 3) % 2 else 1]  # library buffer first, then caller buffers switched every third step
            obs, _, _, info = b.step(leaf_idx=b.random_policy(5, t), out=tgt)
            out.append(obs.clone())
        assert not b.decode_info(info)["flags"].any()
        res.append(torch.stack(out).cpu().numpy())
        b.close()
    assert np.array_equal(res[0], res[1])


def test_delta_with_alternating_buffers_and_f64(monkeypatch):
    ref = _trace(1, 300, 40, False, monkeypatch, alternate=True, obs_dtype=torch.float64)
    got = _trace(1, 300, 40, True, monkeypatch, alternate=True, obs_dtype=torch.float64)
    assert np.array_equal(ref, got)


def test_delta_inside_a_captured_graph(monkeypatch):
    import pct_b200
    res = []
    for delta in ("0", "1"):
        monkeypatch.setenv("PCT_B200_OBS_DELTA", delta)
        roll = pct_b200.GraphedRollout(pct_b200.PctBatch(256, 1, item_set=ITEM_SET, seed=8), 4, policy_seed=2, use_graph=True)
        acc = []
        for _ in range(5):
            obs, rew, done, act = roll.run()
            acc.append(obs.clone())
        res.append(torch.stack(acc).cpu().numpy())
    assert np.array_equal(res[0], res[1])


def test_delta_through_the_zero_copy_host_path(monkeypatch):
    from test_zzz_gpu_host_zerocopy import _drive
    monkeypatch.setenv("PCT_B200_HOST_ZEROCOPY", "0")
    monkeypatch.setenv("PCT_B200_OBS_DELTA", "0")
    ref = _drive(1536, 1, 40, True)
    monkeypatch.setenv("PCT_B200_HOST_ZEROCOPY", "1")
    monkeypatch.setenv("PCT_B200_OBS_DELTA", "1")
    got = _drive(1536, 1, 40, True)
    assert all(np.array_equal(a, b) for a, b in zip(ref, got))
    monkeypatch.setenv("PCT_B200_HOST_ZEROCOPY", "0")  # staged host path + delta (env ranges on several streams)
    got = _drive(1536, 1, 40, True)
    assert all(np.array_equal(a, b) for a, b in zip(ref, got))
