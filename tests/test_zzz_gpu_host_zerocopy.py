"""GPU: the zero-copy (default since round 2) observation delivery of pct_step_host (PCT_B200_HOST_ZEROCOPY=1: the kernels write the observation
straight into the pinned host buffer) must return exactly what the staged path returns, and fall back to it for unpinned buffers.

Zero-copy is the default of pct_step_host.
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
from harness import ITEM_SET  # noqa: E402

pytestmark = pytest.mark.gpu


def _drive(n, setting, steps, pinned, continuous=False):
    import pct_b200
    if continuous:
        b = pct_b200.PctBatch(n, setting, container_size=(1.0, 1.0, 1.0), continuous=True, sample_from_distribution=True, seed=9)
    else:
        b = pct_b200.PctBatch(n, setting, item_set=ITEM_SET, seed=9)
    mk = (lambda shape, dt: torch.empty(shape, dtype=dt, pin_memory=True).numpy()) if pinned else (lambda shape, dt: torch.empty(shape, dtype=dt).numpy())
    obs, rew, done = mk((n, b.obs_len), torch.float32), mk((n,), torch.float32), mk((n,), torch.uint8)
    info, idx = mk((n, 8), torch.int32), mk((n,), torch.int32)
    b.reset_host(obs)
    out = [obs.copy()]
    rng = np.random.RandomState(4)
    for t in range(steps):
        nvalid = (obs.reshape(n, -1, 9)[:, b.nb:b.nb + b.nl, 8] == 1).sum(1)
        idx[:] = (rng.randint(0, 1 << 30, n) % np.maximum(nvalid, 1)).astype(np.int32)
        b.step_host(obs, rew, done, info, leaf_idx=idx)
        # every byte of the info records too (as 16-bit halves, exact in float32)
        out.append(np.concatenate([obs.ravel(), rew, done.astype(np.float32), info.view(np.uint16).ravel().astype(np.float32)]))
    b.close()
    return out


@pytest.mark.parametrize("setting,n,continuous", [(1, 2048, False), (2, 1500, False), (1, 600, True)])
def test_zero_copy_equals_staged(setting, n, continuous, monkeypatch):
    monkeypatch.setenv("PCT_B200_HOST_ZEROCOPY", "0")
    ref = _drive(n, setting, 40, True, continuous)
    monkeypatch.setenv("PCT_B200_HOST_ZEROCOPY", "1")
    got = _drive(n, setting, 40, True, continuous)
    assert all(np.array_equal(a, b) for a, b in zip(ref, got))
    got = _drive(n, setting, 10, False, continuous)  # pageable buffers: the staged path serves them
    assert all(np.array_equal(a, b) for a, b in zip(ref[:11], got))
