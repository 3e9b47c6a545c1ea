"""GPU: a pct_create that fails on an allocation reports it, and leaves nothing behind that the next handle of the same thread would trip over."""
import ctypes as C

import pytest

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

ITEMS = [(i, j, k) for i in range(1, 6) for j in range(1, 6) for k in range(1, 6)]


def test_failed_create_reports_and_does_not_leak_into_the_next_handle(monkeypatch):
    import pct_b200
    from importlib import import_module
    m = import_module("pct_b200._lib")
    lib = m.lib()
    # ~4 M continuous envs: the env records alone need hundreds of GB, so their allocation fails on any device, while every buffer allocated
    # before them (item footprint rows, hand-over flags; no delta / alias state with these two switches) stays near 100 MB
    monkeypatch.setenv("PCT_B200_OBS_DELTA", "0")
    monkeypatch.setenv("PCT_B200_ALIAS", "0")
    cfg = m.Config()
    cfg.domain = m.PCT_CONTINUOUS
    cfg.setting = 1
    cfg.internal_node_holder, cfg.leaf_node_holder = 80, 50
    for i in range(3):
        cfg.container_size[i] = 1.0
    cfg.item_mode = m.PCT_ITEMS_RANDOM
    cfg.sample_from_distribution = 1
    cfg.sample_left_bound, cfg.sample_right_bound = 0.1, 0.5
    cfg.size_minimum = 0.1
    h = C.c_void_p()
    rc = lib.pct_create(C.byref(cfg), 4 << 20, 0, C.byref(h))
    assert rc == -2 and not h.value  # PCT_ERR_CUDA
    assert b"pct_create" in lib.pct_last_error(None)
    monkeypatch.undo()
    # new handles of both domains, same thread: their first reset and step succeed
    for b in (pct_b200.PctBatch(8, 1, item_set=ITEMS, seed=3),
              pct_b200.PctBatch(8, 1, container_size=(1.0, 1.0, 1.0), continuous=True, sample_from_distribution=True, seed=3)):
        b.reset()
        b.step(leaf_idx=b.random_policy(5, 0))
        torch.cuda.synchronize()
