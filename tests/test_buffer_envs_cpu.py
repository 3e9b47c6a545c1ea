"""CPU: the selected-env and snapshot calls of buffered handles need no device for their declarations and their binding."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CALLS = ["pct_buffer_step_envs", "pct_buffer_reset_envs", "pct_buffer_snapshot_bytes", "pct_buffer_snapshot", "pct_buffer_restore"]


def test_header_declares_the_calls():
    src = open(os.path.join(ROOT, "include", "pct_b200.h")).read()
    for name in CALLS:
        assert re.search(r"\b%s\(pct_handle h" % name, src), name
    assert re.search(r"int64_t pct_buffer_snapshot_bytes\(pct_handle h\)", src)


def test_binding_exports_the_calls():
    from pct_b200 import _lib
    assert set(CALLS) <= set(_lib.EXPORTS)
    src = open(os.path.join(ROOT, "online-3d-bpp-pct_b200", "_lib.py")).read()
    for name in CALLS:
        assert "L.%s.argtypes" % name in src, name
    assert "L.pct_buffer_snapshot_bytes.restype = i64" in src


def test_batch_has_the_methods():
    from pct_b200 import PctBatch
    for name in ("buffer_step_envs", "buffer_reset_envs", "buffer_snapshot", "buffer_restore"):
        assert callable(getattr(PctBatch, name)), name
    assert isinstance(PctBatch.buffer_snapshot_bytes, property)
