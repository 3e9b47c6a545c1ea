"""CPU: the C-ABI shared library loads, exports every function include/pct_b200.h declares, its structs have the layout
the ctypes binding assumes, and it fails loudly (no CPU fallback) when there is no GPU.  No compute calls."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    import pct_b200
    if not os.path.exists(pct_b200.LIB_PATH):
        pct_b200.build()
    return C.CDLL(pct_b200.LIB_PATH)


def test_every_declared_symbol_is_exported():
    hdr = open(os.path.join(ROOT, "include", "pct_b200.h")).read()
    body = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    names = re.findall(r"\b(pct_[a-z0-9_]+)\s*\(", body)
    assert len(set(names)) >= 16
    lib = _lib()
    for n in sorted(set(names)):
        assert hasattr(lib, n), "missing export %s" % n
    from importlib import import_module
    assert set(import_module("pct_b200._lib").EXPORTS) <= set(names)


def test_struct_layouts_match_header():
    from importlib import import_module
    m = import_module("pct_b200._lib")
    assert C.sizeof(m.StepInfo) == 32
    assert C.sizeof(m.StateDump) == 16 + 8 + 24 + 8 + 80 * 7 * 8 + 256 * 6 * 8
    assert C.sizeof(m.SupportGraph) == 4 * (6 + 5 * 82 + 3 * 256) + 8 * (256 * 4 + 256 * 2 + 82 * 2 + 82 * 4) == 20960
    assert C.sizeof(m.Config) == 112  # + shuffle (round 2); pct_api.cu static_asserts the C side


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from importlib import import_module
    m = import_module("pct_b200._lib")
    lib = m.lib()
    cfg = m.Config()
    cfg.setting = 1
    cfg.internal_node_holder, cfg.leaf_node_holder = 80, 50
    for i in range(3):
        cfg.container_size[i] = 10
    h = C.c_void_p()
    rc = lib.pct_create(C.byref(cfg), 4, 0, C.byref(h))
    assert rc == -3 and b"no CPU fallback" in lib.pct_last_error(None)
    import pct_b200
    with pytest.raises(pct_b200.PctError):
        pct_b200.PctBatch(4, 1)
