"""CPU: the buffered-packing surface that needs no device — the C ABI declarations and exports, the ctypes binding, and the helper that
fits the reference's DRL_GAT to a buffered observation."""
import os
import re
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CALLS = ["pct_set_buffer", "pct_buffer_obs_len", "pct_buffer_reset", "pct_buffer_step", "pct_buffer_items", "pct_buffer_policy_random"]


def test_header_declares_the_buffered_calls():
    src = open(os.path.join(ROOT, "include", "pct_b200.h")).read()
    for name in CALLS:
        assert re.search(r"\b%s\(pct_handle h" % name, src), name


def test_binding_exports_the_buffered_calls():
    from pct_b200 import _lib
    assert set(CALLS) <= set(_lib.EXPORTS)
    src = open(os.path.join(ROOT, "online-3d-bpp-pct_b200", "_lib.py")).read()
    for name in CALLS:
        assert "L.%s.argtypes" % name in src, name


def test_buffered_drl_gat_sets_the_encoder_graph_size():
    from pct_b200.rollout import buffered_drl_gat
    net = types.SimpleNamespace(actor=types.SimpleNamespace(embedder=types.SimpleNamespace(graph_size=131)))
    assert buffered_drl_gat(net, 3, 80, 50) is net
    assert net.actor.embedder.graph_size == 80 + 3 * 50 + 3
    buffered_drl_gat(net, 1, 80, 50)
    assert net.actor.embedder.graph_size == 131  # B = 1: the plain observation's node count
