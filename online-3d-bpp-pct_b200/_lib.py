"""ctypes binding of the C ABI declared in include/pct_b200.h (libpct_b200.so, built in-tree by csrc/Makefile).

The library is the product: if it is missing this module raises — there is no Python / CPU fallback."""
import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("PCT_B200_LIB", os.path.join(_HERE, "libpct_b200.so"))  # env override: tuning experiments only

PCT_DISCRETE, PCT_CONTINUOUS = 0, 1
PCT_F32, PCT_F64 = 0, 1
PCT_ITEMS_RANDOM, PCT_ITEMS_STREAM = 0, 1
FLAG_NAMES = {1: "box_overflow", 2: "bad_action", 4: "ems_overflow", 8: "cand_overflow", 16: "edge_overflow", 32: "support_overflow",
              64: "sync_timeout", 128: "bad_snapshot"}


class Config(C.Structure):
    _fields_ = [("domain", C.c_int32), ("setting", C.c_int32), ("container_size", C.c_double * 3),
                ("internal_node_holder", C.c_int32), ("leaf_node_holder", C.c_int32), ("obs_dtype", C.c_int32),
                ("item_mode", C.c_int32), ("size_minimum", C.c_double), ("sample_from_distribution", C.c_int32),
                ("sample_left_bound", C.c_double), ("sample_right_bound", C.c_double), ("seed", C.c_uint64),
                ("env_id_base", C.c_int64), ("no_auto_reset", C.c_int32), ("lnes", C.c_int32), ("shuffle", C.c_int32)]


LNES_CODES = {"EMS": 0, "EV": 1, "EP": 2, "CP": 3, "FC": 4, "EVM": 5}
HEURISTIC_CODES = {"LSAH": 0, "OnlineBPH": 1, "BR": 2, "MACS": 3, "DBL": 4, "HM": 5, "RANDOM": 6}  # heuristic.py:593-606 names


class StepInfo(C.Structure):
    _fields_ = [("counter", C.c_int32), ("flags", C.c_int32), ("ratio", C.c_float), ("ep_reward", C.c_float),
                ("ep_len", C.c_int32), ("n_leaf", C.c_int32), ("n_cand", C.c_int32), ("n_ems", C.c_int32)]


class StateDump(C.Structure):
    _fields_ = [("n_boxes", C.c_int32), ("n_ems", C.c_int32), ("n_leaf", C.c_int32), ("flags", C.c_int32),
                ("draw_pos", C.c_int64), ("next_box", C.c_double * 3), ("next_den", C.c_double),
                ("boxes", (C.c_double * 7) * 80), ("ems", (C.c_double * 6) * 256)]


class SupportGraph(C.Structure):
    _fields_ = [("n_box", C.c_int32), ("n_edge", C.c_int32), ("n_poly", C.c_int32), ("alias", C.c_int32), ("alias_stale", C.c_int32), ("pad_", C.c_int32),
                ("sup_off", C.c_int32 * 82), ("load_off", C.c_int32 * 82), ("poly_off", C.c_int32 * 82), ("poly_pos", C.c_int32 * 82),
                ("has_split", C.c_int32 * 82), ("sup", C.c_int32 * 256), ("load_upper", C.c_int32 * 256), ("load_alias", C.c_int32 * 256),
                ("load", (C.c_double * 4) * 256), ("poly", (C.c_double * 2) * 256), ("split", (C.c_double * 2) * 82),
                ("own_stack", (C.c_double * 4) * 82)]


def graph_to_dict(d):
    """pct_support_graph -> the canonical per-env form (tests/harness.py): lists per placed box, floats as numpy float64"""
    import numpy as np
    f = lambda name: np.ctypeslib.as_array(getattr(d, name)).copy()
    nb = d.n_box
    so, lo, po = f("sup_off"), f("load_off"), f("poly_off")
    sup, up, al, load, poly, split, own = f("sup"), f("load_upper"), f("load_alias"), f("load"), f("poly"), f("split"), f("own_stack")
    return dict(n_box=nb, n_edge=d.n_edge, n_poly=d.n_poly, alias=bool(d.alias), alias_stale=d.alias_stale,
                supports=[sup[so[u]:so[u + 1]].tolist() for u in range(nb)],
                load_upper=[up[lo[u]:lo[u + 1]].tolist() for u in range(nb)], load_alias=[al[lo[u]:lo[u + 1]].tolist() for u in range(nb)],
                loads=[load[lo[u]:lo[u + 1]] for u in range(nb)], polygon=[poly[po[u]:po[u + 1]] for u in range(nb)],
                poly_pos=f("poly_pos")[:nb].tolist(), split=[split[u] if d.has_split[u] else None for u in range(nb)],
                own_stack=own[:nb] if d.alias else None)


EXPORTS = ["pct_create", "pct_destroy", "pct_last_error", "pct_set_item_set", "pct_set_item_stream", "pct_set_trajectory_length", "pct_reset", "pct_step",
           "pct_step_host", "pct_reset_host", "pct_policy_random", "pct_policy_random_dev", "pct_get_state", "pct_obs_len", "pct_num_envs",
           "pct_state_bytes_per_env", "pct_kernel_launches", "pct_version", "pct_profile_enable", "pct_profile_read", "pct_heuristic_actions",
           "pct_heuristic_actions_f64", "pct_query_placement", "pct_query_placement_f64",
           "pct_snapshot_bytes", "pct_snapshot", "pct_restore", "pct_query_placements", "pct_query_placements_f64", "pct_height_maps",
           "pct_preview_items", "pct_set_items", "pct_expand_items", "pct_reset_envs", "pct_get_support_graph",
           "pct_step_envs", "pct_reset_envs_only", "pct_set_items_only", "pct_set_buffer", "pct_buffer_obs_len", "pct_buffer_reset",
           "pct_buffer_step", "pct_buffer_items", "pct_buffer_policy_random", "pct_buffer_step_envs", "pct_buffer_reset_envs",
           "pct_buffer_snapshot_bytes", "pct_buffer_snapshot", "pct_buffer_restore", "pct_buffer_preview_items", "pct_buffer_set_items",
           "pct_buffer_heuristic_actions", "pct_buffer_heuristic_actions_f64", "pct_buffer_step_rows"]


def build(verbose=False):
    """Compile csrc/*.cu for sm_90a into libpct_b200.so (nvcc cross-compiles without a GPU)."""
    subprocess.check_call(["make", "-C", os.path.join(_HERE, "csrc")] + ([] if verbose else ["-s"]))
    return LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("pct_b200: %s is missing — run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU fallback)" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp, i32, i64, u64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64
    L.pct_create.argtypes = [C.POINTER(Config), i32, i32, C.POINTER(vp)]
    L.pct_destroy.argtypes = [vp]
    L.pct_destroy.restype = None
    L.pct_last_error.argtypes = [vp]
    L.pct_last_error.restype = C.c_char_p
    L.pct_set_item_set.argtypes = [vp, C.POINTER(C.c_double), i32]
    L.pct_set_item_stream.argtypes = [vp, C.POINTER(C.c_double), i32]
    L.pct_set_trajectory_length.argtypes = [vp, i32]
    L.pct_reset.argtypes = [vp, vp, vp]
    L.pct_step.argtypes = [vp, vp, i32, vp, vp, vp, vp, vp, vp]
    L.pct_step_host.argtypes = [vp, vp, i32, vp, vp, vp, vp, vp]
    L.pct_reset_host.argtypes = [vp, vp]
    L.pct_policy_random.argtypes = [vp, vp, u64, i64, vp]
    L.pct_policy_random_dev.argtypes = [vp, vp, u64, vp, vp]
    L.pct_get_state.argtypes = [vp, i32, C.POINTER(StateDump)]
    L.pct_get_support_graph.argtypes = [vp, i32, C.POINTER(SupportGraph)]
    L.pct_obs_len.argtypes = [vp]
    L.pct_num_envs.argtypes = [vp]
    L.pct_state_bytes_per_env.argtypes = [vp]
    L.pct_state_bytes_per_env.restype = i64
    L.pct_kernel_launches.argtypes = [vp]
    L.pct_kernel_launches.restype = i64
    L.pct_version.restype = C.c_char_p
    L.pct_profile_enable.argtypes = [vp, i32]
    L.pct_profile_read.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(i32)]
    L.pct_heuristic_actions.argtypes = [vp, i32, vp, u64, i64, vp]
    L.pct_heuristic_actions_f64.argtypes = [vp, i32, vp, vp]
    L.pct_query_placement.argtypes = [vp, i32, C.POINTER(i32), i32, i32, C.c_double, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]
    L.pct_query_placement_f64.argtypes = [vp, i32, C.POINTER(C.c_double), C.c_double, C.c_double, C.c_double, C.POINTER(i32),
                                          C.POINTER(C.c_double)]
    L.pct_snapshot_bytes.argtypes = [vp]
    L.pct_snapshot_bytes.restype = i64
    L.pct_snapshot.argtypes = [vp, vp, i32, vp, vp]
    L.pct_restore.argtypes = [vp, vp, vp, i32, vp, vp, vp]
    L.pct_query_placements.argtypes = [vp, vp, i32, i32, vp, vp, vp, vp, vp]
    L.pct_query_placements_f64.argtypes = [vp, vp, i32, i32, vp, vp, vp, vp, vp]
    L.pct_height_maps.argtypes = [vp, vp, i32, vp, vp]
    L.pct_preview_items.argtypes = [vp, vp, i32, i32, vp, vp]
    L.pct_set_items.argtypes = [vp, vp, i32, vp, vp, vp, vp, vp]
    L.pct_expand_items.argtypes = [vp, vp, i32, i32, vp, vp, vp, vp, vp]
    L.pct_reset_envs.argtypes = [vp, vp, i32, vp, vp, vp, vp]
    L.pct_step_envs.argtypes = [vp, vp, i32, vp, vp, i32, vp, vp, vp, vp, vp, vp]
    L.pct_reset_envs_only.argtypes = [vp, vp, i32, vp, vp, vp, vp]
    L.pct_set_items_only.argtypes = [vp, vp, i32, vp, vp, vp, vp, vp]
    L.pct_set_buffer.argtypes = [vp, i32]
    L.pct_buffer_obs_len.argtypes = [vp]
    L.pct_buffer_reset.argtypes = [vp, vp, vp, vp]
    L.pct_buffer_step.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    L.pct_buffer_items.argtypes = [vp, vp, i32, vp, vp]
    L.pct_buffer_policy_random.argtypes = [vp, vp, u64, vp, vp]
    L.pct_buffer_step_envs.argtypes = [vp, vp, i32, vp, vp, vp, vp, vp, vp, vp]
    L.pct_buffer_reset_envs.argtypes = [vp, vp, i32, vp, vp, vp, vp]
    L.pct_buffer_snapshot_bytes.argtypes = [vp]
    L.pct_buffer_snapshot_bytes.restype = i64
    L.pct_buffer_snapshot.argtypes = [vp, vp, i32, vp, vp]
    L.pct_buffer_restore.argtypes = [vp, vp, vp, i32, vp, vp, vp]
    L.pct_buffer_preview_items.argtypes = [vp, vp, i32, i32, vp, vp]
    L.pct_buffer_set_items.argtypes = [vp, vp, i32, vp, vp, vp, vp]
    L.pct_buffer_heuristic_actions.argtypes = [vp, i32, vp, vp, u64, i64, vp]
    L.pct_buffer_heuristic_actions_f64.argtypes = [vp, i32, vp, vp, vp]
    L.pct_buffer_step_rows.argtypes = [vp, vp, vp, i32, vp, vp, vp, vp, vp]
    _lib = L
    return L
