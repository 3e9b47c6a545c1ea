"""CPU: the DEVICE stability routine (csrc/pct_stability.cuh: the explicit DFS, edge pool, hull / point-in-polygon / lstsq code the
kernels compile) built for the HOST by g++ (tests/host_emul/stab_host.cpp, intrinsics shimmed, -ffp-contract=off) and driven through
whole trajectories next to the CPU oracle: every real placement's verdict (stability_check<true>, with load persistence) and every
virtual feasibility verdict of every candidate (stability_check<false>) must equal the oracle's — which is pinned on
the reference.  This checks the kernels' SOURCE logic without a GPU; warp-level code, staging and SASS remain the GPU tests' business."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from harness import CASES, ITEM_SET, case_stream, make_stream, policy_pick
from pct_oracle import OracleDiscrete

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host_emul", "stab_host.cpp")
OUT = os.path.join(ROOT, "tests", "host_emul", "_build", "libstab_host.so")
CSRC = os.path.join(ROOT, "online-3d-bpp-pct_b200", "csrc")


def _cuda_include():
    for d in (os.environ.get("CUDA_HOME"), "/usr/local/cuda"):
        if d and os.path.isfile(os.path.join(d, "include", "cuda_runtime.h")):
            return os.path.join(d, "include")
    return None


@pytest.fixture(scope="module")
def lib():
    inc = _cuda_include()
    if inc is None:
        pytest.skip("CUDA headers not found")
    deps = [SRC] + [os.path.join(CSRC, f) for f in ("pct_stability.cuh", "pct_geom.cuh", "pct_geom_continuous.cuh", "pct_kernels.h", "pct_pyhash.cuh", "pct_support_graph.h")]
    if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in deps):
        os.makedirs(os.path.dirname(OUT), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-w", "-I" + CSRC,
                               "-I" + os.path.join(ROOT, "include"), "-I" + inc, "-o", OUT, SRC])
    L = C.CDLL(OUT)
    L.sh_create.restype = C.c_void_p
    L.sh_create.argtypes = [C.c_int] * 4
    for f in ("sh_destroy", "sh_reset"):
        getattr(L, f).argtypes = [C.c_void_p]
    L.sh_flags.argtypes = [C.c_void_p]
    L.sh_virtual.argtypes = [C.c_void_p] + [C.c_int] * 5 + [C.c_double, C.POINTER(C.c_int)]
    L.sh_place.argtypes = [C.c_void_p] + [C.c_int] * 5 + [C.c_double]
    L.sh_set_alias.argtypes = [C.c_void_p, C.c_int]
    L.sh_set_holder.argtypes = [C.c_void_p, C.c_int]
    L.sh_use_v2.argtypes = [C.c_int]
    dp = C.POINTER(C.c_double)
    L.shc_create.restype = C.c_void_p
    L.shc_create.argtypes = [C.c_int, C.c_double, C.c_double, C.c_double]
    for f in ("shc_destroy", "shc_reset", "shc_flags"):
        getattr(L, f).argtypes = [C.c_void_p]
    L.shc_set_alias.argtypes = [C.c_void_p, C.c_int]
    L.shc_virtual.argtypes = [C.c_void_p, dp, C.c_double]
    L.shc_place_row.argtypes = [C.c_void_p, dp, dp, C.c_double]
    for f in ("sh_support_graph", "shc_support_graph"):
        getattr(L, f).argtypes = [C.c_void_p, C.c_void_p, C.c_char_p, C.c_int]
    for f in ("sh_pool_field", "shc_pool_field"):
        getattr(L, f).restype = C.c_void_p
        getattr(L, f).argtypes = [C.c_void_p, C.c_int]
    return L


@pytest.fixture(autouse=True)
def _default_routine(lib):
    lib.sh_use_v2(0)
    yield
    lib.sh_use_v2(0)


def _placement(row, next_box):
    """LeafNode2Action (D:bin3D.py:139-150)"""
    if np.sum(row[0:6]) == 0:
        return tuple(next_box), 0, 0
    x, y = int(row[3] - row[0]), int(row[4] - row[1])
    z = list(next_box)
    z.remove(x)
    z.remove(y)
    return (x, y, int(z[0])), int(row[0]), int(row[1])


def _drive(L, env, setting, container, nb, nl, seed, env_id, steps, alias=True):  # alias: the default semantics of oracle and kernels since round 2
    h = L.sh_create(setting, *container)
    L.sh_set_holder(h, nb)
    L.sh_set_alias(h, int(alias))
    L.sh_reset(h)
    o = env.reset()
    n_virtual = n_real = 0
    for t in range(steps):
        cand, feas = env.candidates()
        den = env.next_den
        for p, f in zip(cand, feas):
            if f < 0:
                continue  # beyond the leaf cap: the reference never evaluated it
            mh = C.c_int()  # the item drops to the resting height of its footprint, whatever z the candidate tuple carries (the EMS's)
            got = L.sh_virtual(h, int(p[3] - p[0]), int(p[4] - p[1]), int(p[5] - p[2]), int(p[0]), int(p[1]), den, C.byref(mh))
            assert got == f, "step %d candidate %s: host build %d (rest %d), oracle %d" % (t, p.tolist(), got, mh.value, f)
            n_virtual += 1
        _, row = policy_pick(o, nb, nl, seed, env_id, t)
        (x, y, z), lx, ly = _placement(row, env.next_box)
        o, _, done, _ = env.step(row)
        placed = L.sh_place(h, x, y, z, lx, ly, den)
        assert placed == (not done), "step %d real placement: host build %d, oracle done=%s" % (t, placed, done)
        n_real += 1
        if done:
            # the terminal observation (gym.Env semantics): the virtual checks run on the state the FAILED real placement left behind
            cand, feas = env.candidates()
            for p, f in zip(cand, feas):
                if f >= 0:
                    got = L.sh_virtual(h, int(p[3] - p[0]), int(p[4] - p[1]), int(p[5] - p[2]), int(p[0]), int(p[1]), env.next_den, None)
                    assert got == f, "terminal observation after step %d, candidate %s: host build %d, oracle %d" % (t, p.tolist(), got, f)
            o = env.reset()
            L.sh_reset(h)
    assert L.sh_flags(h) == 0
    L.sh_destroy(h)
    return n_virtual, n_real


# routine: 0 = stability_check<false> (K1's twin, heuristics, round 1's block kernel), 1 = stab_virtual with the supports of the fused
# resting-height scan, 2 = stab_virtual scanning the supports itself, 3 = stab_light + stab_virtual continuation (the sequential walk kernels),
# 4 = stab_light + stab_piece pieces from a queue, verdict = AND (the fork-join walk kernel)
@pytest.mark.parametrize("routine", [0, 1, 2, 3, 4], ids=["stability_check", "stab_virtual_fused", "stab_virtual_scan", "light_then_continuation", "fork_join"])
@pytest.mark.parametrize("setting", [1, 3, 2])
def test_device_stability_source_follows_the_oracle(lib, setting, routine):
    lib.sh_use_v2(routine)
    tot = 0
    for env_id in range(6):
        seed = 300 + setting
        env = OracleDiscrete(setting, stream=make_stream(seed, env_id, 700, setting))
        nv, nr = _drive(lib, env, setting, (10, 10, 10), 80, 50, seed, env_id, 350)
        tot += nv
    assert tot > 20000


@pytest.mark.parametrize("routine", [0, 1, 3, 4], ids=["stability_check", "stab_virtual_fused", "light_then_continuation", "fork_join"])
@pytest.mark.parametrize("name", ["big_s1", "dense16_s1", "flat_s1", "holders_s1"])
def test_device_stability_source_on_other_configurations(lib, name, routine):
    lib.sh_use_v2(routine)
    c = CASES[name]
    env = OracleDiscrete(c["setting"], container_size=c["container"], internal_node_holder=c["nb"], leaf_node_holder=c["nl"],
                         size_minimum=min(min(i) for i in c["items"]), stream=case_stream(c, 91, 2, 600))
    _drive(lib, env, c["setting"], c["container"], c["nb"], c["nl"], 91, 2, 300)


# ---- the ALIAS variant (stability_check<true, G, ALIAS = true>: the reference's object semantics of the load entries, DESIGN.md
# section 3 (b)) against the oracle's alias mode.  The trajectories below are the ones on which the two semantics part
# (scratch/alias_rate.py: BASELINE item streams seed 1234, policy seed 4321): the snapshot build must follow the snapshot oracle and the
# ALIAS build the alias oracle THROUGH the step where they part, and the two oracles must indeed part there. ----------------------------
DIVERGING = [(1, 126, 39), (1, 835, 167), (3, 92, 103)]  # (setting, env id, step of the first difference)


@pytest.mark.parametrize("setting,env_id,step", DIVERGING)
@pytest.mark.parametrize("alias", [False, True], ids=["snapshot", "alias"])
def test_alias_variant_follows_the_alias_oracle(lib, setting, env_id, step, alias):
    env = OracleDiscrete(setting, stream=make_stream(1234, env_id, 600, setting))
    env.set_alias_mode(alias)
    _drive(lib, env, setting, (10, 10, 10), 80, 50, 4321, env_id, step + 25, alias=alias)


@pytest.mark.parametrize("setting,env_id,step", DIVERGING)
def test_the_two_semantics_part_on_these_trajectories(setting, env_id, step):
    a, b = (OracleDiscrete(setting, stream=make_stream(1234, env_id, 600, setting)) for _ in range(2))
    a.set_alias_mode(False)
    b.set_alias_mode(True)
    oa, ob = a.reset(), b.reset()
    for t in range(step + 1):
        assert np.array_equal(oa, ob), t
        _, row = policy_pick(oa, 80, 50, 4321, env_id, t)
        oa, _, da, _ = a.step(row)
        ob, _, db, _ = b.step(row)
        if t < step and da:
            oa, ob = a.reset(), b.reset()
    assert da != db or not np.array_equal(oa, ob)


@pytest.mark.parametrize("setting", [1, 3])
def test_alias_variant_on_ordinary_trajectories(lib, setting):
    for env_id in range(4):
        env = OracleDiscrete(setting, stream=make_stream(300 + setting, env_id, 700, setting))
        env.set_alias_mode(True)
        _drive(lib, env, setting, (10, 10, 10), 80, 50, 300 + setting, env_id, 300, alias=True)


def test_cross_check_is_sensitive(lib):
    """the snapshot build does NOT follow the alias oracle on a diverging trajectory (so the agreement above means something)"""
    setting, env_id, step = DIVERGING[0]
    env = OracleDiscrete(setting, stream=make_stream(1234, env_id, 600, setting))
    env.set_alias_mode(True)
    with pytest.raises(AssertionError):
        _drive(lib, env, setting, (10, 10, 10), 80, 50, 4321, env_id, step + 25, alias=False)


# ---- continuous domain: GeomC + the float64 resting-height / rounding code, against the continuous oracle -------------------------------
def _dpc(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _drive_c(L, env, setting, container, seed, env_id, steps, alias=True):
    h = L.shc_create(setting, *container)
    L.shc_set_alias(h, int(alias))
    L.shc_reset(h)
    o = env.reset()
    n_virtual = 0
    for t in range(steps):
        cand, feas = env.candidates()
        den = env.next_den
        for p, f in zip(cand, feas):
            if f < 0:
                continue
            got = L.shc_virtual(h, _dpc(np.ascontiguousarray(p, dtype=np.float64)), den)
            assert got == f, "step %d candidate %s: host build %d, oracle %d" % (t, p.tolist(), got, f)
            n_virtual += 1
        _, row = policy_pick(o, 80, 50, seed, env_id, t)
        nb = np.array(env.next_box, dtype=np.float64)
        o, _, done, _ = env.step(row)
        placed = L.shc_place_row(h, _dpc(np.ascontiguousarray(row[:6], dtype=np.float64)), _dpc(nb), den)
        assert placed == (not done), "step %d real placement: host build %d, oracle done=%s" % (t, placed, done)
        if done:
            cand, feas = env.candidates()  # terminal observation: virtual checks on the state the failed real placement left behind
            for p, f in zip(cand, feas):
                if f >= 0:
                    got = L.shc_virtual(h, _dpc(np.ascontiguousarray(p, dtype=np.float64)), env.next_den)
                    assert got == f, "terminal observation after step %d, candidate %s: host build %d, oracle %d" % (t, p.tolist(), got, f)
            o = env.reset()
            L.shc_reset(h)
    assert L.shc_flags(h) == 0
    L.shc_destroy(h)
    return n_virtual


@pytest.mark.parametrize("routine", [0, 2, 3, 4], ids=["stability_check", "stab_virtual_scan", "classify_light_continuation", "fork_join"])
@pytest.mark.parametrize("setting", [1, 3, 2])
def test_device_stability_source_follows_the_continuous_oracle(lib, setting, routine):
    from pct_oracle import OracleContinuous, make_continuous_stream
    lib.sh_use_v2(routine)
    tot = 0
    for env_id in range(4):
        env = OracleContinuous(setting, stream=make_continuous_stream(77 + setting, env_id, 600, setting))
        tot += _drive_c(lib, env, setting, (1.0, 1.0, 1.0), 77 + setting, env_id, 250)
    assert tot > 10000


DIVERGING_C = [(1, 1, 169), (1, 548, 152), (1, 597, 103), (1, 638, 163), (3, 635, 215)]  # scratch/alias_rate.py, continuous streams


@pytest.mark.parametrize("setting,env_id,step", DIVERGING_C)
@pytest.mark.parametrize("alias", [False, True], ids=["snapshot", "alias"])
def test_alias_variant_follows_the_alias_oracle_continuous(lib, setting, env_id, step, alias):
    from pct_oracle import OracleContinuous, make_continuous_stream
    env = OracleContinuous(setting, stream=make_continuous_stream(1234, env_id, 600, setting))
    env.set_alias_mode(alias)
    _drive_c(lib, env, setting, (1.0, 1.0, 1.0), 4321, env_id, step + 20, alias=alias)


def test_cross_check_is_sensitive_continuous(lib):
    from pct_oracle import OracleContinuous, make_continuous_stream
    setting, env_id, step = DIVERGING_C[0]
    env = OracleContinuous(setting, stream=make_continuous_stream(1234, env_id, 600, setting))
    env.set_alias_mode(True)
    with pytest.raises(AssertionError):
        _drive_c(lib, env, setting, (1.0, 1.0, 1.0), 4321, env_id, step + 20, alias=False)


def test_terminal_observations_need_the_load_sync(lib, monkeypatch):
    """after a FAILED real placement the ALIAS apply kernel brings the stored snapshots in line with the objects (alias_sync_loads), which
    is what lets the snapshot-only read-only checks reproduce the reference's terminal observation; without it they do not"""
    monkeypatch.setenv("PCT_HOST_EMUL_NO_SYNC", "1")
    failing = 0
    for setting, env_id, step in DIVERGING:
        env = OracleDiscrete(setting, stream=make_stream(1234, env_id, 600, setting))
        env.set_alias_mode(True)
        try:
            _drive(lib, env, setting, (10, 10, 10), 80, 50, 4321, env_id, step + 25, alias=True)
        except AssertionError as ex:
            assert "terminal observation" in str(ex)
            failing += 1
    assert failing >= 2


def test_fast_around6_equals_the_division(lib):
    """around6 (csrc/pct_geom_continuous.cuh) divides by 1e6 with one FMA correction instead of the IEEE division subroutine; it must equal
    np.around(v, 6) = rint(v * 1e6) / 1e6 bit for bit.  Exhaustive proof over every integer numerator |a| <= 2.2e9: scratch/around6_exhaustive.c;
    here: random, half-way, huge (fallback path) and tiny operands through the host build of the device function."""
    lib.sh_around6.restype = C.c_double
    lib.sh_around6.argtypes = [C.c_double]
    rng = np.random.default_rng(11)
    k = rng.integers(-3000000, 3000000, 20000).astype(np.float64)
    vals = np.concatenate([rng.uniform(-3, 3, 60000), rng.uniform(-2300, 2300, 20000), (k + 0.5) / 1e6, np.nextafter((k + 0.5) / 1e6, 9.0),
                           rng.uniform(-1e7, 1e7, 5000), [0.0, -0.0, 1e-7, 4.9999995e-7, 5e-7, 2199.9999995, 2200.0000005, 1e12, -1e12]])
    want = np.rint(vals * 1e6) / 1e6
    got = np.array([lib.sh_around6(float(v)) for v in vals])
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))


def test_integer_hash_double_equals_cpython(lib):
    """hash_double (csrc/pct_pyhash.cuh: _Py_HashDouble as a 61-bit rotation of the integer mantissa) against Python's own hash() of the float — the
    value CPython feeds into the tuple hash that orders the continuous candidate set (C:space.py:563-567) — and against the frexp-loop restatement."""
    lib.sh_hash_double.restype = C.c_longlong
    lib.sh_hash_double.argtypes = [C.c_double, C.c_int]
    rng = np.random.default_rng(3)
    vals = np.concatenate([rng.uniform(-3, 3, 40000), np.round(rng.uniform(0, 1, 40000), 3), np.round(rng.uniform(0, 2.5, 20000), 6),
                           rng.integers(-10**6, 10**6, 5000).astype(np.float64), 2.0 ** rng.integers(-60, 60, 2000), rng.uniform(-1e12, 1e12, 5000),
                           [0.0, -0.0, 1.0, -1.0, 0.5, 0.1, 0.30000000000000004, 1e-300, 5e-324, 2.0 ** 61, 2.0 ** 61 - 1, float(2 ** 61 - 1) * 3, 1e308]])
    for v in vals:
        v = float(v)
        assert lib.sh_hash_double(v, 0) == hash(v) == lib.sh_hash_double(v, 1), v
