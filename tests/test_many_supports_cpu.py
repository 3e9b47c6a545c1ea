"""CPU: the many-support scenarios of tests/many_supports.py.  (1) On the oracle: how often the stability walks of the GPU test's batch visit
nodes on more than KSUP_SMALL = 8 supports (the per-env HBM scratch and its lock), at every size up to KSUP_MAX, in both load-distribution
branches, in the ordinary and the tall walk pool — so the GPU test is known to exercise that path.  (2) Through the host build of the device
stability source (tests/host_emul/stab_host.cpp, every routine, alias mode on and off): every virtual verdict, every real placement and the
support graph after it, bit for bit against the oracle, on envs that cover every plan — what the GPU test checks, rehearsed without a GPU."""
import ctypes as C

import numpy as np
import pytest

import many_supports as M
from harness import compare_graphs
from test_host_emul_stability import lib  # noqa: F401  (the host build, a fixture)
from test_support_graph_cpu import Host

N_GPU = 1024  # envs of the GPU test's large batch
SIZES = (8, 9, 16, 25, 32)


@pytest.mark.parametrize("setting", [1, 3])
@pytest.mark.parametrize("cont", [False, True], ids=["discrete", "continuous"])
def test_coverage_of_the_many_support_path(cont, setting):
    recs = M.trajectories(cont, setting, N_GPU, census=True)
    T = M.STEPS
    own = np.zeros((N_GPU, T), dtype=int)      # walks whose placement rests on > 8 supports
    below = np.zeros((N_GPU, T), dtype=int)    # walks with a box on > 8 supports below them
    hist, branch, lstsq, tall_envs, ordinary_envs = {}, {True: 0, False: 0}, 0, 0, 0
    for e, r in enumerate(recs):
        tall = ordinary = False
        for t, c in enumerate(r["census"]):
            for k, d, tl, bb in zip(c["k"], c["direct"], c["tall"], c["below_big"]):
                if k > M.KSUP_SMALL:
                    own[e, t] += 1
                    branch[d] += 1
                if k >= M.KSUP_SMALL:
                    hist[k] = hist.get(k, 0) + 1
                below[e, t] += bb
                if k > M.KSUP_SMALL or bb:
                    tall |= tl
                    ordinary |= not tl
        tall_envs += tall
        ordinary_envs += ordinary
        inc = np.diff(np.array([0] + r["lstsq"]))
        lstsq += int(inc[inc > 0].sum())  # the count restarts with the env
    heavy = own + below
    print("\n%s setting %d, %d envs x %d steps" % ("continuous" if cont else "discrete", setting, N_GPU, T))
    print("walks per step on > 8 supports: max %d, mean %.0f; with a box on > 8 supports below: max %d, mean %.0f" % (
        own.sum(0).max(), own.sum(0).mean(), below.sum(0).max(), below.sum(0).mean()))
    print("walks by supports (8 .. 32):", dict(sorted(hist.items())))
    print("> 8 supports: direct %d, least squares %d; lstsq solves (oracle) %d; envs with such walks in the tall pool %d, ordinary pool %d" % (
        branch[True], branch[False], lstsq, tall_envs, ordinary_envs))
    assert all(hist.get(k, 0) > 0 for k in SIZES), hist
    assert branch[True] > 100 and branch[False] > 100 and lstsq > 10000
    assert own.sum(0).max() >= 1000 and heavy.sum(0).max() >= 5000
    per_env = heavy.sum(1)
    print("such walks per env: min %d (env %d), 10th percentile %d, median %d" % (per_env.min(), per_env.argmin(), np.percentile(per_env, 10),
                                                                            np.median(per_env)))
    assert per_env.min() >= 2 and np.percentile(per_env, 10) >= 10
    assert tall_envs >= N_GPU // 8 and ordinary_envs >= N_GPU // 2


def _replay(L, cont, setting, env, alias, routine):
    """the env's scenario trajectory on the oracle and on the host build in lock-step: every candidate's virtual verdict, every real placement,
    the support graph after it (auto-reset on done, like trajectory())"""
    stream, brows, _ = M.plan(cont, setting, env)
    orc = M.make_oracle(cont, setting, stream, alias)
    host = Host(L, cont, setting, M.container(cont), M.NB, alias)
    o = orc.reset()
    n_virtual = 0
    for t in range(M.STEPS):
        where = "env %d step %d" % (env, t)
        cand, feas = orc.candidates()
        den = orc.next_den
        for p, f in zip(cand, feas):
            if f < 0:
                continue
            if cont:
                got = L.shc_virtual(host.h, np.ascontiguousarray(p, dtype=np.float64).ctypes.data_as(C.POINTER(C.c_double)), den)
            else:
                got = L.sh_virtual(host.h, int(p[3] - p[0]), int(p[4] - p[1]), int(p[5] - p[2]), int(p[0]), int(p[1]), den, None)
            assert got == f, "%s candidate %s: feasible %d, oracle %d" % (where, p.tolist(), got, f)
            n_virtual += 1
        row = brows[t] if t < len(brows) else M.policy_pick(o, M.NB, M.NL, M.PSEED, env, t)[1]
        nbx = orc.next_box
        o, _, done, _ = orc.step(row)
        placed = host.place(row, nbx, den)
        assert placed == (not done), "%s real placement: placed %d, oracle done=%s" % (where, placed, done)
        compare_graphs(host.graph(), orc.support_graph(), where + ":")
        if done:
            o = orc.reset()
            host.reset()
    assert (L.shc_flags if cont else L.sh_flags)(host.h) == 0
    host.close()
    return n_virtual


ENVS = range(10)  # every plan, with and without the tall columns


@pytest.mark.parametrize("alias", [True, False], ids=["alias", "snapshot"])
@pytest.mark.parametrize("setting", [1, 3])
@pytest.mark.parametrize("cont", [False, True], ids=["discrete", "continuous"])
def test_host_build_replays_the_scenarios(lib, cont, setting, alias):
    """routines: 0 stability_check, 1 stab_virtual on the fused scan's supports (discrete), 2 stab_virtual scanning, 3 light prefix + continuation,
    4 light prefix + fork-join pieces (tests/test_host_emul_stability.py)"""
    tot = 0
    try:
        for routine in ((0, 2, 3, 4) if cont else (0, 1, 2, 3, 4)):
            lib.sh_use_v2(routine)
            for env in ENVS:
                try:
                    tot += _replay(lib, cont, setting, env, alias, routine)
                except AssertionError as ex:
                    raise AssertionError("routine %d, %s" % (routine, ex)) from None
    finally:
        lib.sh_use_v2(0)
    print("virtual verdicts compared:", tot)
    assert tot > 20000
