"""Scenarios whose stability walks visit nodes on MORE than KSUP_SMALL = 8 supports (test infrastructure).

At that size the hull, the contact rectangles and the least-squares split of a visit no longer fit the lane-local arrays: they move to the env's
one scratch in HBM (BigScratch, csrc/pct_kernels.h), which a per-env lock serialises, and the walks of one env sit in different warps and SMs.
Random-policy trajectories almost never get there, so each env here lays floors of small boxes ("patches": a grid of columns of one height) by
explicit placement rows, puts larger items on some of them, and then continues under the shared policy with a stream of large flat items, so that
many candidates of every env rest on > 8 supports, real placements land on them and virtual walks descend through the placed many-support boxes.

    supports      a patch of nx x ny columns under an item of the same footprint: 8 (2 x 4), 9 (3 x 3), 16 (4 x 4), 25 (5 x 5), 32 (4 x 8 = KSUP_MAX)
    branches      odd x odd footprints put the centre of mass strictly inside the middle column (direct), the others on a grid corner (least squares)
    variation     the plan (which patches, which of them get their item), a permuted floor order (scan order = support order = the least-squares
                  row order), column heights 1 and 2, the item sequence; every fourth env builds columns 0.6 H (discrete) / 0.625 H (continuous)
                  high, so that its walks rest at >= 0.6 H and go to the tall pool of the continuation kernel (a batch has one container)
    domains       discrete: cells of 1 in the 10 x 10 x 10 bin; continuous: cells of 0.125 in the unit cube (dyadic: every sum is exact)

Everything stays inside NB_MAX boxes, KSUP_MAX supports per visit and STAB_SUP_POOL support slots along one DFS path; trajectory() checks this on the
oracle, so a capacity flag on the device is a bug.  Each env's trajectory is a pure function of (domain, setting, env, alias mode): the GPU test
replays the rows recorded here and compares what the device returns with what the oracle returned."""
import hashlib

import numpy as np

from pct_oracle import OracleContinuous, OracleDiscrete, policy_pick, rnd_u64

KSUP_SMALL, KSUP_MAX, STAB_SUP_POOL, STAB_DEPTH, NB_MAX = 8, 32, 48, 14, 80  # csrc/pct_kernels.h
NB, NL = 80, 50
PSEED = 5  # policy seed
STEPS = 75  # build-up (at most 51 placements) + policy steps
BUILD_MAX = 51
CHECKPOINTS = (BUILD_MAX - 1, STEPS - 1)  # support graphs compared after these steps: the end of every env's build-up, the end

# patch = (nx, ny, cx, cy, item on top): nx x ny columns from cell (cx, cy) of an 8 x 8 cell grid at the container's origin
PLANS = [
    [(4, 8, 0, 0, True), (4, 4, 4, 0, False)],                                             # 32 placed; 16 open
    [(5, 5, 0, 0, True), (3, 3, 5, 0, False), (4, 2, 0, 5, True)],                         # 25, 8 placed; 9 open
    [(4, 4, 0, 0, True), (3, 3, 4, 0, True), (2, 4, 0, 4, False), (3, 3, 4, 4, False)],    # 16, 9 placed; 8, 9 open
    [(4, 8, 0, 0, False), (3, 3, 4, 0, True), (2, 4, 4, 4, True)],                         # 9, 8 placed; 32 open
    [(5, 5, 0, 0, False), (3, 3, 5, 0, True), (2, 4, 5, 3, True)],                         # 9, 8 placed; 25 open
]
# the items of the policy phase, in cells: mostly large and flat, so that they land on the patches and on the items on top of them
POLICY_ITEMS = [(3, 3, 1), (4, 4, 1), (3, 4, 1), (4, 5, 1), (5, 5, 1), (3, 5, 1), (4, 8, 1), (4, 4, 2), (3, 3, 2), (2, 5, 1)]


def unit(cont):
    return 0.125 if cont else 1


def container(cont):
    return (1.0, 1.0, 1.0) if cont else (10, 10, 10)


def is_tall(env):
    return env % 4 == 3


def plan(cont, setting, env):
    """-> (stream (n, 4): x, y, z, density per draw, rows of the build-up placements (one per draw), the plan's patches)"""
    u = unit(cont)
    patches = PLANS[(env + env // len(PLANS)) % len(PLANS)]
    items, rows = [], []
    for i, (nx, ny, cx, cy, top) in sorted(enumerate(patches), key=lambda ip: not ip[1][4]):  # the patches that get an item first
        h = 6 if is_tall(env) else 1 + rnd_u64(71, env, i) % 2  # column height in cells (tall: 0.6 H of the discrete bin; 0.625 H of the unit cube)
        if is_tall(env) and cont:
            h = 5
        cells = [(cx + x, cy + y) for x in range(nx) for y in range(ny)]
        for j in sorted(range(len(cells)), key=lambda j: rnd_u64(72, env, 100 * i + j)):  # permuted floor order
            items.append((1, 1, h))
            rows.append((cells[j][0], cells[j][1], 1, 1))
        if top:  # right away: the columns laid after it are candidates on top of it, whose walks descend through its supports.  Two cells
            items.append((nx, ny, 2))  # high, so that its top is level with no column (a surface of 32 + 17 supports would exceed STAB_SUP_POOL)
            rows.append((cx, cy, nx, ny))
    n_build = len(items)
    for d in range(BUILD_MAX + 200 - n_build):  # streams of one length (a batch takes one array)
        items.append(POLICY_ITEMS[rnd_u64(73, env, d) % len(POLICY_ITEMS)])
    s = np.zeros((len(items), 4))
    for d, it in enumerate(items):
        s[d, :3] = [v * u for v in it]
        s[d, 3] = max((rnd_u64(74, env, d) >> 11), 1) / float(1 << 53) if setting == 3 else 1.0
    r = np.zeros((n_build, 9))
    for d, (x, y, dx, dy) in enumerate(rows):
        r[d, :6] = [x * u, y * u, 0, (x + dx) * u, (y + dy) * u, 0]
        r[d, 8] = 1
    return s, r, patches


def make_oracle(cont, setting, stream, alias=True):
    o = (OracleContinuous(setting, stream=stream, size_minimum=0.125) if cont
         else OracleDiscrete(setting, stream=stream, size_minimum=1))
    o.set_alias_mode(alias)
    return o


def streams(cont, setting, n):
    return np.stack([plan(cont, setting, e)[0] for e in range(n)])


# ---- what the walks of one state visit, from the oracle's box list ------------------------------------------------------------
def _boxes(orc):
    """placed boxes as (lx, ly, lz, hx, hy, hz) float64, placement order"""
    p = np.array(orc.packed, dtype=np.float64).reshape(-1, 7)
    return np.stack([p[:, 3], p[:, 4], p[:, 5], p[:, 3] + p[:, 0], p[:, 4] + p[:, 1], p[:, 5] + p[:, 2]], axis=1)


def _supports(b, fx1, fy1, fx2, fy2, z):
    """indices of the boxes a footprint resting at height z stands on (positive-area overlap, top at z), scan order"""
    if len(b) == 0 or z <= 0:
        return np.zeros(0, dtype=np.int64)
    ov = (np.minimum(b[:, 3], fx2) - np.maximum(b[:, 0], fx1) > 1e-9) & (np.minimum(b[:, 4], fy2) - np.maximum(b[:, 1], fy1) > 1e-9)
    return np.nonzero(ov & (np.abs(b[:, 5] - z) < 1e-6))[0]


def _slots(s, pool):
    """support slots the DFS of the stability routine holds at its deepest point below a node with supports s (scan order), given those of
    every support: the node's frame keeps its k slots while it descends into supports 0 .. k-2 and is gone when it descends into the last one"""
    k = len(s)
    return max(k + (pool[s[:-1]].max() if k > 1 else 0), k, pool[s[-1]])


def walk_census(orc, cont):
    """The stability walks of the current state (every candidate the reference evaluates that is in bounds, fits under the lid and rests on
    boxes) -> dict: k (supports of each walk's placement), direct (the footprint's centre lies strictly inside one contact rectangle: no
    least squares at the root), tall (it rests at >= 0.6 H), below_big (a box on > KSUP_SMALL supports lies below it: the walk descends to it
    unless it fails first), sup_pool (largest sum of support counts along one root-to-floor path), depth (longest such path), k_box
    (largest support count of a placed box)."""
    W, L, H = container(cont)
    b = _boxes(orc)
    n = len(b)
    # per placed box: the support slots of its deepest DFS descent, the depth below it, whether a box on > KSUP_SMALL supports is reachable
    pool, depth, big, k_box = np.zeros(n, dtype=int), np.zeros(n, dtype=int), np.zeros(n, dtype=bool), 0
    for i in range(n):
        s = _supports(b[:i], b[i, 0], b[i, 1], b[i, 3], b[i, 4], b[i, 2])
        k_box = max(k_box, len(s))
        big[i] = len(s) > KSUP_SMALL
        if len(s):
            pool[i] = _slots(s, pool)
            depth[i] = 1 + depth[s].max()
            big[i] |= big[s].any()
    cand, feas = orc.candidates()
    out = dict(k=[], direct=[], tall=[], below_big=[], sup_pool=0, depth=0, k_box=k_box)
    for p, f in zip(cand, feas):
        if f < 0:
            continue
        fx1, fy1, fx2, fy2, dz = p[0], p[1], p[3], p[4], p[5] - p[2]
        if fx2 - 1e-6 > W or fy2 - 1e-6 > L:
            continue
        ov = (np.minimum(b[:, 3], fx2) - np.maximum(b[:, 0], fx1) > 1e-9) & (np.minimum(b[:, 4], fy2) - np.maximum(b[:, 1], fy1) > 1e-9)
        z = b[ov, 5].max() if ov.any() else 0.0
        if z <= 1e-6 or z + dz - 1e-6 > H:
            continue
        s = _supports(b, fx1, fy1, fx2, fy2, z)
        cx, cy = (fx1 + fx2) * 0.5, (fy1 + fy2) * 0.5
        x1, y1 = np.maximum(b[s, 0], fx1), np.maximum(b[s, 1], fy1)
        x2, y2 = np.minimum(b[s, 3], fx2), np.minimum(b[s, 4], fy2)
        out["k"].append(len(s))
        out["direct"].append(bool(((cx - x1 > 1e-6) & (x2 - cx > 1e-6) & (cy - y1 > 1e-6) & (y2 - cy > 1e-6)).any()))
        out["tall"].append(bool(z * 5 >= 3 * H - 1e-9))
        out["below_big"].append(bool(big[s].any()))
        out["sup_pool"] = max(out["sup_pool"], _slots(s, pool))
        out["depth"] = max(out["depth"], 1 + depth[s].max())
    return out


def _digest(o):
    return hashlib.blake2b(np.ascontiguousarray(o, dtype=np.float64).tobytes(), digest_size=16).digest()


def trajectory(args):
    """One env's lock-step record on the oracle: build-up rows, then the shared policy, auto-reset on done (ShmemVecEnv semantics).
    args = (cont, setting, env, alias, census).  -> dict: rows (T, 9), reward, done, counter, obs digests (T + 1: after the reset and after
    every step, the next episode's first observation on a done step), graphs {step: oracle support graph after it}, and with census: per step the
    walk census of the state the step's candidates come from, lstsq (n_lstsq after the step).  Raises AssertionError if the trajectory leaves
    the capacities the device has (then it is no test of the many-support path) or a build-up placement ends the episode."""
    cont, setting, env, alias, census = args
    stream, brows, _ = plan(cont, setting, env)
    orc = make_oracle(cont, setting, stream, alias)
    o = orc.reset()
    rec = dict(rows=np.zeros((STEPS, 9)), reward=np.zeros(STEPS), done=np.zeros(STEPS, dtype=bool), counter=np.zeros(STEPS, dtype=np.int64),
               obs=[_digest(o)], graphs={}, census=[], lstsq=[], n_build=len(brows))
    for t in range(STEPS):
        if census:
            c = walk_census(orc, cont)
            where = "%s setting %d env %d step %d" % ("continuous" if cont else "discrete", setting, env, t)
            assert max(c["k"] + [0]) <= KSUP_MAX and c["k_box"] <= KSUP_MAX, where
            assert c["sup_pool"] <= STAB_SUP_POOL and c["depth"] <= STAB_DEPTH, where
            rec["census"].append(c)
        row = brows[t] if t < len(brows) else policy_pick(o, NB, NL, PSEED, env, t)[1]
        o, r, d, info = orc.step(row)
        assert "error" not in info, "env %d step %d: %s" % (env, t, info)
        assert not (d and t < len(brows)), "env %d: build-up placement %d ends the episode" % (env, t)
        if census:
            rec["lstsq"].append(orc.n_lstsq)
        rec["rows"][t], rec["reward"][t], rec["done"][t], rec["counter"][t] = row, r, d, info["counter"]
        if d:
            o = orc.reset()
        if t in CHECKPOINTS:
            rec["graphs"][t] = orc.support_graph()  # after the auto-reset, as the device holds it
        rec["obs"].append(_digest(o))
    return rec


def trajectories(cont, setting, n, alias=True, census=False, workers=None):
    """trajectory() of envs 0 .. n-1, on a process pool (spawned: the parent may hold a CUDA context)"""
    import multiprocessing as mp
    import os
    from concurrent.futures import ProcessPoolExecutor
    args = [(cont, setting, e, alias, census) for e in range(n)]
    if n <= 4:
        return [trajectory(a) for a in args]
    workers = workers or min(32, os.cpu_count() or 1)
    with ProcessPoolExecutor(workers, mp_context=mp.get_context("spawn")) as ex:
        return list(ex.map(trajectory, args, chunksize=max(1, n // (4 * workers))))


def digest_rows(obs):
    """per-env digests of a (n, obs_len) float64 array, as trajectory() records them"""
    return [_digest(o) for o in obs]
