"""Shared helpers for the parity tests (test infrastructure)."""
import numpy as np

from pct_oracle import OracleDiscrete, policy_pick, rnd_u64  # noqa: F401  (oracle/ is on sys.path via conftest)

ITEM_SET = [(i, j, k) for i in range(1, 6) for j in range(1, 6) for k in range(1, 6)]  # givenData.py:7-14
# the same 125 sizes scaled to the unit container of the continuous domain (givenData.py:4 `container_size = [1,1,1]`)
CONT_ITEM_SET = [(round(0.1 * i, 1), round(0.1 * j, 1), round(0.1 * k, 1)) for i in range(1, 6) for j in range(1, 6) for k in range(1, 6)]


def make_stream(seed, env, n, setting):
    """Deterministic per-env draw sequence (x,y,z,density) over the 125-item set."""
    s = np.zeros((n, 4))
    for d in range(n):
        s[d, :3] = ITEM_SET[rnd_u64(seed, env, d) % 125]
        s[d, 3] = max((rnd_u64(seed ^ 0xABCDEF, env, d) >> 11), 1) / float(1 << 53) if setting == 3 else 1.0
    return s


# ---- non-default configurations (tests/golden/make_golden_cases.py records them from the reference; the GPU cases of
# tests/test_gpu_discrete_cases.py use the same containers / item sets) ----------------------------------------------------
def _case(setting, container, items, nb=80, nl=50, steps=90, lnes="EMS"):
    return dict(setting=setting, container=tuple(container), items=[tuple(i) for i in items], nb=nb, nl=nl, steps=steps, lnes=lnes)


_BIG = [(i, j, k) for i in (4, 6, 9) for j in (5, 8) for k in (3, 7, 10)]
_SMALL = [(2, 2, 2), (3, 3, 2), (2, 3, 3), (4, 2, 2), (3, 4, 3)]
CASES = {
    "big_s1": _case(1, (20, 18, 24), _BIG), "big_s2": _case(2, (20, 18, 24), _BIG), "big_s3": _case(3, (20, 18, 24), _BIG),
    "holders_s1": _case(1, (10, 10, 10), ITEM_SET, nb=60, nl=30), "holders_s2": _case(2, (10, 10, 10), ITEM_SET, nb=80, nl=64),
    "dense16_s1": _case(1, (16, 16, 16), _SMALL, steps=70), "dense16_s2": _case(2, (16, 16, 16), _SMALL, steps=70),
    "flat_s1": _case(1, (12, 7, 9), [(i, j, k) for i in (1, 2, 4) for j in (1, 3) for k in (2, 3)], nb=70, nl=40),
    "cp_big_s1": _case(1, (14, 12, 10), ITEM_SET, steps=70, lnes="CP"), "ep_big_s2": _case(2, (14, 12, 10), ITEM_SET, steps=70, lnes="EP"),
    # found by scratch/soak_oracle_vs_reference.py: in extreme2D the dict newEps received key 2 before key 0 and the two points collide in
    # the 8-slot set table, so list(set(newEps.values())) lists them in the other order (D:PctTools.py:113-133)
    "ep_dictorder_s2": dict(_case(2, (14, 12, 10), ITEM_SET, steps=70, lnes="EP"), seed=134366, env=3),
    # the BASELINE-stream trajectories (items seed 1234, policy seed 4321) on which the object-alias semantics of the reference's real placement and
    # the snapshot semantics of round 1 part (scratch/alias_rate.py; DESIGN.md section 3 (b)) — recorded from the reference through and 30 steps past
    # the parting step; only the alias semantics (default since round 2) replays them
    "alias_d1_e126": dict(_case(1, (10, 10, 10), ITEM_SET, steps=69), seed=1234, pseed=4321, env=126),
    "alias_d1_e835": dict(_case(1, (10, 10, 10), ITEM_SET, steps=197), seed=1234, pseed=4321, env=835),
    "alias_d3_e92": dict(_case(3, (10, 10, 10), ITEM_SET, steps=133), seed=1234, pseed=4321, env=92),
}
NEEDS_ALIAS_D = ("alias_d1_e126", "alias_d1_e835", "alias_d3_e92")


def case_stream(c, seed, env, n):
    """draw sequence (x, y, z, density) over the case's item set"""
    s = np.zeros((n, 4))
    for d in range(n):
        s[d, :3] = c["items"][rnd_u64(seed, env, d) % len(c["items"])]
        s[d, 3] = max((rnd_u64(seed ^ 0xABCDEF, env, d) >> 11), 1) / float(1 << 53) if c["setting"] == 3 else 1.0
    return s


def _ccase(setting, container, lo, hi, nb=80, nl=50, steps=110):
    return dict(setting=setting, container=tuple(container), lo=lo, hi=hi, low=lo, nb=nb, nl=nl, steps=steps)


# continuous: a non-unit container (bounds scale like tools.py:178-181: U(0.1, 0.5) x min side) and other holder sizes
CONT_CASES = {"box2_s1": _ccase(1, (2.0, 1.5, 2.5), 0.15, 0.75), "box2_s2": _ccase(2, (2.0, 1.5, 2.5), 0.15, 0.75),
              "box2_s3": _ccase(3, (2.0, 1.5, 2.5), 0.15, 0.75), "holders_s1": _ccase(1, (1.0, 1.0, 1.0), 0.1, 0.5, nb=60, nl=25),
              # found by scratch/soak_oracle_vs_reference.py: a real placement whose verdict depends on Python object aliasing in the reference
              # (`up_edges[self] = self.thisStack` stores the live Stack object; DESIGN.md section 3).  Replayed exactly only under the object-alias semantics (default since round 2).
              "alias_s1": dict(_ccase(1, (2.0, 1.5, 2.5), 0.15, 0.75, steps=95), seed=136818, env=2)}
NEEDS_ALIAS = ("alias_s1",)  # records only the object-alias semantics (the default of the oracle AND of the kernels since round 2) reproduces; the
#                              snapshot mode (PCT_ORACLE_ALIAS=0 / PCT_B200_ALIAS=0) must NOT: tests/test_oracle_golden.py


def cont_case_stream(c, seed, env, n):
    """x, y = round(U(lo, hi), 3); z likewise (setting 2) or one of five levels (C:bin3D.py:103-115 scaled to the container)"""
    s = np.zeros((n, 4))
    lo, hi = c["lo"], c["hi"]
    u = lambda salt, d: ((rnd_u64(seed ^ salt, env, d) >> 11) / float(1 << 53))
    levels = [round(lo * k, 3) for k in (1, 2, 3, 4, 5)]
    for d in range(n):
        s[d, 0] = round(lo + (hi - lo) * u(0x11, d), 3)
        s[d, 1] = round(lo + (hi - lo) * u(0x22, d), 3)
        s[d, 2] = round(lo + (hi - lo) * u(0x33, d), 3) if c["setting"] == 2 else levels[rnd_u64(seed ^ 0x44, env, d) % 5]
        s[d, 3] = max((rnd_u64(seed ^ 0xABCDEF, env, d) >> 11), 1) / float(1 << 53) if c["setting"] == 3 else 1.0
    return s


# ---- fixed capacities of the step kernels (include/pct_b200.h flags; DESIGN.md section 7) ----------------------------------
# name -> (flag bit, capacity).  Every count the oracle reports is compared with its capacity: a count above it must flag.
FLAG_BOX, FLAG_EMS, FLAG_CAND = 1, 4, 8
CAPS = {
    "discrete": {"ems": (FLAG_EMS, 128), "ems_tmp": (FLAG_EMS, 256), "cand": (FLAG_CAND, 1228), "raw": (FLAG_CAND, 2048)},
    "continuous": {"ems": (FLAG_EMS, 256), "ems_tmp": (FLAG_EMS, 512), "cand": (FLAG_CAND, 1228)},
}


def load_capacity_cases():
    """name -> case dict of tests/golden/capacity_cases.npz (tests/golden/make_capacity_cases.py), its item stream under 'stream'"""
    import json
    import os
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "capacity_cases.npz"))
    out = {}
    for c in json.loads(str(z["meta"])):
        c.update(stream=z[c["name"]], container=tuple(c["container"]))
        out[c["name"]] = c
    return out


def capacity_oracle(c):
    """oracle env of a capacity case (tests/golden/capacity_cases.npz)"""
    from pct_oracle import OracleContinuous
    if c["domain"] == "continuous":
        return OracleContinuous(c["setting"], container_size=c["container"], internal_node_holder=c["nb"], leaf_node_holder=c["nl"],
                                size_minimum=c["size_minimum"], stream=c["stream"])
    return OracleDiscrete(c["setting"], container_size=c["container"], internal_node_holder=c["nb"], leaf_node_holder=c["nl"],
                          size_minimum=c["size_minimum"], stream=c["stream"], lnes=c.get("lnes", "EMS"))


def oracle_counts(orc, lnes="EMS"):
    """the oracle's list lengths after its last reset / step, by capacity name"""
    d = {"ems": len(orc.ems()), "ems_tmp": orc.n_ems_intermediate(), "cand": len(orc.candidates()[0])}
    if isinstance(orc, OracleDiscrete) and lnes in ("EP", "CP", "FC"):
        d["raw"] = orc.n_raw_candidates()
    return d


def expected_flags(c, counts, step_info):
    """flag bits the kernels must raise on a step whose oracle counts / info are these"""
    f = 0
    for name, (bit, cap) in CAPS[c["domain"]].items():
        if counts.get(name, 0) > cap:
            f |= bit
    if step_info.get("error") == 1:  # more boxes than internal_node_holder: IndexError in the reference
        f |= FLAG_BOX
    return f


def capacity_trace(c):
    """Replay a capacity case on the oracle with the shared policy (env 0 of seed c['pseed']), for at most c['steps'] steps, up to the
    first step that ends the episode or must flag.  -> dict: reset_flags (flags the reset's counts call for), n_steps (steps run),
    t_star (index of the first step that must flag, -1: none), flag (its bits), done (the last step ended the episode),
    peak (largest count per name and box count over the reset and every step before t_star)."""
    orc = capacity_oracle(c)
    lnes = c.get("lnes", "EMS")
    obs = orc.reset()
    cnt = oracle_counts(orc, lnes)
    peak = dict(cnt, boxes=0)
    out = dict(reset_flags=expected_flags(c, cnt, {}), n_steps=0, t_star=-1, flag=0, done=False)
    for t in range(c["steps"]):
        _, row = policy_pick(obs, c["nb"], c["nl"], c["pseed"], 0, t)
        obs, _, done, info = orc.step(row)
        cnt = oracle_counts(orc, lnes)
        f = expected_flags(c, cnt, info)
        out.update(n_steps=t + 1, done=bool(done))
        if f:
            out.update(t_star=t, flag=f, star=cnt)
            break
        for k, v in cnt.items():
            peak[k] = max(peak[k], v)
        peak["boxes"] = max(peak["boxes"], len(orc.packed))
        if done:
            break
    out["peak"] = peak
    return out


class OracleVec(object):
    """N independent oracle envs with the ShmemVecEnv worker semantics (auto-reset on done,
    wrapper/shmem_vec_env.py:139-143) and the shared deterministic policy."""

    def __init__(self, n, setting, streams, nb=80, nl=50, container=(10, 10, 10)):
        self.envs = [OracleDiscrete(setting, container_size=container, internal_node_holder=nb, leaf_node_holder=nl, stream=streams[i])
                     for i in range(n)]
        self.n, self.nb, self.nl = n, nb, nl

    def reset(self):
        return np.stack([e.reset() for e in self.envs])

    def step(self, actions):
        obs, rew, done, infos = [], [], [], []
        for e, a in zip(self.envs, actions):
            o, r, d, i = e.step(a)
            if d:
                o = e.reset()
            obs.append(o); rew.append(r); done.append(d); infos.append(i)
        return np.stack(obs), np.array(rew), np.array(done), infos

    def pick(self, obs, seed, t, env_id_base=0):
        idx, rows = [], []
        for e in range(self.n):
            k, row = policy_pick(obs[e], self.nb, self.nl, seed, env_id_base + e, t)
            idx.append(k); rows.append(row)
        return np.array(idx, dtype=np.int32), np.stack(rows)


# ---- batched-evaluation parity helpers (evaluation_tools.py:7-52 restated as a plain loop) -------------------------------
def eval_policy_np(obs, nb=80, nl=50):
    """deterministic test policy: a fixed function of (#valid leaves, #valid internal rows)"""
    o = obs.reshape(nb + nl + 1, 9)
    nv, nbx = int((o[nb:nb + nl, 8] == 1).sum()), int((o[:nb, 8] == 1).sum())
    return (7 * nv + 3 * nbx) % max(nv, 1)


def eval_policy_torch(obs, batch):
    import torch
    o = obs.reshape(obs.shape[0], batch.nb + batch.nl + 1, 9)
    nv, nbx = (o[:, batch.nb:batch.nb + batch.nl, 8] == 1).sum(1), (o[:, :batch.nb, 8] == 1).sum(1)
    return ((7 * nv + 3 * nbx) % torch.clamp(nv, min=1)).to(torch.int32)


def sequential_eval(make_env, episodes, nb=80, nl=50):
    """the reference's evaluation loop on any single env with its call surface (reference env or oracle):
    per episode -> (ratio, counter, packed)"""
    out = []
    for ep in range(episodes):
        env, obs = make_env(ep)
        while True:
            k = eval_policy_np(obs, nb, nl)
            row = obs.reshape(nb + nl + 1, 9)[nb + k].copy()
            items = env.packed
            obs, _, done, info = env.step(row)
            if done:
                out.append((float(info["ratio"]), int(info["counter"]), [list(p) for p in items]))
                break
    return out


# ---- the support graph an env keeps between steps (stability settings) -----------------------------------------------------
POLY_MAX = 256  # csrc/pct_kernels.h: entries of an env's polygon pool


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _fma(a, b, c):
    """a * b + c rounded once (math.fma arrives with Python 3.13)"""
    from fractions import Fraction
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def split_direction(c2d):
    """the two-support split direction from the two contact centres (D:space.py:107-112: the line through them over its squared length;
    np.linalg.norm of a 2-vector = sqrt of the ddot, whose second product is fused)"""
    import math
    lx, ly = float(c2d[0][0] - c2d[1][0]), float(c2d[0][1] - c2d[1][1])
    ln = math.sqrt(_fma(ly, ly, lx * lx))
    return np.array([lx / (ln * ln), ly / (ln * ln)])


def compare_graphs(dev, orc, where=""):
    """Compare two support graphs in the CANONICAL FORM: per env, slot-independent,

        per placed box u, in placement order:
          supports[u]   indices of the boxes u rests on, in stored order (= scan order at its placement, the reference's bottom_edges)
          loads[u]      rows (cx, cy, cz, mass) resting on u in insertion order (the reference's up_edges dict), with load_upper[u] = the box each
                        comes from and load_alias[u] = the entry is that box's own stack object
          polygon[u]    stored shrunk support polygon, vertices in stored order (empty if none is stored)
          own_stack[u]  (cx, cy, cz, mass) of the box's own stack (alias mode only)
        counts n_box, n_edge, n_poly

    `dev` is the product's side (PctBatch.support_graph / the host build's decoder), `orc` the oracle's (Oracle*.support_graph).  Floats are
    compared as bit patterns, never with a tolerance.  What each side holds, and what is therefore compared how:
      * cz of a load: virtual walks do not carry it, real placements store it on both sides -> compared like the other columns.
      * a load's value is the one the next walk reads: in alias mode the oracle reads an object entry through the upper box's live stack;
        the device keeps that value in the stored load too (after a completed descent they are equal, after a failed one alias_sync_loads
        copies them) -> compared, and the device's object entries must equal the upper box's own_stack.
      * box index n_box = the box of a FAILED real placement.  Both sides keep the entries its descent wrote until the env resets (the
        reference's up_edges keep them under a key no live box has, so they keep their last value; the device keeps the pool's tail).
      * polygons: the device stores one only for boxes with >= 2 supports (a single support is a rectangle test in registers, pinned by
        tests/test_gpu_geometry_units.py) and only while the pool has room (else the walk recomputes it) -> single-support polygons of the
        oracle are not compared; with >= 2 supports the device's is the oracle's, or empty exactly when it did not fit.
      * n_poly counts pool entries: vertices of the stored polygons plus one split direction per stored two-support box, the failed box's included.
      * the split direction has no oracle field -> compared with split_direction() of the oracle's two contact centres.
      * own_stack of a box that rests on the floor and carries nothing is never written by the device and never read -> not compared.
      * alias bits at or beyond n_edge are leftovers of earlier episodes (every appended edge rewrites its bit) -> reported, not compared.
    Raises AssertionError naming box and field; returns the numbers of compared loads / vertices / splits / own stacks."""
    n = dict(loads=0, vertices=0, splits=0, own=0)
    assert dev["n_box"] == orc["n_box"], "%s n_box: %d, oracle %d" % (where, dev["n_box"], orc["n_box"])
    assert dev["n_edge"] == orc["n_edge"], "%s n_edge: %d, oracle %d" % (where, dev["n_edge"], orc["n_edge"])
    both_alias = dev["alias"] and orc["alias"]
    acc = 0
    for u in range(dev["n_box"]):
        w = "%s box %d" % (where, u)
        assert dev["supports"][u] == orc["supports"][u], "%s supports: %s, oracle %s" % (w, dev["supports"][u], orc["supports"][u])
        assert dev["load_upper"][u] == orc["load_upper"][u], "%s loads come from boxes %s, oracle %s" % (w, dev["load_upper"][u], orc["load_upper"][u])
        for i, name in enumerate(("cx", "cy", "cz", "mass")):
            a, b = _bits(dev["loads"][u][:, i]), _bits(orc["loads"][u][:, i])
            assert np.array_equal(a, b), "%s load %s: row %d (from box %d) %r, oracle %r" % (
                w, name, int(np.nonzero(a != b)[0][0]), dev["load_upper"][u][int(np.nonzero(a != b)[0][0])],
                dev["loads"][u][int(np.nonzero(a != b)[0][0]), i], orc["loads"][u][int(np.nonzero(a != b)[0][0]), i])
        n["loads"] += len(dev["load_upper"][u])
        if both_alias:
            assert dev["load_alias"][u] == orc["load_alias"][u], "%s load is_alias: %s, oracle %s" % (w, dev["load_alias"][u], orc["load_alias"][u])
        if dev["alias"]:
            for i, (up, al) in enumerate(zip(dev["load_upper"][u], dev["load_alias"][u])):
                if al and up < dev["n_box"]:
                    assert np.array_equal(_bits(dev["loads"][u][i]), _bits(dev["own_stack"][up])), \
                        "%s load row %d is box %d's own stack object but holds %s, own_stack %s" % (w, i, up, dev["loads"][u][i], dev["own_stack"][up])
        k, m = len(orc["supports"][u]), len(orc["polygon"][u])
        stored = k >= 2 and acc + m + (k == 2) <= POLY_MAX
        if stored:
            assert dev["poly_pos"][u] == acc, "%s polygon pool position %d, expected %d" % (w, dev["poly_pos"][u], acc)
            assert dev["polygon"][u].shape == orc["polygon"][u].shape and np.array_equal(_bits(dev["polygon"][u]), _bits(orc["polygon"][u])), \
                "%s polygon: %s, oracle %s" % (w, dev["polygon"][u].tolist(), orc["polygon"][u].tolist())
            n["vertices"] += m
            acc += m + (k == 2)
            if k == 2:
                want = split_direction(orc["c2d"][u])
                assert dev["split"][u] is not None and np.array_equal(_bits(dev["split"][u]), _bits(want)), \
                    "%s split direction: %s, from the contact centres %s" % (w, dev["split"][u], want)
                n["splits"] += 1
        else:
            assert len(dev["polygon"][u]) == 0, "%s polygon: %d vertices stored where none is expected (%d supports)" % (w, len(dev["polygon"][u]), k)
        if both_alias and (k >= 1 or len(orc["load_upper"][u])):
            assert np.array_equal(_bits(dev["own_stack"][u]), _bits(orc["own_stack"][u])), \
                "%s own_stack: %s, oracle %s" % (w, dev["own_stack"][u], orc["own_stack"][u])
            n["own"] += 1
    has, k, m = orc["failed_box"]
    if has and k >= 2 and acc + m + (k == 2) <= POLY_MAX:
        acc += m + (k == 2)
    assert dev["n_poly"] == acc, "%s n_poly: %d, expected %d" % (where, dev["n_poly"], acc)
    return n
