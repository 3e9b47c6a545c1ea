"""A buffered env (PctBatch(..., buffer=B); DESIGN.md section 18) on the CPU oracle (test infrastructure).

One oracle per env, in alias mode, shuffle off.  The model keeps the env's B items itself by the refill rule; its observation is built
with Oracle*.set_next (`env.next_box = item`): the internal rows, then for every slot the first NL feasible candidates of the slot's item on
the current state (the oracle's leaf rows for it), then one item row per slot.  A step makes the chosen item current (set_next) and steps the
oracle with the chosen leaf row; on done the oracle resets and the buffer is refilled.  The record's flags follow the plain step's rule
(tests/test_gpu_capacities.py): the placement's come from the EMS counts after the step and the step's info, the candidate / raw-key ones
from every slot's counts; they are sticky until the env resets.  n_leaf / n_cand are the sums over the slots.  policy() restates
pct_buffer_policy_random, so that a whole buffered trajectory is predicted on the CPU.
"""
import numpy as np

from harness import CASES, CONT_BINS, ITEM_SET, case_stream, cont_case_stream, expected_flags, load_capacity_cases, make_stream
from pct_oracle import OracleContinuous, OracleDiscrete, make_continuous_stream, rnd_u64


def refill(buf, pos, stream, done, j, traj=0):
    """The buffer's refill rule (DESIGN.md section 18) on a host copy: a placed item's slot j takes the next draw; a finished episode (and
    the first reset, from pos 0) refills slots 0 .. B-1 with the next B draws, under a trajectory length from the next trajectory's start.
    buf: (B, 4) array, changed in place; pos: the env's next draw position.  -> the new position"""
    L = len(stream)
    if done:
        if traj and pos % traj:
            pos += traj - pos % traj
        buf[:] = stream[[(pos + k) % L for k in range(len(buf))]]
        return pos + len(buf)
    buf[j] = stream[pos % L]
    return pos + 1


def buffer_policy(n_leaf, nl, seed, env, t):
    """pct_buffer_policy_random: a uniform valid flat index j * NL + l over the leaf counts of the slots (0 when there is none)"""
    total = int(sum(n_leaf))
    if total == 0:
        return 0
    k, j = rnd_u64(seed, env, t) % total, 0
    while k >= n_leaf[j]:
        k -= n_leaf[j]
        j += 1
    return j * nl + int(k)


def config(name, nl=50):
    """-> (configuration (keys: domain, setting, container, nb, nl, size_minimum, lnes, items), stream maker (seed, env, n)) of a named
    configuration: d1-d3 / c1-c3 (the default bins), a case of harness.CASES / harness.CONT_BINS, or side255 (the 255-cell cube of the
    capacity cases)"""
    if name[0] in "dc" and name[1:] in ("1", "2", "3"):
        s = int(name[1])
        if name[0] == "d":
            return dict(domain="discrete", setting=s, container=(10, 10, 10), nb=80, nl=nl, size_minimum=1, items=ITEM_SET), \
                lambda seed, e, n: make_stream(seed, e, n, s)
        return dict(domain="continuous", setting=s, container=(1.0, 1.0, 1.0), nb=80, nl=nl, size_minimum=0.1), \
            lambda seed, e, n: make_continuous_stream(seed, e, n, s)
    if name == "side255":
        c = load_capacity_cases()["d_side255_s1"]
        c = dict(c, items=[tuple(i) for i in c["items"]])
    elif name in CASES:
        c = dict(CASES[name], size_minimum=1)
    else:
        c = CONT_BINS[name]
        return dict(domain="continuous", setting=c["setting"], container=c["container"], nb=c["nb"], nl=nl, size_minimum=c["low"]), \
            lambda seed, e, n: cont_case_stream(c, seed, e, n)
    cfg = dict(domain="discrete", setting=c["setting"], container=tuple(c["container"]), nb=c["nb"], nl=nl if nl != 50 else c["nl"],
               size_minimum=c["size_minimum"], lnes=c.get("lnes", "EMS"), items=c["items"])
    return cfg, lambda seed, e, n: case_stream(c, seed, e, n)


def capacity_steps(c):
    """buffered steps a capacity case of tests/golden/capacity_cases.npz runs (its first flag comes by then at B = 3 and B = 16)"""
    return min(int(c["steps"]) + 40, len(c["stream"]) - 40, 110)


def make_oracle(c, stream):
    """the oracle env of configuration c (keys: domain, setting, container, nb, nl, size_minimum, lnes) in alias mode"""
    if c["domain"] == "continuous":
        o = OracleContinuous(c["setting"], container_size=c["container"], internal_node_holder=c["nb"], leaf_node_holder=c["nl"],
                             size_minimum=c["size_minimum"], stream=stream)
    else:
        o = OracleDiscrete(c["setting"], container_size=c["container"], internal_node_holder=c["nb"], leaf_node_holder=c["nl"],
                           size_minimum=c["size_minimum"], stream=stream, lnes=c.get("lnes", "EMS"))
    o.set_alias_mode(True)
    return o


class BufferedOracle(object):
    """one buffered env of configuration c with B slots on item stream `stream` ((L, 4), read cyclically, as the device reads it)"""

    def __init__(self, c, stream, B, traj=0):
        self.c, self.B, self.nb, self.nl, self.traj = c, B, c["nb"], c["nl"], traj
        self.stream = np.ascontiguousarray(stream, dtype=np.float64)
        self.orc = make_oracle(c, self.stream)
        self.buf = np.zeros((B, 4))
        self.pos = 0
        self.sticky = 0

    def reset(self, pos=None):
        """env.reset() with the buffer refilled from draw position `pos` (default: the model's own) -> observation"""
        if pos is not None:
            self.pos = pos
        self.orc.reset()
        self.pos = refill(self.buf, self.pos, self.stream, True, 0, self.traj)
        self._observe()
        self.sticky = self.slot_flags
        return self.obs

    def _observe(self):
        """the buffered observation of the current state, and per slot: leaf count, candidate count, the candidates' capacity flags"""
        nb, nl, B = self.nb, self.nl, self.B
        rows = np.zeros((nb + B * nl + B, 9))
        self.n_leaf, self.n_cand, self.slot_fl = np.zeros(B, dtype=np.int64), np.zeros(B, dtype=np.int64), np.zeros(B, dtype=np.int64)
        self.stored = np.zeros((B, nl, 6))  # each slot's leaves as the placements they stand for (x1, y1, z1, x2, y2, z2): the stored blocks
        lnes = self.c.get("lnes", "EMS")
        for j in range(B):
            o = self.orc.set_next(self.buf[j]).reshape(-1, 9)
            if j == 0:
                rows[:nb] = o[:nb]
            rows[nb + j * nl:nb + (j + 1) * nl] = o[nb:nb + nl]
            rows[nb + B * nl + j] = o[nb + nl]
            cand, feas = self.orc.candidates()
            self.stored[j] = 0
            live = cand[feas == 1][:nl]
            self.stored[j, :len(live)] = live
            cnt = {"cand": len(cand)}
            if isinstance(self.orc, OracleDiscrete) and lnes in ("EP", "CP", "FC"):
                cnt["raw"] = self.orc.n_raw_candidates()
            self.n_leaf[j] = int((o[nb:nb + nl, 8] == 1).sum())
            self.n_cand[j] = cnt["cand"]
            self.slot_fl[j] = expected_flags(self.c, cnt, {})
        self.obs = rows.reshape(-1)
        self.slot_flags = int(np.bitwise_or.reduce(self.slot_fl))

    @property
    def blocks(self):
        nb, nl, B = self.nb, self.nl, self.B
        return self.obs.reshape(-1, 9)[nb:nb + B * nl].reshape(B, nl, 9)

    def policy(self, seed, env, t):
        return buffer_policy(self.n_leaf, self.nl, seed, env, t)

    def step(self, flat):
        """buffered step with flat index j * NL + l (outside [0, B * NL): slot 0, the zero action) -> (obs, reward, done, record) where
        record = dict(counter, flags, n_leaf, n_cand, n_ems, ratio (done only), placement_flags, slot_flags (per slot, of the new
        expansion))"""
        B, nl = self.B, self.nl
        if 0 <= flat < B * nl:
            j, l = flat // nl, flat % nl
            row = self.blocks[j, l].copy()
        else:
            j, row = 0, np.zeros(9)
        self.orc.set_next(self.buf[j])
        _, r, d, info = self.orc.step(row)
        cnt = {"ems": len(self.orc.ems()), "ems_tmp": self.orc.n_ems_intermediate()}
        pf = expected_flags(self.c, cnt, info)
        rec = dict(counter=info["counter"], placement_flags=pf)
        if d:
            rec["ratio"] = info["ratio"]
            self.orc.reset()
            before = self.sticky | pf
        self.pos = refill(self.buf, self.pos, self.stream, d, j, self.traj)
        self._observe()
        if d:
            rec["flags"] = before | self.slot_flags
            self.sticky = self.slot_flags
        else:
            self.sticky |= pf | self.slot_flags
            rec["flags"] = self.sticky
        rec.update(n_leaf=int(self.n_leaf.sum()), n_cand=int(self.n_cand.sum()), n_ems=len(self.orc.ems()), slot_flags=self.slot_fl.copy())
        return self.obs, r, d, rec


# ---- a buffered env on the many-support floors of tests/many_supports.py ----------------------------------------------------------------
MS_B, MS_NL, MS_STEPS = 16, 64, 26  # buffer, leaf holder, buffered steps after the floors
MS_N, MS_CHECK, MS_PSEED = 1024, tuple(range(0, 1024, 128)), 61  # envs of the batch, the envs held against the model, policy seed


def many_support_items(cont, setting, env, B=MS_B):
    """the B buffered items a floor env starts with: large flat items of many_supports.POLICY_ITEMS, which land on the patches"""
    import many_supports as M
    it = np.zeros((B, 4))
    for j in range(B):
        it[j, :3] = [v * M.unit(cont) for v in M.POLICY_ITEMS[rnd_u64(76, env, j) % len(M.POLICY_ITEMS)]]
        it[j, 3] = max((rnd_u64(77, env, j) >> 11), 1) / float(1 << 53) if setting == 3 else 1.0
    return it


def many_support_config(cont, setting, nl=MS_NL):
    import many_supports as M
    return dict(domain="continuous" if cont else "discrete", setting=setting, container=M.container(cont), nb=M.NB, nl=nl,
                size_minimum=M.unit(cont))


def many_support_model(cont, setting, env, B=MS_B, nl=MS_NL):
    """many_supports env `env` after its build-up placements (laid by rows), holding many_support_items: -> (model, build-up rows).  Its draw
    position is the plain env's after the build-up (the reset's draw and one per placement)."""
    import many_supports as M
    stream, brows, _ = M.plan(cont, setting, env)
    m = BufferedOracle(many_support_config(cont, setting, nl), stream, B)
    m.orc.reset()
    for r in brows:
        _, _, d, info = m.orc.step(r)
        assert not d and "error" not in info, "env %d: a build-up placement ends the episode" % env
    m.pos = len(brows) + 1
    m.buf[:] = many_support_items(cont, setting, env, B)
    m._observe()
    m.sticky = m.slot_flags
    return m, brows


def slot_census(m):
    """many_supports.walk_census of every slot's item on the model's current state (the walks of the slots' expansions)"""
    import many_supports as M
    out = []
    for j in range(m.B):
        m.orc.set_next(m.buf[j])
        out.append(M.walk_census(m.orc, m.c["domain"] == "continuous"))
    return out


def _start(args):
    cont, setting, env = args
    m, _ = many_support_model(cont, setting, env)
    return m.buf.copy(), m.n_leaf.copy(), m.stored.copy()


def many_support_starts(cont, setting, n, workers=None):
    """(items (B, 4), leaf counts (B,), stored blocks (B, NL, 6)) of many_support_model of envs 0 .. n-1, on a process pool (spawned: the
    parent may hold a CUDA context)"""
    import multiprocessing as mp
    import os
    from concurrent.futures import ProcessPoolExecutor
    args = [(cont, setting, e) for e in range(n)]
    if n <= 4:
        return [_start(a) for a in args]
    workers = workers or min(32, os.cpu_count() or 1)
    with ProcessPoolExecutor(workers, mp_context=mp.get_context("spawn")) as ex:
        return list(ex.map(_start, args, chunksize=max(1, n // (4 * workers))))
