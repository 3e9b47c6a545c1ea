"""The heuristic baselines of buffered envs (pct_buffer_heuristic_actions, pct_buffer_step_rows; DESIGN.md section 22) on the CPU oracle
(test infrastructure).

The buffered choice is composed from the plain oracle baseline (oracle/pct_oracle_heuristics.py `choose`) run for every slot's item on the
env's current state (Oracle*.set_next), by the rules of include/pct_b200.h: the best score in the baseline's direction (OnlineBPH: the lowest
EMS rank), ties to the lowest slot; RANDOM draws a slot among those with a placement under a key of its own.  Each slot's score and rank are
recomputed from the plain choice, so that a test can see why a slot was picked:
    LSAH / DBL / HM / MACS  the baseline's score of the chosen placement (it depends on the placement alone);
    BR                      the best EMS score among the EMSs at the chosen origin that hold the chosen orientation (they are all feasible
                            candidates of that placement, and the strict `>` keeps the first of the best);
    OnlineBPH               the rank, in the (z, y, x) order, of the first EMS at the chosen origin: an earlier EMS at the same origin would
                            have yielded the same first feasible rotation there (no fit test).
"""
import numpy as np

import pct_oracle_heuristics as H
from buffer_oracle import BufferedOracle, refill
from harness import expected_flags
from pct_oracle import rnd_u64

BUF_SLOT_SALT = 0xB0FF510F  # csrc/pct_kernels.h: RANDOM's slot draw rnd_u64(seed ^ BUF_SLOT_SALT, env id, t)
LOWER = ("LSAH", "DBL", "HM")  # the least score wins; BR and MACS: the greatest


def choice_score(name, view, state, item_set, choice):
    """-> (score, rank) of the plain choice `choice` ((dims, lx, ly)) for view's current item; (None, None) without one"""
    if choice is None:
        return None, None
    d, lx, ly = choice
    if name == "OnlineBPH":
        ems = sorted([list(e) for e in view.ems()], key=lambda e: (e[2], e[1], e[0]))
        return None, next(i for i, e in enumerate(ems) if e[0] == lx and e[1] == ly)
    if name == "BR":
        best = None
        for e in view.ems():
            ext = (e[3] - e[0], e[4] - e[1], e[5] - e[2])
            if e[0] == lx and e[1] == ly and ext[0] >= d[0] and ext[1] >= d[1] and ext[2] >= d[2]:
                fits = sum(1 for b in item_set if ext[0] >= b[0] and ext[1] >= b[1] and ext[2] >= b[2])
                s = ext[0] * ext[1] * ext[2] + fits + (10 if fits == len(item_set) else 0)
                best = s if best is None or s > best else best
        return best, None
    if name == "RANDOM":
        return None, None
    ok, h = view.drop_box_virtual(d, lx, ly)
    assert ok, "the plain choice is feasible"
    if name == "LSAH":
        ex = max(lx + d[0], state["max"][0]) - min(lx, state["min"][0])
        ey = max(ly + d[1], state["max"][1]) - min(ly, state["min"][1])
        return ex * ey + (h + d[2]) * ey + (h + d[2]) * ex, None
    if name == "DBL":
        return lx + ly + 100 * h, None
    plain = view.plain()
    if name == "MACS":
        return H.macs_score(plain, d, lx, ly, h), None
    foot = plain[lx:lx + d[0], ly:ly + d[1]]
    return lx + ly + 100 * (int(plain.sum()) - int(foot.sum()) + foot.size * (h + d[2])), None


def buffered_choose(name, view, buf, state, item_set=None, seed=0, gid=0, t=0):
    """The buffered baseline on `view` (an Oracle* env) holding items buf ((B, 4)) -> (slot, choice or None, per-slot plain choices,
    scores, ranks).  Leaves view holding the chosen slot's item."""
    choices, scores, ranks = [], [], []
    for j in range(len(buf)):
        view.set_next(buf[j])
        c = H.choose(name, view, state, item_set, seed, gid, t)
        s, r = choice_score(name, view, state, item_set, c)
        choices.append(c)
        scores.append(s)
        ranks.append(r)
    live = [j for j in range(len(buf)) if choices[j] is not None]
    if not live:
        slot = 0
    elif name == "RANDOM":
        slot = live[rnd_u64(seed ^ BUF_SLOT_SALT, gid, t) % len(live)]
    else:
        slot = live[0]
        for j in live[1:]:
            if name == "OnlineBPH":
                better = ranks[j] < ranks[slot]
            elif name in LOWER:
                better = scores[j] < scores[slot]
            else:
                better = scores[j] > scores[slot]
            if better:
                slot = j
    view.set_next(buf[slot])
    return slot, choices[slot], choices, scores, ranks


class RowBufferedOracle(BufferedOracle):
    """BufferedOracle with the row step of pct_buffer_step_rows and the LSAH footprint a buffered baseline keeps"""

    def reset(self, pos=None):
        self.hstate = H.fresh_state(self.c["container"])
        return BufferedOracle.reset(self, pos)

    def step_row(self, j, row):
        """pct_buffer_step_rows of slot j with action row `row` (slot outside [0, B): slot 0, the zero action): set_next(item j), the plain
        step with the row, then the refill of BufferedOracle.step -> (obs, reward, done, record)"""
        if not 0 <= j < self.B:
            j, row = 0, np.zeros(9)
        self.orc.set_next(self.buf[j])
        _, r, d, info = self.orc.step(np.asarray(row, dtype=np.float64))
        cnt = {"ems": len(self.orc.ems()), "ems_tmp": self.orc.n_ems_intermediate()}
        pf = expected_flags(self.c, cnt, info)
        rec = dict(counter=info["counter"], placement_flags=pf)
        if d:
            rec["ratio"] = info["ratio"]
            self.orc.reset()
            self.hstate = H.fresh_state(self.c["container"])
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

    def heuristic(self, name, item_set=None, seed=0, gid=0, t=0):
        """the buffered baseline's (slot, row, choice, scores, ranks) on the current state; LSAH's footprint takes the choice"""
        slot, c, _, scores, ranks = buffered_choose(name, self.orc, self.buf, self.hstate, item_set, seed, gid, t)
        cont = self.c["domain"] == "continuous"
        if c is not None and name == "LSAH":
            H.note_placement(self.hstate, c)
        return slot, H.action_row(c, self.c["container"], cont), c, scores, ranks
