"""CPU model of LNES='EVM' (include/pct_b200.h, PCT_LNES_EVM): the reference's EventPoint (D:space.py:613-693) over the EMS list and ZMAP
that GENEMS maintains, composed on the oracle (test infrastructure).

The env state is the oracle's under LNES='EMS', which runs GENEMS after every placement, exactly as the reference does when it is built with
LNES='EMS' and Space.EMSPoint is rebound to Space.EventPoint.  Only the observation's leaf rows differ: this model rebuilds them from the
placed boxes (the ZMAP), the EMS list, CPython's own set, the keyed shuffle and the oracle's placement test."""
import numpy as np

from pct_oracle import OracleDiscrete, rnd_u64

SET_MAX = 1228   # entries of one level's set the device's set emulation holds
LIST_MAX = 1228  # entries of the concatenated list
FLAG_CAND_OVERFLOW = 8


def zmap(boxes, W, L, H):
    """the ZMAP from the placed boxes (x1, y1, z1, x2, y2, z2) in placement order: {level: (x_up, y_left, x_bottom, y_right)}, levels in
    the reference's key order, lists sorted (maintainEventBottom / AddNewEMSZ, D:PctTools.py:41-80)"""
    Z = {0: (set([0]), set([0]), set([W]), set([L]))}
    for x1, y1, z1, x2, y2, z2 in boxes:
        xu, yl, xb, yr = Z[z1]
        if x2 < W:
            xu.add(x2)
        xb.add(x1)
        if y2 < L:
            yl.add(y2)
        yr.add(y1)
        if z2 < H:
            xu, yl, xb, yr = Z.setdefault(z2, (set(), set(), set(), set()))
            xu.add(x1); yl.add(y1); xb.add(x2); yr.add(y2)
    return {k: tuple(sorted(v) for v in r) for k, r in Z.items()}


def rotations(nb, setting):
    """the oriented sizes EventPoint visits (D:space.py:629-651)"""
    a, b, c = nb
    out = [(a, b, c)]
    if setting == 2:
        if b != a: out.append((b, a, c))
        if not (a == c == b): out.append((a, c, b))
        if not (b == c == a): out.append((b, c, a))
        if c != a: out.append((c, a, b))
        if c != b: out.append((c, b, a))
    elif b != a:
        out.append((b, a, c))
    return out


def event_points(Z, ems, nb, setting):
    """-> (list of (xs, ys, zs, xe, ye, ze), flags): EventPoint with the device's capacity rule"""
    out, flags = [], 0
    rots = rotations(nb, setting)
    for k, (xu, yl, xb, yr) in Z.items():
        lev = [e for e in ems if e[2] == k]
        if not lev:
            continue
        pos = set()
        for sx, sy, sz in rots:
            for xs in list(xu) + [xe - sx for xe in xb]:
                for ys in list(yl) + [ye - sy for ye in yr]:
                    pos.add((xs, ys, k, xs + sx, ys + sy, k + sz))
        if len(pos) > SET_MAX:
            return out, flags | FLAG_CAND_OVERFLOW
        out += [p for p in pos if any(e[0] <= p[0] and e[1] <= p[1] and p[3] <= e[3] and p[4] <= e[4] for e in lev)]
        if len(out) > LIST_MAX:
            return out[:LIST_MAX], flags | FLAG_CAND_OVERFLOW
    return out, flags


class EvmOracle(object):
    """OracleDiscrete's call surface under LNES='EVM'.  `flags` holds the candidate-overflow bit of the latest observation."""

    def __init__(self, setting, container_size=(10, 10, 10), internal_node_holder=80, leaf_node_holder=50, size_minimum=1, stream=None):
        self.o = OracleDiscrete(setting, container_size, internal_node_holder, leaf_node_holder, size_minimum, stream, lnes="EMS")
        self.o.set_alias_mode(True)
        self.setting, self.container = int(setting), tuple(int(c) for c in container_size)
        self.nb, self.nl = internal_node_holder, leaf_node_holder
        self.shuffle = None
        self.flags = 0
        self.last_cand = []

    def set_stream(self, stream):
        self.o.set_stream(stream)

    def set_random_items(self, item_set, seed, gid):
        self.o.set_random_items(item_set, seed, gid)

    def set_trajectory_length(self, n):
        self.o.set_trajectory_length(n)

    def set_shuffle(self, seed, gid, on=True):
        self.shuffle = (int(seed) & ((1 << 64) - 1), int(gid)) if on else None

    def boxes(self):
        return [(lx, ly, lz, lx + x, ly + y, lz + z) for x, y, z, lx, ly, lz, _ in self.o.packed]

    def zmap(self):
        return zmap(self.boxes(), *self.container)

    def _obs(self, ob):
        W, L, H = self.container
        cand, self.flags = event_points(self.zmap(), self.o.ems().tolist(), self.o.next_box, self.setting)
        if self.shuffle is not None and len(cand) > 1:
            seed, gid = self.shuffle
            pos = self.o.stream_pos
            keys = [rnd_u64(seed ^ 0x5AFE5EED, gid, (pos << 16) | i) for i in range(len(cand))]
            cand = [cand[i] for i in sorted(range(len(cand)), key=lambda i: keys[i])]
        self.last_cand = cand
        leaf = np.zeros((self.nl, 9))
        self.last_feas = np.full(len(cand), -1)
        n = 0
        for i, (xs, ys, zs, xe, ye, ze) in enumerate(cand):
            self.last_feas[i] = ok = int(self.o.drop_box_virtual((xe - xs, ye - ys, ze - zs), xs, ys)[0])
            if ok:
                leaf[n] = (xs, ys, zs, xe, ye, H, 0, 0, 1)
                n += 1
                if n >= self.nl:
                    break
        ob = ob.copy()
        ob[9 * self.nb:9 * (self.nb + self.nl)] = leaf.reshape(-1)
        return ob

    def reset(self):
        return self._obs(self.o.reset())

    def step(self, action):
        ob, r, d, info = self.o.step(action)
        return self._obs(ob), r, d, info

    def set_next(self, item):
        return self._obs(self.o.set_next(item))

    def ems(self):
        return self.o.ems()

    def candidates(self):
        """the latest list and its placement verdicts (-1: not tested, the leaf cap was reached before it), as OracleDiscrete.candidates"""
        return np.array(self.last_cand, dtype=np.int32).reshape(-1, 6), self.last_feas.copy()

    def n_ems_intermediate(self):
        return self.o.n_ems_intermediate()

    def support_graph(self):
        return self.o.support_graph()

    @property
    def packed(self):
        return self.o.packed

    @property
    def next_box(self):
        return self.o.next_box

    @property
    def stream_pos(self):
        return self.o.stream_pos
