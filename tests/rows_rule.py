"""A seeded "placement rule of one's own": the action rows a caller builds itself (README: query_placements is the primitive for such rules,
and the baselines hand pct_step rows of their own), as opposed to rows copied from the leaf list.  It reads nothing but the observation, so
the reference, the oracle and the kernels are driven by the same rows.  Used by tests/golden/make_golden_rows.py (records from the
reference), tests/test_rows_cpu.py (oracle) and tests/test_gpu_rows.py (kernels).

Each step picks one KIND:
  leaf      a valid leaf row
  corner    an orientation (any pair of the item's sides: LeafNode2Action accepts every one in every setting) at a corner of a placed box or
            flush with one of its far sides, preferring positions that rest on boxes, so that the real stability descent runs
  stack     an orientation on top of a box that itself rests on boxes, flush with one of its corners and on it alone, preferring an item
            centre outside what that box rests on: the load travels down the stack, so the real descent writes loads before a lower box fails
  grid      the same at an arbitrary point (integer cell / 3-decimal coordinate), preferring positions over boxes
  zero      the all-zero row (the item unrotated at the origin)
discrete only, each on its own step:
  frac      fractional coordinates, which int() truncates towards zero
  zerosum   a row whose first six entries sum to zero without being zero ([a, 0, 0, -a, 0, 0]): taken as the zero row
  twoequal  x == y on an item that has that side twice
  single    x == y on an item that has that side once: list.remove raises ValueError
  edge      a footprint that starts at W / L, at max(W, L), past them, or at a small negative value: np.max of an empty slice raises where
            Python's slice of plain is empty, a non-empty slice fails the bounds test
continuous only:
  nomatch   extents that match no side: the box keeps the row's extents, z is what is left of the item
  tol       an extent within (4e-7, 1e-6) or just outside (2e-6) the 1e-6 match tolerance of a side
  cedge     positions at 0 and at W - x / L - y, and 5e-7 and 2e-6 either side of them
"""
import itertools

import numpy as np

from pct_oracle import rnd_u64

D_KINDS = ["leaf"] * 24 + ["corner"] * 8 + ["stack"] * 16 + ["grid"] * 3 + ["zero", "frac", "zerosum", "twoequal", "single", "edge"]
C_KINDS = ["leaf"] * 24 + ["corner"] * 8 + ["stack"] * 16 + ["grid"] * 3 + ["zero", "nomatch", "tol", "cedge"]
RAISING = ("frac", "single", "edge")  # discrete kinds that make the reference raise in these records (frac: a truncated extent no side matches)


def _boxes(o, nb):
    b = o[:nb]
    return b[b[:, 5] > 0]


def rest_height(boxes, lx, ly, x, y, eps=0.0):
    """max top of the placed boxes whose footprint overlaps [lx, lx + x) x [ly, ly + y) (0 on the floor)"""
    m = 0.0
    for r in boxes:
        if r[0] < lx + x - eps and lx < r[3] - eps and r[1] < ly + y - eps and ly < r[4] - eps:
            m = max(m, float(r[5]))
    return m


class Rng(object):
    def __init__(self, seed, env, t):
        self.seed, self.env, self.t, self.k = seed, env, t, 0

    def int(self, n):
        self.k += 1
        return int(rnd_u64(self.seed, self.env, (self.t << 8) + self.k) % max(int(n), 1))

    def unit(self):
        self.k += 1
        return (rnd_u64(self.seed, self.env, (self.t << 8) + self.k) >> 11) / float(1 << 53)

    def choice(self, seq):
        return seq[self.int(len(seq))]


def _row(lx, ly, x, y, H):
    return np.array([lx, ly, 0, lx + x, ly + y, H, 0, 0, 1], dtype=np.float64)


def _positions(rng, boxes, x, y, W, L, cont):
    """corner / flush positions of the placed boxes that keep the footprint inside the container"""
    out = []
    for r in boxes:
        lx0, ly0, hx, hy = (float(v) for v in (r[0], r[1], r[3], r[4]))
        for px, py in ((hx, ly0), (lx0, hy), (lx0, ly0), (hx - x, ly0), (lx0, hy - y), (hx - x, hy - y), (hx, hy), (lx0 + (hx - lx0) / 2, ly0),
                       (hx - x / 2, ly0), (lx0, hy - y / 2), (hx - x / 2, hy - y / 2)):  # the last three straddle the box's far edges
            if cont:
                px, py = round(px, 6), round(py, 6)
            else:
                px, py = int(px), int(py)
            if 0 <= px <= W - x + 1e-9 and 0 <= py <= L - y + 1e-9:
                out.append((px, py))
    return out


def _pick_on_boxes(rng, cands, boxes, x, y, eps):
    """prefer (4 in 5) a candidate that rests on a box"""
    if not cands:
        return None
    high = [c for c in cands if rest_height(boxes, c[0], c[1], x, y, eps) > eps]
    if high and rng.int(5):
        return rng.choice(high)
    return rng.choice(cands)


def pick(obs, nb, nl, container, cont, seed, env, t, f32=False, warm=8):
    """-> (row float64 (9,), kind).  f32: the rows go out as float32, whose contract is 1e-6 on coordinates (tests/test_f32_rows.py), so
    the kinds that sit within float32 noise of a 1e-6 tolerance (tol, cedge) are not drawn"""
    rng = Rng(seed, env, t)
    o = np.asarray(obs, dtype=np.float64).reshape(-1, 9)
    W, L, H = container
    sides = [float(v) for v in o[nb + nl, 3:6]] if cont else [int(v) for v in o[nb + nl, 3:6]]
    leaf = o[nb:nb + nl]
    nvalid = int((leaf[:, 8] == 1).sum())
    boxes = _boxes(o, nb)
    kinds = [k for k in C_KINDS if not (f32 and k in ("tol", "cedge"))] if cont else D_KINDS
    kind = rng.choice(kinds) if len(boxes) >= warm or rng.int(4 * warm) == 0 else "leaf"  # build `warm` boxes first
    if kind == "leaf":
        if nvalid == 0:
            return np.zeros(9), "zero"
        return leaf[rng.int(nvalid)].copy(), kind
    if kind == "zero":
        return np.zeros(9), kind
    perm = rng.choice(list(itertools.permutations(range(3))))
    x, y = sides[perm[0]], sides[perm[1]]
    eps = 1e-6 if cont else 0.0
    if kind in ("corner", "grid", "nomatch", "tol"):
        if kind == "nomatch":
            x = round(0.1 * min(W, L) + 0.4 * min(W, L) * rng.unit(), 3)
            if any(abs(x - s) < 2e-6 for s in sides):
                x = round(x + 0.001, 3)
        elif kind == "tol":
            x = x + rng.choice([4e-7, -4e-7, 1e-6, -1e-6, 2e-6, -2e-6])
        if kind == "corner" or (kind != "grid" and rng.int(2)):
            p = _pick_on_boxes(rng, _positions(rng, boxes, x, y, W, L, cont), boxes, x, y, eps)
        else:
            p = None
        if p is None:
            cands = []
            for _ in range(8):
                if cont:
                    cands.append((round(rng.unit() * max(W - x, 0.0), 3), round(rng.unit() * max(L - y, 0.0), 3)))
                else:
                    cands.append((rng.int(W - x + 1), rng.int(L - y + 1)))
            p = _pick_on_boxes(rng, cands, boxes, x, y, eps)
        return _row(p[0], p[1], x, y, H), kind
    if kind == "stack":
        up = [r for r in boxes if r[2] > eps]
        cands = []
        outside = []
        for r in up:
            lx0, ly0, hx, hy, top = (float(v) for v in (r[0], r[1], r[3], r[4], r[5]))
            # the bounding box of what r rests on: an item whose centre lands outside it pulls r's load off its supports
            sup = [b for b in boxes if abs(b[5] - r[2]) <= eps and b[0] < hx - eps and lx0 < b[3] - eps and b[1] < hy - eps and ly0 < b[4] - eps]
            sx0, sy0 = max(min(b[0] for b in sup), lx0), max(min(b[1] for b in sup), ly0)
            sx1, sy1 = min(max(b[3] for b in sup), hx), min(max(b[4] for b in sup), hy)
            for px, py in ((lx0, ly0), (hx - x, ly0), (lx0, hy - y), (hx - x, hy - y)):
                px, py = (round(px, 6), round(py, 6)) if cont else (int(px), int(py))
                on_r = lx0 - eps <= px and px + x <= hx + eps and ly0 - eps <= py and py + y <= hy + eps
                if on_r and 0 <= px <= W - x + 1e-9 and 0 <= py <= L - y + 1e-9 and abs(rest_height(boxes, px, py, x, y, eps) - top) <= eps:
                    cands.append((px, py))
                    cx, cy = px + x / 2, py + y / 2
                    if not (sx0 <= cx <= sx1 and sy0 <= cy <= sy1):
                        outside.append((px, py))
        if outside and rng.int(4):
            cands = outside
        if not cands:
            return (leaf[rng.int(nvalid)].copy(), "leaf") if nvalid else (np.zeros(9), "zero")
        p = rng.choice(cands)
        return _row(p[0], p[1], x, y, H), kind
    if kind == "cedge":
        dl = rng.choice([0.0, 5e-7, -5e-7, 2e-6, -2e-6])
        px, py = rng.choice([0.0, W - x]), rng.choice([0.0, L - y])
        if rng.int(2):
            px += dl
        else:
            py += dl
        return _row(px, py, x, y, H), kind
    # ---- discrete odd encodings ----
    if kind == "frac":
        lx, ly = rng.int(W - x + 1), rng.int(L - y + 1)
        f = rng.choice([(0.3, 0.7, 0.5, 0.2), (0.9, 0.1, 0.95, 0.15), (-0.5, 0.0, -0.25, 0.4)])
        r = _row(lx, ly, x, y, H)
        r[0] += f[0]; r[1] += f[1]; r[3] += f[2]; r[4] += f[3]
        return r, kind
    if kind == "zerosum":
        a = float(rng.choice([1, 2, 3]))
        r = np.zeros(9)
        r[rng.choice([0, 1, 2])] = a
        r[rng.choice([3, 4, 5])] = -a
        r[8] = 1
        return r, kind
    if kind in ("twoequal", "single"):
        twice = [s for s in set(sides) if sides.count(s) >= 2]
        once = [s for s in set(sides) if sides.count(s) == 1]
        pool = twice if kind == "twoequal" else once
        if not pool:
            return np.zeros(9), "zero"
        s = sorted(pool)[rng.int(len(pool))]
        return _row(rng.int(max(W - s, 0) + 1), rng.int(max(L - s, 0) + 1), s, s, H), kind
    # edge: one axis starts at W / L, max(W, L), past them, or just below 0; the other in range
    n = max(W, L)
    starts_x = [W, n, n + 1, W - 1, -1, -2, -3, -x, -x - 1, -n, -n - 2]
    starts_y = [L, n, n + 1, L - 1, -1, -2, -3, -y, -y - 1, -n, -n - 2]
    if rng.int(2):
        lx, ly = rng.choice(starts_x), rng.int(max(L - y, 0) + 1)
    else:
        lx, ly = rng.int(max(W - x, 0) + 1), rng.choice(starts_y)
    return _row(lx, ly, x, y, H), kind


def is_leaf(row, obs, nb, nl):
    """the row equals one of the observation's valid leaf rows in its first six entries"""
    o = np.asarray(obs, dtype=np.float64).reshape(-1, 9)
    leaf = o[nb:nb + nl]
    leaf = leaf[leaf[:, 8] == 1]
    return bool(len(leaf)) and bool((np.abs(leaf[:, :6] - np.asarray(row, dtype=np.float64)[:6]).max(axis=1) == 0).any())


# ---- the configurations tests/golden/make_golden_rows.py records, and their oracles ----------------------------------------------------
FLAT_ITEMS = [(i, j, k) for i in (1, 2, 4) for j in (1, 3) for k in (2, 3)]  # harness.CASES["flat_s1"]
MIN_COUNTS = dict(failed_with_loads=20, offleaf_multi=50, lstsq=3, raised=10)  # totals over the records of make_golden_rows.py


def make_oracle(g, alias=True):
    """the oracle of a record's configuration, on the record's stream"""
    from pct_oracle import OracleContinuous, OracleDiscrete
    cls = OracleContinuous if str(g["domain"]) == "c" else OracleDiscrete
    o = cls(int(g["setting"]), container_size=tuple(g["container"].tolist()), internal_node_holder=int(g["nb"]), leaf_node_holder=int(g["nl"]),
            size_minimum=float(g["size_minimum"]), stream=g["stream"])
    o.set_alias_mode(alias)
    return o


def oracle_counts_step(orc, row, obs_before, res, nb, nl, lstsq_before):
    """what one oracle step exercised: a failed real descent that wrote loads, an off-leaf success on >= 2 supports, least-squares splits"""
    _, _, d, info = res
    c = dict(failed_with_loads=0, offleaf_multi=0, lstsq=max(orc.n_lstsq - lstsq_before, 0))
    g = orc.support_graph()
    if d and not info.get("error"):
        c["failed_with_loads"] = int(bool(g["failed_box"][0]))  # the failed box's descent left load entries behind
    if not d and not is_leaf(row, obs_before, nb, nl) and len(g["supports"][g["n_box"] - 1]) >= 2:
        c["offleaf_multi"] = 1
    return c
