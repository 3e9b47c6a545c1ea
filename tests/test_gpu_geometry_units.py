"""The stability check's FP64 primitives, one by one, on the device against exact references.

tests/device_units/geom_units.cu includes the product headers unchanged and runs the product's own orient3, cross_left, pip_edge,
pip_rect, hull_coords, pip_shrunk, pip_stored, split2_dir / dot2, lstsq_ratios, around6, hash_double and the resting-height / support
loops, one thread per input.  Every result is compared with a plain restatement in Python floats (IEEE double, correctly rounded
+ - * / and sqrt; fma through fractions.Fraction) and, where the oracle exports the operation, with the oracle (pcto_hull_shrunk,
pcto_pip, pcto_lstsq, pcto_hash_double), bit for bit.  The least-squares solutions are also held against the minimum-norm solution
at 60 digits (mpmath), which oracle parity cannot replace: the oracle shares the solver's truncation rule and sweep cap.

Inputs sit where these functions go wrong: near-ties of the float pre-filters, shared and collinear corners, the `fast` rounding
boundary of pip_rect, rank-deficient and nearly switching least-squares systems, the quick-reject boundaries.  Three mutants show
that the comparisons have teeth: the -fmad=true build of the same source, the pre-filters with tolerance 0, and (CPU) a least-squares
solve without truncation.

The tests without the gpu mark run anywhere: they pin the Python references and the generators against the oracle, and check that
the generators produce the near-ties and branch mixes the GPU tests rely on.
"""
import ctypes as C
import math
import os
from fractions import Fraction

import numpy as np
import pytest

import pct_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UNITS = os.path.join(ROOT, "tests", "device_units", "_build")
OL = pct_oracle.lib()
NB_MAX, KSUP_MAX = 80, 32
EPS = 2.0 ** -52
gpu = pytest.mark.gpu


# ================================================= Python-float references =================================================
def fma(a, b, c):
    """fused multiply-add, correctly rounded (Python 3.12 has no math.fma); an exact zero takes IEEE's sign rule"""
    r = Fraction(a) * Fraction(b) + Fraction(c)
    if r == 0:
        prod_neg = (math.copysign(1.0, a) * math.copysign(1.0, b)) < 0
        return -0.0 if (a * b == 0 and c == 0 and prod_neg and math.copysign(1.0, c) < 0) else 0.0
    return float(r)


def dot2(u0, u1, v0, v1):
    """np.dot on 2-vectors = OpenBLAS ddot: fma(u1, v1, u0 * v0)"""
    return fma(u1, v1, u0 * v0)


def slope(ax, ay, bx, by):
    if bx != ax:
        return (by - ay) / (bx - ax)
    return (by - ay) * math.inf  # 0 * inf = nan, like the reference


def orientation(s1, s2):
    if abs(s1) == math.inf and abs(s2) == math.inf:
        return 0
    d = s2 - s1
    if d > 0:
        return -1
    if d == 0:
        return 0
    return 1


def np_orient(t):
    """orientation(slope(a, b), slope(b, c)) elementwise on an (n, 6) array: numpy's float64 + - * / are the same IEEE operations"""
    ax, ay, bx, by, cx, cy = t.T
    with np.errstate(all="ignore"):
        def sl(px, py, qx, qy):
            dx, dy = qx - px, qy - py
            return np.where(dx != 0, dy / np.where(dx != 0, dx, 1.0), dy * np.inf)
        s1, s2 = sl(ax, ay, bx, by), sl(bx, by, cx, cy)
        d = s2 - s1
        r = np.where(d > 0, -1, np.where(d == 0, 0, 1))
        return np.where(np.isinf(s1) & np.isinf(s2), 0, r).astype(np.int32)


def cross_left_ref(ix, iy, jx, jy, lat, lon):
    t = (lon - iy) / (jy - iy)
    u = t * (jx - ix)
    return ix + u < lat


def hull_ref(pts):
    """ConvexHull of UNPERTURBED points (the perturbation x += y * 1e-6 is applied here, as in pcto_hull_shrunk)"""
    P = sorted([(x + y * 1e-6, y) for x, y in pts], key=lambda p: p[0])  # stable sort by x
    out = []
    for chain in (P, P[::-1]):
        H = []
        for p in chain:
            while len(H) >= 2 and orientation(slope(*H[-2], *H[-1]), slope(*H[-1], *p)) != -1:
                H.pop()
                if H[0] == H[-1]:
                    break
            H.append(p)
        out += H[:-1]
    return out


def scale_down(poly):
    """scale_down in po_scale_down's operation order: sequential sums (not Python's compensated sum()), one division, v - d * 0.1"""
    sx = sy = 0.0
    for x, y in poly:
        sx += x
        sy += y
    n = float(len(poly))
    cx, cy = sx / n, sy / n
    return [(x - (x - cx) * 0.1, y - (y - cy) * 0.1) for x, y in poly]


def pip_ref(lat, lon, c):
    j, odd = len(c) - 1, False
    for i in range(len(c)):
        a0, a1 = c[i][0] - lat, c[i][1] - lon
        b0, b1 = lat - c[j][0], lon - c[j][1]
        if a0 * b1 - a1 * b0 == 0:
            return False
        if (c[i][1] < lon <= c[j][1]) or (c[j][1] < lon <= c[i][1]):
            if cross_left_ref(c[i][0], c[i][1], c[j][0], c[j][1], lat, lon):
                odd = not odd
        j = i
    return odd


def rect_points(rects):
    """combine_contact_points order: (x1,y1) (x1,y2) (x2,y1) (x2,y2) per contact rectangle"""
    return [p for x1, y1, x2, y2 in rects for p in ((x1, y1), (x1, y2), (x2, y1), (x2, y2))]


def oracle_hull_shrunk(pts):
    p = np.ascontiguousarray(pts, dtype=np.float64)
    out = np.zeros((2 * len(pts), 2))
    m = OL.pcto_hull_shrunk(pct_oracle._dp(p), len(pts), pct_oracle._dp(out))
    return np.ascontiguousarray(out[:m])


def oracle_pip(lat, lon, hull):
    return bool(OL.pcto_pip(lat, lon, pct_oracle._dp(hull), len(hull)))


def ls_system(c2x, c2y, cx, cy):
    """the dense system lstsq_ratios streams: one row per pair (a < b), then the row of ones (rhs 1)"""
    k = len(c2x)
    A = []
    for a in range(k - 1):
        for b in range(a + 1, k):
            row = [0.0] * k
            lx, ly = c2x[a] - c2x[b], c2y[a] - c2y[b]
            mol = dot2(cx - c2x[a], cy - c2y[a], lx, ly)
            if mol != 0:
                row[a] = 1.0
                row[b] = -(abs(dot2(cx - c2x[b], cy - c2y[b], lx, ly)) / mol)
            A.append(row)
    A.append([1.0] * k)
    A = np.array(A, dtype=np.float64)
    b = np.zeros(len(A))
    b[-1] = 1.0
    return A, b


def oracle_lstsq(A, b):
    A = np.ascontiguousarray(A)
    x = np.zeros(A.shape[1])
    OL.pcto_lstsq(pct_oracle._dp(A), A.shape[0], A.shape[1], pct_oracle._dp(np.ascontiguousarray(b)), pct_oracle._dp(x))
    return x


def r_diag_ratio(A):
    """max / min |R_ii| of ls_add_row's streaming Givens QR (Python floats, same operation order): the solver back-substitutes iff < 1e4"""
    k = A.shape[1]
    R = [[0.0] * k for _ in range(k)]
    for row in A.tolist():
        for i in range(k):
            bb = row[i]
            if bb == 0:
                continue
            a = R[i][i]
            r = math.sqrt(a * a + bb * bb)
            c, sn = a / r, bb / r
            for j in range(i, k):
                rij, vj = R[i][j], row[j]
                R[i][j] = c * rij + sn * vj
                row[j] = c * vj - sn * rij
    d = [abs(R[i][i]) for i in range(k)]
    return max(d) / min(d) if min(d) > 0 else math.inf


def mp_min_norm(A, rank):
    """minimum-norm least-squares solution at 60 digits: normal equations in mpmath (exact products of the doubles), solved directly
    for full rank, else projected onto the top-`rank` eigenvectors"""
    from mpmath import mp
    mp.dps = 60
    k = A.shape[1]
    G = mp.matrix(k, k)
    for row in A.tolist():
        nz = [(j, mp.mpf(v)) for j, v in enumerate(row) if v != 0]
        for i, vi in nz:
            for j, vj in nz:
                G[i, j] += vi * vj
    rhs = mp.matrix([mp.mpf(v) for v in A[-1]])  # A^T b: b is e_last
    if rank == k:
        x = mp.lu_solve(G, rhs)
        return np.array([float(v) for v in x])
    E, Q = mp.eigsy(G)
    idx = sorted(range(k), key=lambda i: -E[i])[:rank]
    x = [mp.mpf(0)] * k
    for i in idx:
        coef = sum(Q[j, i] * rhs[j] for j in range(k)) / E[i]
        for j in range(k):
            x[j] += Q[j, i] * coef
    return np.array([float(v) for v in x])


# ======================================================= generators =======================================================
def pert(x, y):
    return x + y * 1e-6


def gen_orient(seed=1, scale=1):
    """(n, 6) triples by family: random corners (discrete / continuous), slope near-ties (ulps), relative gaps around the pre-filter
    tolerance (reltol), signs and zeros, vertical segments, horizontal runs, dx made only of the perturbation"""
    rng = np.random.default_rng(seed)
    S = {}
    n = 300000 * scale // 1
    gx, gy = rng.integers(0, 256, (2, n, 3)).astype(np.float64)
    S["disc"] = np.stack([pert(gx, gy), gy], -1).reshape(n, 6)
    cx, cy = np.round(rng.uniform(0, 4, (2, n, 3)), 6)
    S["cont"] = np.stack([pert(cx, cy), cy], -1).reshape(n, 6)
    # near-ties: c continues the line a -> b, then c.y is moved by j ulps (j = -100..100)
    m = 1000 * scale
    fam = []
    for disc in (True, False):
        if disc:
            p = rng.integers(0, 256, (m, 3, 2)).astype(np.float64)
        else:
            p = np.round(rng.uniform(0, 3, (m, 3, 2)), 6)
        ax, ay = pert(p[:, 0, 0], p[:, 0, 1]), p[:, 0, 1]
        bx, by = pert(p[:, 1, 0], p[:, 1, 1]), p[:, 1, 1]
        ok = bx != ax
        ax, ay, bx, by = ax[ok], ay[ok], bx[ok], by[ok]
        dx2 = np.where(rng.random(ax.size) < 0.5, bx - ax, (bx - ax) * rng.uniform(0.1, 3, ax.size))
        s = (by - ay) / (bx - ax)
        cx0, cy0 = bx + dx2, by + s * dx2
        for j in range(-100, 101):
            fam.append(np.stack([ax, ay, bx, by, cx0, cy0 + j * np.spacing(cy0)], 1))
        # exactly collinear: c = 2b - a (exact on these operands), so both slopes are the same quotient
        fam.append(np.stack([ax, ay, bx, by, 2 * bx - ax, 2 * by - ay], 1))
    S["ulps"] = np.concatenate(fam)
    # relative slope gaps g: the float gap / tolerance is ~ g / 2e-4, so 2e-4 * (1 +- 2^-10) straddles the tolerance, 1e-4 sits at half of it
    fam = []
    for g0 in (2e-4, 1e-4):
        for f in (1 + 2.0 ** -10, 1 - 2.0 ** -10):
            fam.append(g0 * f)
    gaps = np.concatenate([np.repeat(fam, 10000 * scale), rng.uniform(5e-5, 6e-4, 60000 * scale)])
    q = gaps.size
    p = np.where(rng.random((q, 1, 1)) < 0.5, rng.integers(0, 256, (q, 2, 2)), np.round(rng.uniform(0, 3, (q, 2, 2)), 6))
    ax, ay = pert(p[:, 0, 0], p[:, 0, 1]), p[:, 0, 1]
    bx, by = pert(p[:, 1, 0], p[:, 1, 1]), p[:, 1, 1]
    ok = (bx != ax) & (by != ay)
    ax, ay, bx, by, gaps = ax[ok], ay[ok], bx[ok], by[ok], gaps[ok]
    s = (by - ay) / (bx - ax)
    dx2 = (bx - ax) * rng.uniform(0.2, 2, ax.size)
    sign = np.where(rng.random(ax.size) < 0.5, 1.0, -1.0)
    S["reltol"] = np.stack([ax, ay, bx, by, bx + dx2, by + s * (1 + sign * gaps) * dx2], 1)
    # signs and zeros: slopes of opposite sign around 0, +-0 numerators (including -0.0 - +0.0 = -0.0)
    k = 20000 * scale
    e = rng.integers(-3, 4, (k, 3)).astype(np.float64) * 1e-6
    x = np.sort(rng.uniform(0, 3, (k, 3)), axis=1)
    y0 = np.choose(rng.integers(0, 3, (k, 3)), [np.zeros((k, 3)), -np.zeros((k, 3)), e])
    S["signs"] = np.stack([x[:, 0], y0[:, 0], x[:, 1], y0[:, 1], x[:, 2], y0[:, 2]], 1)
    # vertical segments (dx == 0), horizontal runs (dy == 0), dx made only of the perturbation (same x before x += y * 1e-6)
    xs = rng.integers(0, 256, (k, 3)).astype(np.float64)
    ys = rng.integers(0, 256, (k, 3)).astype(np.float64)
    xv = xs.copy()
    xv[:, 1] = np.where(rng.random(k) < 0.5, xv[:, 0], xv[:, 2])
    S["vertical"] = np.stack([xv[:, 0], ys[:, 0], xv[:, 1], ys[:, 1], xv[:, 2], ys[:, 2]], 1)
    yh = np.repeat(ys[:, :1], 3, 1)
    yh[:, 2] = np.where(rng.random(k) < 0.5, yh[:, 2], ys[:, 2])
    S["horizontal"] = np.stack([pert(xs[:, 0], yh[:, 0]), yh[:, 0], pert(xs[:, 1], yh[:, 1]), yh[:, 1], pert(xs[:, 2], yh[:, 2]), yh[:, 2]], 1)
    xp = np.repeat(xs[:, :1], 3, 1)
    xp[:, 2] = np.where(rng.random(k) < 0.5, xp[:, 2], xs[:, 2])
    S["pert_dx"] = np.stack([pert(xp[:, 0], ys[:, 0]), ys[:, 0], pert(xp[:, 1], ys[:, 1]), ys[:, 1], pert(xp[:, 2], ys[:, 2]), ys[:, 2]], 1)
    return S


def prefilter_f32(t):
    """float32 emulation of orient3's pre-filter (exact float division instead of __fdividef): coverage accounting only.
    Returns (branch, |gap| / tol) with branch 0 exact path, 1 decided, 2 horizontal early-out"""
    ax, ay, bx, by, cx, cy = t.T
    d1x, d1y, d2x, d2y = bx - ax, by - ay, cx - bx, cy - by
    with np.errstate(all="ignore"):
        f1 = d1y.astype(np.float32) / d1x.astype(np.float32)
        f2 = d2y.astype(np.float32) / d2x.astype(np.float32)
        gap = f2 - f1
        tol = np.float32(1e-4) * (np.abs(f1) + np.abs(f2))
        ratio = np.abs(gap) / tol
    live = (d1x != 0) & (d2x != 0)
    hor = live & (d1y == 0) & (d2y == 0)
    dec = live & ~hor & (np.abs(gap) > tol) & (np.abs(f1) < 1e30) & (np.abs(f2) < 1e30)
    return np.where(hor, 2, np.where(dec, 1, 0)), np.where(live & ~hor, ratio, -1.0)


def gen_cross(seed=2):
    """(n, 6) = (ix, iy, jx, jy, lat, lon) with lon strictly between iy and jy; lat = the crossing abscissa the exact expression gives,
    moved by 0, +-1, +-k ulps, and lat at the pre-filter boundary 1e-4 * scale * (1 +- 2^-10).  Integer, 6-decimal and shrunk-looking edges."""
    rng = np.random.default_rng(seed)
    rows = []
    for kind in range(3):
        n = 6000
        if kind == 0:
            e = rng.integers(0, 256, (n, 4)).astype(np.float64)
        elif kind == 1:
            e = np.round(rng.uniform(0, 4, (n, 4)), 6)
        else:
            e = rng.uniform(0, 255, (n, 4)) + rng.integers(0, 256, (n, 4)) * 1e-6
        ix, iy, jx, jy = e.T
        ok = iy != jy
        ix, iy, jx, jy = ix[ok], iy[ok], jx[ok], jy[ok]
        lo, hi = np.minimum(iy, jy), np.maximum(iy, jy)
        lon = lo + (hi - lo) * rng.uniform(0.01, 0.99, ix.size)
        X = ix + (lon - iy) / (jy - iy) * (jx - ix)
        for j in list(range(-4, 5)) + [-64, -16, 16, 64]:
            rows.append(np.stack([ix, iy, jx, jy, X + j * np.spacing(X), lon], 1))
        sc = np.abs(ix) + np.abs(jx - ix) + np.abs(X)
        for f in (1 + 2.0 ** -10, 1 - 2.0 ** -10, 2.0):
            for sg in (1, -1):
                rows.append(np.stack([ix, iy, jx, jy, X + sg * 1e-4 * sc * f, lon], 1))
    return np.concatenate(rows)


def gen_layouts(seed=3):
    """contact-rectangle layouts with k = 1..32 supports: (kind, rects)"""
    rng = np.random.default_rng(seed)
    L = []
    for k in range(1, 33):
        for rep in range(3):
            # unit grid (shared corners and collinear edges)
            cells = rng.choice(64, size=k, replace=False)
            L.append(("grid", [(float(c % 8), float(c // 8), float(c % 8 + 1), float(c // 8 + 1)) for c in cells]))
            # adjacent rectangles in a row / column sharing corners and one collinear edge line
            x = np.cumsum(rng.integers(1, 8, k + 1)).astype(float)
            y0, y1 = float(rng.integers(0, 100)), float(rng.integers(101, 255))
            L.append(("row", [(x[i], y0, x[i + 1], y1) for i in range(k)]))
            # random rectangles in a 255-wide bin (largest perturbation)
            r = []
            for _ in range(k):
                a, b = sorted(rng.choice(256, 2, replace=False))
                c, d = sorted(rng.choice(256, 2, replace=False))
                r.append((float(a), float(c), float(b), float(d)))
            L.append(("bin255", r))
            # continuous 6-decimal rectangles, and rectangles only 1e-6 wide
            r = []
            for _ in range(k):
                a, c = np.round(rng.uniform(0, 3, 2), 6)
                w, h = np.round(rng.uniform(1e-6, 1, 2), 6)
                r.append((a, c, round(a + w, 6), round(c + h, 6)))
            L.append(("cont", r))
            r = []
            for _ in range(k):
                a, c = np.round(rng.uniform(0, 3, 2), 6)
                h = round(float(rng.uniform(1e-6, 2)), 6)
                r.append((a, c, round(a + 1e-6, 6), round(c + h, 6)))
            L.append(("thin", r))
    # k = 1: the `fast` precondition of pip_rect around its rounding boundary (width w, height ~ w * 1e6: x2 + t1 vs x1 + t2)
    for _ in range(400):
        a, c = np.round(rng.uniform(0, 255, 2), 6)
        w = float(rng.choice([1e-6, 2e-6, 5e-6]))
        h = w * 1e6 * float(rng.choice([0.5, 1 - 1e-6, 1.0, 1 + 1e-6, 2.0]))
        L.append(("fastb", [(a, c, a + w, round(c + h, 6))]))
    return L


def layout_queries(rects, hull_shrunk, rng):
    """the centre, vertices and shrunk edges of the polygon, one ulp on either side, the unperturbed rectangle edges, random points"""
    q = []
    xs = [v[0] for v in hull_shrunk]
    ys = [v[1] for v in hull_shrunk]
    q.append(((min(xs) + max(xs)) * 0.5, (min(ys) + max(ys)) * 0.5))
    m = len(hull_shrunk)
    for i in range(m):
        (x0, y0), (x1, y1) = hull_shrunk[i], hull_shrunk[(i + 1) % m]
        for px, py in ((x0, y0), ((x0 + x1) * 0.5, (y0 + y1) * 0.5)):
            q.append((px, py))
            q.append((math.nextafter(px, math.inf), py))
            q.append((math.nextafter(px, -math.inf), py))
            q.append((px, math.nextafter(py, math.inf)))
            q.append((px, math.nextafter(py, -math.inf)))
    for x1, y1, x2, y2 in rects[:4]:
        q += [(x1, y1), (x2, y2), ((x1 + x2) * 0.5, y1), (x1, (y1 + y2) * 0.5), ((x1 + x2) * 0.5, (y1 + y2) * 0.5)]
    lo_x, hi_x, lo_y, hi_y = min(xs), max(xs), min(ys), max(ys)
    for _ in range(6):
        q.append((float(rng.uniform(lo_x - 0.1, hi_x + 0.1)), float(rng.uniform(lo_y - 0.1, hi_y + 0.1))))
    return q


def gen_lstsq(seed=4, n_random=1400):
    """least-squares systems of lstsq_ratios: (kind, centres x, centres y, com x, com y, rank by construction or None = full)
    rank-deficient families: every centre identical (all pair rows zero: rank 1), and two clusters whose centre of mass projects exactly
    onto the cluster P (molecular == 0): with the other cluster Q first, the rows of Q force x_Q = 0 (rank |Q| + 1); with P first every
    row is zero (rank 1).  The minimum-norm solutions are 1/k each, resp. 0 on Q and 1/|P| on P."""
    rng = np.random.default_rng(seed)
    S = []

    def centre(r):
        return (r[0] + r[2]) * 0.5, (r[1] + r[3]) * 0.5
    for i in range(n_random):
        k = int(rng.choice(list(range(3, 9)) * 3 + list(range(9, 33)))) if i % 4 else int(rng.integers(3, 33))
        disc = i % 2 == 0
        cx2, cy2 = [], []
        for _ in range(k):
            if disc:
                a, b = sorted(rng.choice(256, 2, replace=False))
                c, d = sorted(rng.choice(256, 2, replace=False))
                x, y = centre((float(a), float(c), float(b), float(d)))
            else:
                a, c = np.round(rng.uniform(0, 3, 2), 6)
                w, h = np.round(rng.uniform(1e-6, 1, 2), 6)
                x, y = centre((a, c, round(a + w, 6), round(c + h, 6)))
            cx2.append(x)
            cy2.append(y)
        com = (float(rng.uniform(min(cx2), max(cx2))), float(rng.uniform(min(cy2), max(cy2))))
        if not disc:
            com = (round(com[0], 6), round(com[1], 6))
        S.append(("random", cx2, cy2, com[0], com[1], None))
    # collinear centres (a horizontal / vertical / diagonal line) and symmetric grids with the centre of mass at their centre
    for i in range(200):
        k = int(rng.integers(3, 33))
        t = sorted(rng.choice(512, k, replace=False) * 0.5)
        d = i % 3
        cx2 = [float(v) if d != 1 else 7.5 for v in t]
        cy2 = [3.0 if d == 0 else float(v) for v in t]
        com = (float(rng.uniform(min(cx2), max(cx2) + 1)), float(rng.uniform(min(cy2), max(cy2) + 1)))
        S.append(("collinear", cx2, cy2, com[0], com[1], None))
    for i in range(120):
        nx, ny = int(rng.integers(2, 6)), int(rng.integers(2, 7))
        sx, sy = float(rng.integers(1, 9)), float(rng.integers(1, 9))
        cx2 = [1.5 + sx * a for a in range(nx) for b in range(ny)]
        cy2 = [2.5 + sy * b for a in range(nx) for b in range(ny)]
        S.append(("grid", cx2, cy2, 1.5 + sx * (nx - 1) * 0.5, 2.5 + sy * (ny - 1) * 0.5, None))
    # rank-deficient by construction
    for i in range(140):
        k = int(rng.integers(3, 33))
        p = (float(rng.integers(0, 256)) + 0.5, float(rng.integers(0, 256)))
        S.append(("same", [p[0]] * k, [p[1]] * k, float(rng.uniform(0, 256)), float(rng.uniform(0, 256)), 1))
    for i in range(240):
        k = int(rng.integers(3, 33))
        nq = int(rng.integers(1, k - 1))  # |P| = k - nq >= 2
        p = (float(rng.integers(0, 200)) + 0.5, float(rng.integers(0, 200)))
        u = (float(rng.integers(-4, 5)), float(rng.integers(1, 5)))  # direction P -> Q; the centre of mass sits on the perpendicular through P
        s, t = float(rng.integers(1, 8)), float(rng.integers(-6, 7))
        q = (p[0] + s * u[0], p[1] + s * u[1])
        com = (p[0] - t * u[1], p[1] + t * u[0])
        q_first = i % 2 == 0
        if q_first:
            cx2, cy2, rank = [q[0]] * nq + [p[0]] * (k - nq), [q[1]] * nq + [p[1]] * (k - nq), nq + 1
        else:
            cx2, cy2, rank = [p[0]] * (k - nq) + [q[0]] * nq, [p[1]] * (k - nq) + [q[1]] * nq, 1
        S.append(("perp_q" if q_first else "perp_p", cx2, cy2, com[0], com[1], rank))
    # R diagonal ratio near the 1e4 switch between back-substitution and the SVD: the centre of mass approaches one centre
    sw = 0
    while sw < 160:
        k = int(rng.integers(3, 7))
        cx2 = [float(v) + 0.5 for v in rng.integers(0, 100, k)]
        cy2 = [float(v) for v in rng.integers(0, 100, k)]
        if len(set(zip(cx2, cy2))) < k:
            continue
        ang = rng.uniform(0, 2 * np.pi)
        for dlt in np.logspace(-1, -6, 120):
            com = (cx2[0] + dlt * math.cos(ang), cy2[0] + dlt * math.sin(ang))
            A, _ = ls_system(cx2, cy2, *com)
            r = r_diag_ratio(A)
            if 5e3 < r < 2e4:
                S.append(("switch", cx2, cy2, com[0], com[1], None))
                sw += 1
    return S


def closed_form(kind, cx2, cy2, rank):
    k = len(cx2)
    if rank == 1:
        return np.full(k, 1.0 / k)
    p = (cx2[-1], cy2[-1])  # perp_q: P is the tail
    on_p = np.array([(x, y) == p for x, y in zip(cx2, cy2)])
    return np.where(on_p, 1.0 / on_p.sum(), 0.0)


# ================================================ device unit library access ================================================
def _torch():
    return pytest.importorskip("torch")


def _units(fmad=False):
    path = os.path.join(UNITS, "libgeom_units_fmad.so" if fmad else "libgeom_units.so")
    if not os.path.exists(path):
        raise RuntimeError("%s is missing: build() (make -C tests/device_units) builds it" % path)
    return C.CDLL(path)


def _dev(a, dtype=None):
    torch = _torch()
    return torch.from_numpy(np.ascontiguousarray(a if dtype is None else np.asarray(a, dtype=dtype))).cuda()


def _run(fn, *args):
    torch = _torch()
    conv = []
    for a in args:
        if torch.is_tensor(a):
            conv.append(C.c_void_p(a.data_ptr()))
        elif isinstance(a, tuple):  # ("ll", value): a 64-bit integer argument
            conv.append(C.c_longlong(a[1]))
        else:
            conv.append(C.c_int(a))
    rc = fn(*conv)
    assert rc == 0, "CUDA error %d" % rc


def dev_orient3(t, L=None):
    torch = _torch()
    L = L or _units()
    d = _dev(t, np.float64)
    out = torch.zeros((len(t), 4), dtype=torch.int32, device="cuda")
    ratio = torch.zeros(len(t), dtype=torch.float32, device="cuda")
    _run(L.gu_orient3, d, len(t), out, ratio)
    return out.cpu().numpy(), ratio.cpu().numpy()


def dev_cross_left(t, L=None):
    torch = _torch()
    L = L or _units()
    out = torch.zeros((len(t), 3), dtype=torch.int32, device="cuda")
    _run(L.gu_cross_left, _dev(t, np.float64), len(t), out)
    return out.cpu().numpy()


def dev_polygons(polys, L=None):
    """hull_coords of each polygon's perturbed points -> (m, hx, hy, raw device tensors)"""
    torch = _torch()
    L = L or _units()
    off = np.zeros(len(polys) + 1, dtype=np.int32)
    off[1:] = np.cumsum([len(p) for p in polys])
    assert max(len(p) for p in polys) <= 4 * KSUP_MAX
    pts = np.array([(pert(x, y), y) for p in polys for x, y in p], dtype=np.float64)
    px, py = _dev(pts[:, 0]), _dev(pts[:, 1])
    hx = torch.zeros(2 * int(off[-1]), dtype=torch.float64, device="cuda")
    hy = torch.zeros_like(hx)
    m = torch.zeros(len(polys), dtype=torch.int32, device="cuda")
    offd = _dev(off)
    _run(L.gu_hull, px, py, offd, len(polys), hx, hy, m)
    return m, hx, hy, _dev(2 * off[:-1])


# ======================================================= CPU tests =======================================================
def test_references_match_oracle_hull_and_pip():
    rng = np.random.default_rng(7)
    n_pip = 0
    for kind, rects in gen_layouts()[::3]:
        pts = rect_points(rects)
        want = oracle_hull_shrunk(pts)
        got = scale_down(hull_ref(pts))
        assert np.array_equal(np.array(got), want), kind
        for lat, lon in layout_queries(rects, got, rng):
            assert pip_ref(lat, lon, got) == oracle_pip(lat, lon, want)
            n_pip += 1
    assert n_pip > 10000


def test_references_match_oracle_orientation():
    """np_orient (the vectorised reference the GPU test uses) against the scalar restatement that hull_ref, pinned to the oracle's hull
    above, is built on: every family, including the near-ties"""
    S = gen_orient(scale=1)
    for name in ("ulps", "reltol", "signs", "vertical", "horizontal", "pert_dx"):
        t = S[name][::97]
        want = [orientation(slope(*r[:4]), slope(*r[2:])) for r in t.tolist()]
        assert np.array_equal(np_orient(t), np.array(want, dtype=np.int32)), name


def test_references_match_oracle_lstsq():
    """ls_system (Fraction fma for dot2) + pcto_lstsq on the generated systems: the oracle solves them at the minimum-norm solution"""
    S = gen_lstsq(n_random=300)
    worst = 0.0
    for kind, cx2, cy2, cx, cy, rank in S[::3]:
        A, b = ls_system(cx2, cy2, cx, cy)
        x = oracle_lstsq(A, b)
        ref, cond = _lstsq_reference(kind, A, cx2, cy2, rank)
        err = np.max(np.abs(x - ref)) / max(np.max(np.abs(ref)), 1e-300)
        worst = max(worst, err / (cond * EPS))
        assert err <= LS_C * len(cx2) * cond * EPS, (kind, len(cx2), err, cond)
    assert worst > 0


LS_C = 8  # tolerance factor of the least-squares comparison: |x - x*|_inf <= LS_C * k * cond * eps * |x*|_inf


def _lstsq_reference(kind, A, cx2, cy2, rank):
    """(minimum-norm solution, condition number of the kept spectrum); the numerical rank must equal the construction's, with a gap"""
    k = A.shape[1]
    s = np.linalg.svd(A, compute_uv=False)
    r = k if rank is None else rank
    assert s[r - 1] > 1e-9 * s[0] and (r == k or s[r] < 1e-13 * s[0]), (kind, k, s[0], s[r - 1], s[r] if r < k else None)
    if rank is None:
        ref = mp_min_norm(A, k)
    else:
        ref = closed_form(kind, cx2, cy2, rank)
    return ref, s[0] / s[r - 1]


def test_rank_deficient_closed_forms_are_the_minimum_norm_solutions():
    S = [s for s in gen_lstsq(n_random=0) if s[5] is not None and len(s[1]) <= 10]
    for kind, cx2, cy2, cx, cy, rank in S[::4]:
        A, _ = ls_system(cx2, cy2, cx, cy)
        assert np.allclose(mp_min_norm(A, rank), closed_form(kind, cx2, cy2, rank), rtol=1e-14, atol=1e-15), kind


def test_rank_deficient_set_separates_a_solve_without_truncation():
    """the normal equations solved without truncation miss the minimum-norm solution on the rank-deficient family"""
    S = [s for s in gen_lstsq(n_random=0) if s[5] is not None]
    miss = 0
    for kind, cx2, cy2, cx, cy, rank in S:
        A, b = ls_system(cx2, cy2, cx, cy)
        ref = closed_form(kind, cx2, cy2, rank)
        try:
            x = np.linalg.solve(A.T @ A, A.T @ b)
            miss += not np.allclose(x, ref, rtol=1e-6, atol=1e-9)
        except np.linalg.LinAlgError:
            miss += 1
    assert miss >= len(S) // 2, (miss, len(S))


def test_dot2_set_separates_an_unfused_dot():
    """u0 * v0 + u1 * v1 without the fma differs from dot2 on the two-support split inputs"""
    T = gen_split2()
    diff = sum(dot2(r[4] - r[1], r[5] - r[3], r[0] - r[1], r[2] - r[3]) != (r[4] - r[1]) * (r[0] - r[1]) + (r[5] - r[3]) * (r[2] - r[3])
               for r in T.tolist())
    assert diff > 100


def test_generators_cover_both_prefilter_branches():
    S = gen_orient(scale=1)
    n = sum(len(v) for v in S.values())
    assert n >= 1_000_000
    br, ratio = prefilter_f32(np.concatenate([S["ulps"], S["reltol"]]))
    assert np.sum((br == 1) & (ratio <= 2)) >= 10000 and np.sum(br == 0) >= 10000
    br, _ = prefilter_f32(np.concatenate([S["vertical"], S["horizontal"], S["pert_dx"], S["signs"]]))
    assert np.sum(br == 2) >= 1000 and np.sum(br == 0) >= 1000


def test_generators_produce_exact_near_ties():
    """the ulps family holds exactly collinear triples and triples whose exact slopes differ by a few ulps (classified with Fraction)"""
    t = gen_orient(scale=1)["ulps"][::41]
    same = close = 0
    for ax, ay, bx, by, cx, cy in t.tolist():
        if bx == ax or cx == bx:
            continue
        s1 = (Fraction(by) - Fraction(ay)) / (Fraction(bx) - Fraction(ax))
        s2 = (Fraction(cy) - Fraction(by)) / (Fraction(cx) - Fraction(bx))
        if s1 == s2:
            same += 1
        elif abs(s2 - s1) <= 100 * abs(s1) * Fraction(EPS):
            close += 1
    assert same >= 20 and close >= 1000, (same, close)


def test_generators_reach_the_lstsq_switch_and_the_svd():
    S = gen_lstsq(n_random=200)
    kinds = {}
    svd = back = 0
    for kind, cx2, cy2, cx, cy, rank in S[::2]:
        kinds[kind] = kinds.get(kind, 0) + 1
        if len(cx2) <= 8:
            A, _ = ls_system(cx2, cy2, cx, cy)
            r = r_diag_ratio(A)
            svd += r >= 1e4
            back += r < 1e4
            if kind == "switch":
                assert 5e3 < r < 2e4
    assert svd >= 20 and back >= 20, (svd, back)
    assert min(kinds.values()) >= 10, kinds
    assert max(len(s[1]) for s in S) == 32


def gen_split2(seed=5):
    """(n, 7) = (px0, px1, py0, py1, cx, cy, m): two contact-rectangle centres (halves of integer / 6-decimal sums), a stack centre, a mass"""
    rng = np.random.default_rng(seed)
    n = 20000
    disc = rng.random(n) < 0.5
    p = np.where(disc[:, None], rng.integers(0, 511, (n, 4)) * 0.5, np.round(rng.uniform(0, 6, (n, 4)), 6) * 0.5)
    c = np.where(disc[:, None], rng.uniform(0, 255, (n, 2)), np.round(rng.uniform(0, 3, (n, 2)), 6))
    mass = np.where(disc, rng.integers(1, 2000, n).astype(float), np.round(rng.uniform(0.001, 8, n), 6))
    t = np.stack([p[:, 0], p[:, 1], p[:, 2], p[:, 3], c[:, 0], c[:, 1], mass], 1)
    return t[(t[:, 0] != t[:, 1]) | (t[:, 2] != t[:, 3])]


def split2_ref(r):
    px0, px1, py0, py1, cx, cy, m = r
    lx, ly = px0 - px1, py0 - py1
    ln = math.sqrt(fma(ly, ly, lx * lx))
    l2 = ln * ln
    lx, ly = lx / l2, ly / l2
    return (lx, ly, m * abs(dot2(cx - px1, cy - py1, lx, ly)), m * abs(dot2(cx - px0, cy - py0, lx, ly)), dot2(px0, py0, px1, py1), 0.0)


# ======================================================= GPU tests =======================================================
@gpu
def test_orient3_on_device():
    S = gen_orient(scale=1)
    L = _units()
    n_dec2 = n_fall = 0
    mut = 0
    for name, t in S.items():
        out, ratio = dev_orient3(t, L)
        want = np_orient(t)
        bad = np.nonzero(out[:, 0] != want)[0]
        assert bad.size == 0, (name, bad.size, t[bad[:3]].tolist(), out[bad[:3]].tolist(), want[bad[:3]].tolist())
        assert np.array_equal(out[:, 1], want), name  # the exact path alone
        if name in ("ulps", "reltol"):
            n_dec2 += int(np.sum((out[:, 2] == 1) & (ratio <= 2)))
            n_fall += int(np.sum(out[:, 2] == 0))
            mut += int(np.sum(out[:, 3] != want))
    assert n_dec2 >= 10000 and n_fall >= 10000, (n_dec2, n_fall)
    assert mut > 0, "orient3 with tolerance 0 agrees with the reference on every near-tie"


@gpu
def test_cross_left_on_device():
    t = gen_cross()
    out = dev_cross_left(t)
    want = np.array([cross_left_ref(*r) for r in t.tolist()], dtype=np.int32)
    assert np.array_equal(out[:, 0], want)
    assert np.sum(out[:, 1] == 0) >= 10000 and np.sum(out[:, 1] == 1) >= 10000
    assert np.sum(out[:, 2] != want) > 0, "cross_left with tolerance 0 agrees with the reference on every near-tie"


def _polygon_sets(seed=7):
    rng = np.random.default_rng(seed)
    lays = gen_layouts()
    polys, shrunk, queries = [], [], []
    for kind, rects in lays:
        pts = rect_points(rects)
        hs = oracle_hull_shrunk(pts)
        polys.append(pts)
        shrunk.append(hs)
        queries.append(layout_queries(rects, [tuple(v) for v in hs.tolist()], rng))
    return lays, polys, shrunk, queries


def _device_polygons(L, lays, polys, shrunk, queries):
    """hull_coords, pip_shrunk, pip_stored, pip_rect and pip_edge of every layout on the device"""
    torch = _torch()
    m, hx, hy, hoff = dev_polygons(polys, L)
    m_h = m.cpu().numpy()
    hx_h, hy_h, hoff_h = hx.cpu().numpy(), hy.cpu().numpy(), hoff.cpu().numpy()
    hulls = [list(zip(hx_h[o:o + c], hy_h[o:o + c])) for o, c in zip(hoff_h, m_h)]
    qpoly = np.array([i for i, q in enumerate(queries) for _ in q], dtype=np.int32)
    qxy = np.array([p for q in queries for p in q], dtype=np.float64)
    res = torch.zeros(len(qpoly), dtype=torch.int32, device="cuda")
    _run(L.gu_pip_shrunk, hx, hy, hoff, m, _dev(qpoly), _dev(qxy), len(qpoly), res)
    pip_sh = res.cpu().numpy()
    soff = np.zeros(len(shrunk) + 1, dtype=np.int32)
    soff[1:] = np.cumsum([len(s) for s in shrunk])
    _run(L.gu_pip_stored, _dev(np.concatenate(shrunk).reshape(-1)), _dev(soff), _dev(qpoly), _dev(qxy), len(qpoly), res)
    pip_st = res.cpu().numpy()
    # k = 1: pip_rect where `fast` holds
    one = [(i, lays[i][1][0]) for i in range(len(lays)) if len(lays[i][1]) == 1]
    rq = np.array([(*r, *p) for i, r in one for p in queries[i]], dtype=np.float64)
    rres = torch.zeros((len(rq), 2), dtype=torch.int32, device="cuda")
    _run(L.gu_pip_rect, _dev(rq), len(rq), rres)
    return m_h, hulls, qpoly, qxy, pip_sh, pip_st, one, rq, rres.cpu().numpy()


@gpu
def test_polygons_on_device():
    lays, polys, shrunk, queries = _polygon_sets()
    L = _units()
    m_h, hulls, qpoly, qxy, pip_sh, pip_st, one, rq, rres = _device_polygons(L, lays, polys, shrunk, queries)
    for i, h in enumerate(hulls):
        assert m_h[i] == len(shrunk[i]), (lays[i][0], i)
        assert np.array_equal(np.array(scale_down(h)), shrunk[i]), (lays[i][0], i)
    want = np.array([oracle_pip(x, y, shrunk[p]) for p, (x, y) in zip(qpoly, qxy)], dtype=np.int32)
    assert np.array_equal(pip_sh, want)
    assert np.array_equal(pip_st, want)
    assert np.sum(want == 1) >= 1000 and np.sum(want == 0) >= 1000
    fast = rres[:, 0] == 1
    assert fast.sum() >= 1000 and (~fast).sum() >= 100, (fast.sum(), (~fast).sum())
    rwant = np.array([oracle_pip(r[4], r[5], oracle_hull_shrunk(rect_points([tuple(r[:4])]))) for r in rq], dtype=np.int32)
    assert np.array_equal(rres[fast, 1], rwant[fast])
    # pip_edge on the edges of the shrunk hulls: 2 (collinear) / 1 (toggle) / 0, as point_in_polygen decides per edge
    ed = []
    for p, (x, y) in list(zip(qpoly, qxy))[::5]:
        h = shrunk[p]
        for i in range(len(h)):
            j = i - 1
            ed.append((h[i][0], h[i][1], h[j][0], h[j][1], x, y))
    ed = np.array(ed, dtype=np.float64)
    torch = _torch()
    eres = torch.zeros(len(ed), dtype=torch.int32, device="cuda")
    _run(L.gu_pip_edge, _dev(ed), len(ed), eres)

    def edge_ref(ix, iy, jx, jy, lat, lon):
        if (ix - lat) * (lon - jy) - (iy - lon) * (lat - jx) == 0:
            return 2
        if (iy < lon <= jy) or (jy < lon <= iy):
            return int(cross_left_ref(ix, iy, jx, jy, lat, lon))
        return 0
    ew = np.array([edge_ref(*r) for r in ed.tolist()], dtype=np.int32)
    assert np.array_equal(eres.cpu().numpy(), ew)
    assert np.sum(ew == 2) > 0 and np.sum(ew == 1) > 0


@gpu
def test_split2_and_dot2_on_device():
    torch = _torch()
    t = gen_split2()
    out = torch.zeros((len(t), 6), dtype=torch.float64, device="cuda")
    _run(_units().gu_split2, _dev(t), len(t), out)
    want = np.array([split2_ref(r) for r in t.tolist()])
    got = out.cpu().numpy()
    assert np.array_equal(got.view(np.int64), want.view(np.int64))


def _lstsq_inputs(S):
    off = np.zeros(len(S) + 1, dtype=np.int32)
    off[1:] = np.cumsum([len(s[1]) for s in S])
    c2x = np.concatenate([s[1] for s in S]).astype(np.float64)
    c2y = np.concatenate([s[2] for s in S]).astype(np.float64)
    com = np.array([(s[3], s[4]) for s in S], dtype=np.float64)
    return off, c2x, c2y, com


def dev_lstsq(S, L):
    torch = _torch()
    off, c2x, c2y, com = _lstsq_inputs(S)
    assert max(len(s[1]) for s in S) <= KSUP_MAX
    stride = L.gu_lstsq_stride()
    scratch = torch.full((len(S) * stride,), float("nan"), dtype=torch.float64, device="cuda")
    x = torch.zeros(int(off[-1]), dtype=torch.float64, device="cuda")
    _run(L.gu_lstsq, _dev(c2x), _dev(c2y), _dev(off), _dev(com), len(S), scratch, x)
    xh = x.cpu().numpy()
    return [xh[off[i]:off[i + 1]] for i in range(len(S))]


@gpu
def test_lstsq_on_device():
    S = gen_lstsq()
    assert len(S) >= 2000
    xs = dev_lstsq(S, _units())
    for (kind, cx2, cy2, cx, cy, rank), x in zip(S, xs):
        A, b = ls_system(cx2, cy2, cx, cy)
        want = oracle_lstsq(A, b)
        assert np.array_equal(x.view(np.int64), want.view(np.int64)), (kind, len(cx2), x, want)
        ref, cond = _lstsq_reference(kind, A, cx2, cy2, rank)
        err = np.max(np.abs(x - ref)) / np.max(np.abs(ref))
        assert err <= LS_C * len(cx2) * cond * EPS, (kind, len(cx2), err, cond)


@gpu
def test_around6_exhaustive_on_device():
    """every integer |a| <= 2.2e9 (4.4e9 operands, in chunks) and the operands around the 2.2e9 fallback boundary"""
    torch = _torch()
    L = _units()
    cnt = torch.zeros(4, dtype=torch.int64, device="cuda")
    lim, step = 2_200_000_000, 1 << 30
    lo = -lim
    while lo <= lim:
        hi = min(lo + step, lim + 1)
        _run(L.gu_around6_range, ("ll", lo), ("ll", hi), cnt)
        lo = hi
    for c in (lim, -lim):
        _run(L.gu_around6_range, ("ll", c - 1_000_000), ("ll", c + 1_000_000), cnt)
    bad_rint, bad, bad_q0, seen = cnt.cpu().tolist()
    assert seen == 2 * lim + 1 + 4_000_000
    assert bad_rint == 0 and bad == 0
    assert 0.2 * seen < bad_q0 < 0.4 * seen  # the uncorrected quotient alone would be wrong on ~30 % of them


@gpu
def test_around6_and_hash_double_samples_on_device():
    torch = _torch()
    L = _units()
    rng = np.random.default_rng(9)
    k = rng.integers(-3_000_000_000, 3_000_000_000, 200000).astype(np.float64)
    with np.errstate(over="ignore"):
        v = np.concatenate([rng.uniform(-3000, 3000, 400000), (k + 0.5) / 1e6, np.nextafter((k + 0.5) / 1e6, np.inf),
                            np.nextafter((k + 0.5) / 1e6, -np.inf), rng.uniform(-1, 1, 100000) * 10.0 ** rng.integers(3, 300, 100000),
                            [0.0, -0.0, 2199.9999995, -2199.9999995, 2200.0000005, 2200.000001]])
        want = np.rint(v * 1e6) / 1e6
    out = torch.zeros(v.size, dtype=torch.float64, device="cuda")
    _run(L.gu_around6, _dev(v), v.size, out)
    assert np.array_equal(out.cpu().numpy().view(np.int64), want.view(np.int64))
    bits = rng.integers(0, 2 ** 63 - 1, 300000, dtype=np.int64)
    bits = bits[((bits >> 52) & 0x7FF) != 0x7FF]
    sub = rng.integers(1, 2 ** 52, 100000, dtype=np.int64)
    p61 = float(2 ** 61)
    h = np.concatenate([bits.view(np.float64), sub.view(np.float64), -sub.view(np.float64), rng.uniform(-3, 3, 300000),
                        np.round(rng.uniform(0, 3, 200000), 6), [0.0, -0.0, 5e-324, -5e-324, p61, -p61, 1.0, -1.0, 2.0 ** 1023],
                        np.nextafter(p61, 0) - np.arange(50) * 256.0, p61 + np.arange(50) * 512.0,
                        (2.0 ** 61 - 1) * np.arange(1, 50), [float(2 ** 61 - 1) * 2 ** e for e in range(-70, 70)]])
    assert h.size >= 1_000_000
    outh = torch.zeros(h.size, dtype=torch.int64, device="cuda")
    _run(L.gu_hash_double, _dev(h), h.size, outh)
    want = np.array([hash(float(x)) & ((1 << 64) - 1) for x in h.tolist()], dtype=np.uint64)
    assert np.array_equal(outh.cpu().numpy().view(np.uint64), want)
    sample = h[::997]
    assert all(OL.pcto_hash_double(float(x)) == hash(float(x)) & ((1 << 64) - 1) for x in sample)


def gen_layouts_d(seed=11):
    """discrete box layouts (W = 255 or 10): support boxes with a common top at height 5 over lower boxes; each query footprint overlaps
    them near an edge, with the doubled centre at 2 * X2 + 1 (and its mirror / y analogue) among the sweep"""
    rng = np.random.default_rng(seed)
    lays, qs = [], []
    for li in range(40):
        W = 255 if li % 2 else 10
        boxes = []
        for _ in range(int(rng.integers(1, 12))):
            a, b = sorted(rng.integers(0, W + 1, 2))
            c, d = sorted(rng.integers(0, W + 1, 2))
            if a == b or c == d:
                continue
            top = int(rng.choice([5, 5, 3]))
            boxes.append((a, c, 0, b, d, top))
        if not boxes:
            continue
        arr = np.zeros((NB_MAX, 6), dtype=np.int16)
        arr[:len(boxes)] = boxes
        lay = len(lays)
        lays.append((arr, len(boxes)))
        for a, c, _, b, d, top in boxes:
            for dx in (1, 3, 5, 8):
                for dy in (1, 3, 5):
                    for lx in range(max(a - dx, 0), min(b + 1, W - dx + 1)):
                        for ly in (c, max(c - (dy - 1) // 2, 0), max(d - dy + 1, 0), max(d - (dy - 1) // 2, 0)):
                            if rng.random() < (0.04 if W == 255 else 0.5):
                                qs.append((lay, lx, ly, dx, dy))
    return lays, np.array(qs, dtype=np.int32)


@gpu
def test_discrete_quick_reject_on_device():
    torch = _torch()
    lays, q = gen_layouts_d()
    L = _units()
    boxes = np.stack([a for a, _ in lays])
    nb = np.array([n for _, n in lays], dtype=np.int32)
    out = torch.zeros((len(q), 8), dtype=torch.int32, device="cuda")
    rects = torch.zeros((len(q), KSUP_MAX, 4), dtype=torch.float64, device="cuda")
    scr = torch.zeros(len(q) * L.gu_root_scratch_doubles(), dtype=torch.float64, device="cuda")
    _run(L.gu_root_d, _dev(boxes), _dev(nb), _dev(q), len(q), out, rects, scr)
    o, R = out.cpu().numpy(), rects.cpu().numpy()
    assert np.array_equal(o[:, 0], o[:, 1])  # rest_height == rest_height_supports
    n_edge = 0
    for i, (lay, lx, ly, dx, dy) in enumerate(q.tolist()):
        bx, n = lays[lay]
        mh = max([int(b[5]) for b in bx[:n] if lx < b[3] and lx + dx > b[0] and ly < b[4] and ly + dy > b[1]], default=0)
        sup = [(max(lx, int(b[0])), max(ly, int(b[1])), min(lx + dx, int(b[3])), min(ly + dy, int(b[4])))
               for b in bx[:n] if int(b[5]) == mh and mh > 0 and lx < b[3] and lx + dx > b[0] and ly < b[4] and ly + dy > b[1]]
        assert o[i, 1] == mh and o[i, 2] == len(sup) and (mh == 0 or o[i, 7] == len(sup)), i
        assert [tuple(r) for r in R[i, :len(sup)].tolist()] == [tuple(map(float, s)) for s in sup], i
        if mh == 0:
            continue
        X1, Y1 = min(s[0] for s in sup), min(s[1] for s in sup)
        X2, Y2 = max(s[2] for s in sup), max(s[3] for s in sup)
        c2x, c2y = 2 * lx + dx, 2 * ly + dy
        far = c2x < 2 * X1 or c2x > 2 * X2 or c2y < 2 * Y1 or c2y > 2 * Y2
        assert bool(o[i, 4]) == far, i
        pts = rect_points(sup)
        want = oracle_pip(lx + dx * 0.5, ly + dy * 0.5, oracle_hull_shrunk(pts))
        assert o[i, 5] == int(want), i
        if far:
            assert o[i, 5] == 0, i
            n_edge += c2x in (2 * X2 + 1, 2 * X1 - 1) or c2y in (2 * Y2 + 1, 2 * Y1 - 1)
    assert np.sum(o[:, 4]) >= 1000 and n_edge >= 100, (np.sum(o[:, 4]), n_edge)


def gen_layouts_c(seed=12):
    """continuous layouts in 1-unit and 255-wide containers: 6-decimal boxes of one top height over lower ones; query centres placed at
    X2 + margin and X1 - margin (margin = 2e-6 * (1 + W)) +- a few ulps, in x and in y, and at random"""
    rng = np.random.default_rng(seed)
    lays, qs = [], []
    for li in range(60):
        W = 255.0 if li % 2 else 1.0
        margin = 2e-6 * (1.0 + W)
        boxes = []
        for _ in range(int(rng.integers(1, 8))):
            a, c = np.round(rng.uniform(0, W * 0.8, 2), 6)
            w, h = np.round(rng.uniform(W * 0.01, W * 0.2, 2), 6)
            top = float(rng.choice([0.5, 0.5, 0.25]))
            boxes.append((a, c, 0.0, w, h, top))
        arr = np.zeros((NB_MAX, 6))
        arr[:len(boxes)] = boxes
        lay = len(lays)
        lays.append((arr, len(boxes), W, margin))
        for a, c, _, w, h, _ in boxes:
            for x in (w * 0.5, W * 0.05, W * 0.3):
                x = round(x, 6)
                y = round(float(rng.uniform(W * 0.01, W * 0.2)), 6)
                ly = round(c + h * 0.5 - y * 0.5, 6)
                for edge in (a + w + margin, a - margin):
                    for j in range(-3, 4):
                        lx = (edge - x * 0.5) + j * np.spacing(edge)
                        qs.append((lay, lx, ly, x, y))
                        qs.append((lay, ly - c + a, lx - a + c, y, x))  # the same in y (roughly: the layout is not symmetric)
                for _ in range(4):
                    qs.append((lay, float(rng.uniform(a - x, a + w)), float(rng.uniform(c - y, c + h)), x, y))
    return lays, np.array(qs, dtype=np.float64)


@gpu
def test_continuous_quick_reject_on_device():
    torch = _torch()
    lays, q = gen_layouts_c()
    L = _units()
    boxes = np.stack([a for a, *_ in lays])
    nb = np.array([n for _, n, *_ in lays], dtype=np.int32)
    out = torch.zeros((len(q), 5), dtype=torch.float64, device="cuda")
    rects = torch.zeros((len(q), KSUP_MAX, 4), dtype=torch.float64, device="cuda")
    scr = torch.zeros(len(q) * L.gu_root_scratch_doubles(), dtype=torch.float64, device="cuda")
    _run(L.gu_root_c, _dev(boxes), _dev(nb), _dev(q), len(q), out, rects, scr)
    o, R = out.cpu().numpy(), rects.cpu().numpy()
    assert np.array_equal(o[:, 0], o[:, 1])  # rest_height_c == rest_height_pre
    n_far = n_edge = 0
    for i, (lay, lx, ly, x, y) in enumerate(q.tolist()):
        _, n, W, margin = lays[int(lay)]
        k = int(o[i, 2])
        if o[i, 3] < 0:
            continue
        sup = R[i, :k]
        X1, Y1, X2, Y2 = sup[:, 0].min(), sup[:, 1].min(), sup[:, 2].max(), sup[:, 3].max()
        cx, cy = lx + x * 0.5, ly + y * 0.5
        far = cx < X1 - margin or cx > X2 + margin or cy < Y1 - margin or cy > Y2 + margin
        want = oracle_pip(cx, cy, oracle_hull_shrunk(rect_points([tuple(r) for r in sup.tolist()])))
        assert o[i, 3] == int(want), i
        if far:
            assert o[i, 3] == 0, i
            n_far += 1
        for e in (X2 + margin, X1 - margin, Y2 + margin, Y1 - margin):
            n_edge += abs((cx if e in (X2 + margin, X1 - margin) else cy) - e) <= 2 * np.spacing(e)
    assert n_far >= 500 and n_edge >= 100, (n_far, n_edge)


@gpu
def test_fmad_build_differs():
    """the -fmad=true build of the same source must fail the polygon and least-squares comparisons somewhere"""
    Lf = _units(fmad=True)
    lays, polys, shrunk, queries = _polygon_sets()
    m_h, hulls, qpoly, qxy, pip_sh, pip_st, one, rq, rres = _device_polygons(Lf, lays, polys, shrunk, queries)
    poly_diff = sum(len(h) != len(s) or not np.array_equal(np.array(scale_down(h)), s) for h, s in zip(hulls, shrunk))
    want = np.array([oracle_pip(x, y, shrunk[p]) for p, (x, y) in zip(qpoly, qxy)], dtype=np.int32)
    fast = rres[:, 0] == 1
    rwant = np.array([oracle_pip(r[4], r[5], oracle_hull_shrunk(rect_points([tuple(r[:4])]))) for r in rq], dtype=np.int32)
    pip_diff = int(np.sum(pip_sh != want) + np.sum(rres[fast, 1] != rwant[fast]))
    assert pip_diff + poly_diff > 0
    S = gen_lstsq(n_random=400)
    xs = dev_lstsq(S, Lf)
    ls_diff = sum(not np.array_equal(x.view(np.int64), oracle_lstsq(*ls_system(*s[1:5])).view(np.int64)) for s, x in zip(S, xs))
    assert ls_diff > 0
