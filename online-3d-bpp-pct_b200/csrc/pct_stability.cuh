// Stacking-stability approximation of the PCT environment, restated for one CUDA lane per placement.
//
// Reference semantics (paths relative to the reference repo, D: = pct_envs/PctDiscrete0/):
//   Box.calculated_impact / calculated_impact_virtual   D:space.py:73-267 (recursive, dict-ordered loads)
//   Box.calculate_new_com                               D:space.py:51-71
//   ConvexHull / Line2D / point_in_polygen              D:convex_hull.py:4-112
//   Space.scale_down                                    D:space.py:341-345
//   np.linalg.lstsq for >=3 supports                    D:space.py:137-152, 234-250
//
// CUDA restatement (not a translation):
//   * no objects, no recursion: an explicit DFS over the support DAG with a small per-lane frame stack;
//   * supports, contact rectangles, hulls are recomputed from the packed box records in shared memory
//     instead of being stored per box;
//   * the only persistent stability state is the per-env "load edge" pool in HBM
//     (upper box, lower box, load centre xyz, load mass); dict insertion order of the reference's
//     `up_edges` == pool order, because edges are created in placement order and updated in place;
//   * a virtual (feasibility) check never writes: the virtual load of the path member directly above
//     is carried in the frame, and the real edge of that path member is skipped (== the `involved`
//     gating of D:space.py:55-63);
//   * all FP64 arithmetic is one IEEE operation per source operator (file is compiled with
//     -fmad=false); fma() appears only where it reproduces OpenBLAS ddot on 2-vectors;
//   * the step kernel is instruction-fetch bound (ncu: stalled_no_instruction), so this file is written
//     for SMALL CODE: one runtime-flag routine for real and virtual checks, FP64 division / sqrt and the
//     helpers are shared __noinline__ functions, loops are not unrolled.
#pragma once
#include <cstdint>
#include <math.h>
#include <math_constants.h>
#include "pct_kernels.h"

namespace pct {

static __device__ __noinline__ double ddiv(double a, double b) { return a / b; }
// two / three quotients by the same divisor in ONE routine: the independent Newton chains interleave, so the second and third division cost
// issue slots but (almost) no extra latency on the serial chain of a walk (each is the same correctly rounded a / d as ddiv)
static __device__ __noinline__ void ddiv2(double a, double b, double d, double &qa, double &qb) { qa = a / d; qb = b / d; }
static __device__ __noinline__ void ddiv3(double a, double b, double c, double d, double &qa, double &qb, double &qc) { qa = a / d; qb = b / d; qc = c / d; }
static __device__ __noinline__ double dsqrt(double a) { return sqrt(a); }
__device__ __forceinline__ double dot2(double u0, double u1, double v0, double v1) { return fma(u1, v1, u0 * v0); }

__device__ __forceinline__ double slope_of(double ax, double ay, double bx, double by) {
    if (bx != ax) return ddiv(by - ay, bx - ax);
    return (by - ay) * CUDART_INF;  // 0*inf = nan like the reference (convex_hull.py:14)
}
__device__ __forceinline__ int orient_of(double s1, double s2) {
    if (fabs(s1) == CUDART_INF && fabs(s2) == CUDART_INF) return 0;
    double d = s2 - s1;
    if (d > 0) return -1;
    if (d == 0) return 0;
    return 1;
}
// Line2D(a,b).orientation(Line2D(b,c)) (convex_hull.py:4-32) with a division-saving pre-filter.
// The verdict only depends on the ORDER of the two correctly rounded slopes.  Single-precision estimates of
// both slopes (relative error < 1e-6) that differ by more than 1e-4 relative prove that the exact quotients
// differ by far more than one rounding error, hence that the rounded doubles compare the same way; only
// near-ties (collinear contact points) and vertical segments fall through to the exact FP64 divisions.
__device__ __forceinline__ int orient3(double ax, double ay, double bx, double by, double cx, double cy) {
    const double d1x = bx - ax, d1y = by - ay, d2x = cx - bx, d2y = cy - by;
    if (d1x != 0 && d2x != 0) {
        // three corners on one horizontal line (every contact rectangle contributes two such pairs): both slopes are (+-0) / dx = +-0, their
        // difference is 0 -> collinear (0), without the two IEEE divisions the float estimate below would fall through to
        if (d1y == 0 && d2y == 0) return 0;
        const float f1 = __fdividef((float)d1y, (float)d1x), f2 = __fdividef((float)d2y, (float)d2x);
        const float gap = f2 - f1, tol = 1e-4f * (fabsf(f1) + fabsf(f2));
        if (fabsf(gap) > tol && fabsf(f1) < 1e30f && fabsf(f2) < 1e30f) return gap > 0 ? -1 : 1;
    }
    return orient_of(slope_of(ax, ay, bx, by), slope_of(bx, by, cx, cy));
}

// ConvexHull (convex_hull.py:39-95) on n points already perturbed (x += y*1e-6).
// px/py are sorted IN PLACE (stable insertion sort by x, sorted(key=x[0]) :34-37); the hull (lower chain minus its
// last point, then upper chain minus its last point, :89-92) is written as coordinates to hx/hy (capacity 2n).
// The two topmost chain points live in registers, so the orientation test of the scan needs no reloads.
static __device__ __noinline__ int hull_coords(double *px, double *py, int n, double *hx, double *hy) {
#pragma unroll 1
    for (int i = 1; i < n; i++) {
        const double kx = px[i], ky = py[i];
        int j = i - 1;
#pragma unroll 1
        while (j >= 0 && px[j] > kx) { px[j + 1] = px[j]; py[j + 1] = py[j]; j--; }
        px[j + 1] = kx; py[j + 1] = ky;
    }
    int m = 0;
#pragma unroll 1
    for (int pass = 0; pass < 2; pass++) {
        double *HX = hx + m, *HY = hy + m;  // this chain is built in place behind the previous one
        int nh = 0;
        double tx = 0, ty = 0, ux = 0, uy = 0, fx = 0, fy = 0;  // top, second, first
#pragma unroll 1
        for (int k = 0; k < n; k++) {
            const int p = pass == 0 ? k : n - 1 - k;
            const double qx = px[p], qy = py[p];
#pragma unroll 1
            while (nh >= 2) {
                if (orient3(ux, uy, tx, ty, qx, qy) == -1) break;
                nh--;  // pop
                tx = ux; ty = uy;
                if (nh >= 2) { ux = HX[nh - 2]; uy = HY[nh - 2]; }
                if (fx == tx && fy == ty) break;  // lowerHull[0] == lowerHull[-1] (:58-59), list equality
            }
            HX[nh] = qx; HY[nh] = qy;
            if (nh == 0) { fx = qx; fy = qy; }
            ux = tx; uy = ty; tx = qx; ty = qy;
            nh++;
        }
        m += nh - 1;  // drop the last point of the chain
    }
    return m;
}

// convex_hull.py:108 — is the edge's crossing with the horizontal ray strictly left of the point?
//   coords[i][0] + (lon - coords[i][1]) / (coords[j][1] - coords[i][1]) * (coords[j][0] - coords[i][0]) < lat
// Float estimate first (error < 1e-5 of the operand scale); the exact FP64 expression only near the threshold.
__device__ __forceinline__ bool cross_left(double ix, double iy, double jx, double jy, double lat, double lon) {
    const float xf = (float)ix + __fdividef((float)(lon - iy), (float)(jy - iy)) * (float)(jx - ix);
    const float scale = fabsf((float)ix) + fabsf((float)(jx - ix)) + fabsf((float)lat);
    const float gap = xf - (float)lat;
    if (fabsf(gap) > 1e-4f * scale + 1e-30f) return gap < 0;
    const double t = ddiv(lon - iy, jy - iy);
    const double u = t * (jx - ix);
    return ix + u < lat;
}

// scale_down (D:space.py:341-345) + point_in_polygen (convex_hull.py:97-112) fused: the shrunk polygon is
// never stored, its vertices are produced on the fly from the hull coordinates.
static __device__ __noinline__ bool pip_shrunk(const double *hx, const double *hy, int stride, int m, double lat, double lon) {
    double sx = 0, sy = 0;
#pragma unroll 1
    for (int i = 0; i < m; i++) { sx += hx[i * stride]; sy += hy[i * stride]; }
    double cx, cy;
    ddiv2(sx, sy, (double)m, cx, cy);
    double jx, jy;
    {
        double v = hx[(m - 1) * stride], d = v - cx;
        jx = v - d * 0.1;
        v = hy[(m - 1) * stride]; d = v - cy;
        jy = v - d * 0.1;
    }
    bool odd = false;
#pragma unroll 1
    for (int i = 0; i < m; i++) {
        double v = hx[i * stride], d = v - cx;
        const double ix = v - d * 0.1;
        v = hy[i * stride]; d = v - cy;
        const double iy = v - d * 0.1;
        const double a0 = ix - lat, a1 = iy - lon;
        const double b0 = lat - jx, b1 = lon - jy;
        const double m1 = a0 * b1, m2 = a1 * b0;
        if (m1 - m2 == 0) return false;
        if ((iy < lon && jy >= lon) || (jy < lon && iy >= lon)) {
            if (cross_left(ix, iy, jx, jy, lat, lon)) odd = !odd;
        }
        jx = ix; jy = iy;
    }
    return odd;
}

// The same test on a polygon that was shrunk when it was stored (store_shrunk): the placed boxes' bottom_whole_contact_area is the
// scaled-down hull in the reference too (D:space.py:378-379), so a visit of a placed box only runs the edge loop.
static __device__ __noinline__ bool pip_stored(const double *xy, int m, double lat, double lon) {
    double jx = xy[2 * (m - 1)], jy = xy[2 * (m - 1) + 1];
    bool odd = false;
#pragma unroll 1
    for (int i = 0; i < m; i++) {
        const double ix = xy[2 * i], iy = xy[2 * i + 1];
        const double a0 = ix - lat, a1 = iy - lon;
        const double b0 = lat - jx, b1 = lon - jy;
        const double m1 = a0 * b1, m2 = a1 * b0;
        if (m1 - m2 == 0) return false;
        if ((iy < lon && jy >= lon) || (jy < lon && iy >= lon)) {
            if (cross_left(ix, iy, jx, jy, lat, lon)) odd = !odd;
        }
        jx = ix; jy = iy;
    }
    return odd;
}

// two supports: direction of the line through the two contact-rectangle centres divided by its squared length (D:space.py:383-392);
// a function of the placed geometry only, so it is stored behind the polygon of a placed box with two supports.
__device__ __forceinline__ void split2_dir(const double *px, const double *py, double &lx, double &ly) {
    lx = px[0] - px[1]; ly = py[0] - py[1];
    const double len = dsqrt(fma(ly, ly, lx * lx));
    const double len2 = len * len;
    ddiv2(lx, ly, len2, lx, ly);
}

// Minimum-norm least squares (np.linalg.lstsq restatement: streaming Givens QR + one-sided Jacobi SVD,
// identical operation order to oracle/pct_oracle_common.h po_ls_*).  ld = leading dimension of R and V.
struct LsWork { double *R, *V, *y, *row, *x; int ld; };

static __device__ __noinline__ void ls_add_row(const LsWork &w, int k, double rhs) {
#pragma unroll 1
    for (int i = 0; i < k; i++) {
        const double b = w.row[i];
        if (b == 0) continue;
        const double a = w.R[i * w.ld + i];
        const double r = dsqrt(a * a + b * b);
        const double c = ddiv(a, r), sn = ddiv(b, r);
#pragma unroll 1
        for (int j = i; j < k; j++) {
            const double rij = w.R[i * w.ld + j], vj = w.row[j];
            w.R[i * w.ld + j] = c * rij + sn * vj;
            w.row[j] = c * vj - sn * rij;
        }
        const double yi = w.y[i];
        w.y[i] = c * yi + sn * rhs;
        rhs = c * rhs - sn * yi;
    }
}
static __device__ __noinline__ void ls_solve(const LsWork &w, int k, int rows) {
    double *G = w.R, *V = w.V;
    const int ld = w.ld;
    {   // full column rank and well conditioned (the usual case): the least-squares solution is R x = y
        double rmin = fabs(G[0]), rmax = rmin;
#pragma unroll 1
        for (int i = 1; i < k; i++) { const double a = fabs(G[i * ld + i]); rmin = fmin(rmin, a); rmax = fmax(rmax, a); }
        if (rmin * 1e4 > rmax) {
#pragma unroll 1
            for (int i = k - 1; i >= 0; i--) {
                double acc = w.y[i];
#pragma unroll 1
                for (int j = i + 1; j < k; j++) acc -= G[i * ld + j] * w.x[j];
                w.x[i] = ddiv(acc, G[i * ld + i]);
            }
            return;
        }
    }
#pragma unroll 1
    for (int i = 0; i < k; i++)
#pragma unroll 1
        for (int j = 0; j < k; j++) V[i * ld + j] = (i == j) ? 1.0 : 0.0;
#pragma unroll 1
    for (int sweep = 0; sweep < 60; sweep++) {
        bool rotated = false;
#pragma unroll 1
        for (int p = 0; p < k - 1; p++)
#pragma unroll 1
            for (int q = p + 1; q < k; q++) {
                double alpha = 0, beta = 0, gamma = 0;
#pragma unroll 1
                for (int i = 0; i < k; i++) {
                    const double gp = G[i * ld + p], gq = G[i * ld + q];
                    alpha += gp * gp;
                    beta += gq * gq;
                    gamma += gp * gq;
                }
                if (gamma == 0 || fabs(gamma) <= 1e-15 * dsqrt(alpha * beta)) continue;
                rotated = true;
                const double zeta = ddiv(beta - alpha, 2.0 * gamma);
                const double t = ddiv(zeta >= 0 ? 1.0 : -1.0, fabs(zeta) + dsqrt(1.0 + zeta * zeta));
                const double c = ddiv(1.0, dsqrt(1.0 + t * t)), sn = c * t;
#pragma unroll 1
                for (int i = 0; i < k; i++) {
                    const double gp = G[i * ld + p], gq = G[i * ld + q];
                    G[i * ld + p] = c * gp - sn * gq;
                    G[i * ld + q] = sn * gp + c * gq;
                    const double vp = V[i * ld + p], vq = V[i * ld + q];
                    V[i * ld + p] = c * vp - sn * vq;
                    V[i * ld + q] = sn * vp + c * vq;
                }
            }
        if (!rotated) break;
    }
    double smax = 0;  // singular values (kept in w.row)
#pragma unroll 1
    for (int j = 0; j < k; j++) {
        double a = 0;
#pragma unroll 1
        for (int i = 0; i < k; i++) a += G[i * ld + j] * G[i * ld + j];
        const double s = dsqrt(a);
        w.row[j] = s;
        if (s > smax) smax = s;
    }
    const int M = rows > k ? rows : k;
    const double cutoff = 2.220446049250313e-16 * (double)M * smax;
#pragma unroll 1
    for (int i = 0; i < k; i++) w.x[i] = 0;
#pragma unroll 1
    for (int j = 0; j < k; j++) {
        const double sg = w.row[j];
        if (!(sg > cutoff)) continue;
        double uy = 0;
#pragma unroll 1
        for (int i = 0; i < k; i++) uy += G[i * ld + j] * w.y[i];
        const double coef = ddiv(uy, sg * sg);
#pragma unroll 1
        for (int i = 0; i < k; i++) w.x[i] += V[i * ld + j] * coef;
    }
}

// lstsq load split for k >= 3 supports without a direct edge (D:space.py:134-152 / 231-250):
// c2x/c2y = contact-rectangle centres, (cx,cy) = stack COM; writes the k assignment ratios to w.x
static __device__ __noinline__ void lstsq_ratios(const LsWork &w, int k, const double *c2x, const double *c2y, double cx, double cy) {
#pragma unroll 1
    for (int i = 0; i < k; i++) {
        w.y[i] = 0;
#pragma unroll 1
        for (int j = 0; j < k; j++) w.R[i * w.ld + j] = 0;
    }
    int rows = 0;
#pragma unroll 1
    for (int a = 0; a < k - 1; a++)
#pragma unroll 1
        for (int b = a + 1; b < k; b++) {
#pragma unroll 1
            for (int t = 0; t < k; t++) w.row[t] = 0;
            const double lx = c2x[a] - c2x[b], ly = c2y[a] - c2y[b];
            const double molecular = dot2(cx - c2x[a], cy - c2y[a], lx, ly);
            if (molecular != 0) {
                const double r = ddiv(fabs(dot2(cx - c2x[b], cy - c2y[b], lx, ly)), molecular);
                w.row[a] = 1;
                w.row[b] = -r;
            }
            ls_add_row(w, k, 0.0);
            rows++;
        }
#pragma unroll 1
    for (int t = 0; t < k; t++) w.row[t] = 1;
    ls_add_row(w, k, 1.0);
    rows++;
    ls_solve(w, k, rows);
}

// ---------------------------------------------------------------------------------------------
// Geometry policy G (per lane) provides:
//   typedef Node            footprint corner + dims of a box (ints for discrete, doubles for continuous) + mass
//   int  n_boxes() const
//   void node_box(int id, Node &out) const                       (real box id)
//   void centre(const Node&, double &cx,&cy,&cz) const            (D:space.py:35)
//   bool support(const Node &node, int t, double r[4]) const      (is box t a support? contact rect x1,y1,x2,y2)
//   bool strictly_inside(cx, cy, const double r[4]) const         (direct-edge test)
// ---------------------------------------------------------------------------------------------
struct StabFrame {
    Stack4 st;        // the node's stack for this visit
    uint8_t node;     // real box index, or NODE_NEW
    uint8_t base, k, i;
    uint8_t whole;    // 1: whole stack to the single support; 2: direct edge (others zero); 0: (c2d_i, st.cz) split
    uint8_t eoff;     // pool position of the node's first edge (placed boxes)
};
constexpr int NODE_NEW = 255;

// append the edge (new box -> lower) to the pool and to lower's incoming list
__device__ __forceinline__ bool pool_append(EdgePool &pool, int lower) {
    if (pool.n >= EDGE_MAX) return false;
    const int pos = pool.n++;
    pool.lower[pos] = (uint8_t)lower;
    pool.next[pos] = EDGE_NIL;
    if (pool.first_in[lower] == EDGE_NIL) pool.first_in[lower] = (uint8_t)pos;
    else pool.next[pool.last_in[lower]] = (uint8_t)pos;
    pool.last_in[lower] = (uint8_t)pos;
    return true;
}

// Single support (58 % of all visits): the "hull" of the 4 corners of one contact rectangle.
// With P0=(x1,y1) P1=(x1,y2) P2=(x2,y1) P3=(x2,y2) perturbed by x += y*1e-6 (convex_hull.py:43) and
// P0.x < P1.x < P2.x < P3.x (checked by the caller), ConvexHull's chain scans are fully determined:
//   lower: [P0,P1] -> P2: slope(P0,P1) > 0 > slope(P1,P2) => pop P1 (then first==last => break), push P2;
//          P3: slope(P0,P2) = 0 < slope(P2,P3) => keep                     => [P0,P2,P3] -> drop last
//   upper: [P3,P2] -> P1: slope(P3,P2) > 0 > slope(P2,P1) => pop P2, push P1; P0: slope(P3,P1) = -0 < slope(P1,P0)
//                                                                           => [P3,P1,P0] -> drop last
// so the polygon is [P0,P2,P3,P1]; scale_down + point_in_polygen run on registers, same operation order as
// hull_indices + pip_shrunk.
// one polygon edge (j -> i) of point_in_polygen: returns 2 when the point is collinear with the edge's line (-> False),
// else 1 / 0 for "the ray crossing toggles" / "does not toggle"
__device__ __forceinline__ int pip_edge(double ix, double iy, double jx, double jy, double lat, double lon) {
    const double a0 = ix - lat, a1 = iy - lon;
    const double b0 = lat - jx, b1 = lon - jy;
    const double m1 = a0 * b1, m2 = a1 * b0;
    if (m1 - m2 == 0) return 2;
    if ((iy < lon && jy >= lon) || (jy < lon && iy >= lon)) return cross_left(ix, iy, jx, jy, lat, lon) ? 1 : 0;
    return 0;
}
static __device__ __noinline__ bool pip_rect(double x1, double y1, double x2, double y2, double t1, double t2, double lat, double lon) {
    // t1 = y1*1e-6, t2 = y2*1e-6 ; hull order P0,P2,P3,P1 = (x1+t1,y1) (x2+t1,y1) (x2+t2,y2) (x1+t2,y2)
    const double h0 = x1 + t1, h1 = x2 + t1, h2 = x2 + t2, h3 = x1 + t2;
    const double sx = ((h0 + h1) + h2) + h3, sy = ((y1 + y1) + y2) + y2;
    const double cx = sx * 0.25, cy = sy * 0.25;  // mean of 4 (exact power-of-two division)
    double d;
    d = h0 - cx; const double v0x = h0 - d * 0.1;
    d = h1 - cx; const double v1x = h1 - d * 0.1;
    d = h2 - cx; const double v2x = h2 - d * 0.1;
    d = h3 - cx; const double v3x = h3 - d * 0.1;
    d = y1 - cy; const double vlo = y1 - d * 0.1;  // y of P0, P2
    d = y2 - cy; const double vhi = y2 - d * 0.1;  // y of P3, P1
    // edges in polygon order, j = previous vertex: (P1->P0) (P0->P2) (P2->P3) (P3->P1)
    int r = pip_edge(v0x, vlo, v3x, vhi, lat, lon);
    if (r == 2) return false;
    bool odd = r == 1;
    r = pip_edge(v1x, vlo, v0x, vlo, lat, lon);
    if (r == 2) return false;
    odd ^= (r == 1);
    r = pip_edge(v2x, vhi, v1x, vlo, lat, lon);
    if (r == 2) return false;
    odd ^= (r == 1);
    r = pip_edge(v3x, vhi, v2x, vhi, lat, lon);
    if (r == 2) return false;
    odd ^= (r == 1);
    return odd;
}

// ---- ALIAS variant helpers (the default since round 2; see EdgePoolA) ----------------------------------------------------------------------
// calculate_new_com of a placed box under the reference's object semantics: entries that ARE the upper box's Stack object are read
// through that box's current field, the others are the stored snapshots.  Same operation order as the lazy sum at the end of the DFS loop.
template <class G>
static __device__ __noinline__ void alias_recompute(const G &g, EdgePoolA &pa, int box) {
    typename G::Node sb;
    g.node_box(box, sb);
    double cx, cy, cz, mm = sb.mass;
    g.centre(sb, cx, cy, cz);
    cx *= mm; cy *= mm; cz *= mm;
#pragma unroll 1
    for (int q = pa.first_in[box]; q != EDGE_NIL; q = pa.next[q]) {
        const bool al = (pa.e_alias[q >> 5] >> (q & 31)) & 1u;
        const Stack4 e = al ? pa.box_st[pa.e_upper[q]] : pa.load(q);
        cx += e.cx * e.m; cy += e.cy * e.m; cz += e.cz * e.m;
        mm += e.m;
    }
    Stack4 &d = pa.box_st[box];
    ddiv3(cx, cy, cz, mm, d.cx, d.cy, d.cz); d.m = mm;
}
// SET_EDGE bookkeeping of edge q (upper box `upper`, supporting box `lower`): kind of the entry, then the support's eager recompute
template <class G>
static __device__ __forceinline__ void alias_set_edge(const G &g, EdgePoolA &pa, int q, int upper, int lower, bool is_object) {
    uint32_t &w = pa.e_alias[q >> 5];
    w = is_object ? (w | (1u << (q & 31))) : (w & ~(1u << (q & 31)));
    pa.e_upper[q] = (uint8_t)upper;
    alias_recompute(g, pa, lower);
}

// After a real descent that FAILED midway the object-type entries of boxes whose stack was recomputed but not propagated still read the new
// stack in the reference (the terminal observation's virtual checks see it); the stored snapshots are brought in line here, so the
// read-only checks (stability_check<false>, which only knows snapshots) need no variant.  After a completed descent both are equal already.
static __device__ __noinline__ void alias_sync_loads(EdgePoolA &pa) {
#pragma unroll 1
    for (int q = 0; q < pa.n; q++)
        if ((pa.e_alias[q >> 5] >> (q & 31)) & 1u) pa.load(q) = pa.box_st[pa.e_upper[q]];
}

// The DFS keeps the CURRENT node in registers; frames are pushed to the lane-local stack only for nodes with
// >= 2 supports, and descending into the last (or only) support is a tail call (nothing is left to do in the
// parent once its last child returns True).
#ifdef PCT_PHASE_TIMERS
__device__ long long *g_prof_dummy;
#endif
// Working arrays of one descent.  A lane-local instance lives on the local-memory stack; the apply kernel, whose descent runs on ONE lane per warp,
// hands in a per-warp instance in shared memory instead (aliased onto its EMS scratch, which is idle during the descent): on the stack every hot word
// of that single lane costs a whole 128-byte L1 line.
struct StabScratch {
    StabFrame fr[STAB_DEPTH];
    double sup_m[STAB_SUP_POOL];
    double rect[KSUP_SMALL][4], px[4 * KSUP_SMALL], py[4 * KSUP_SMALL], hx[8 * KSUP_SMALL], hy[8 * KSUP_SMALL];
    double R[KSUP_SMALL * KSUP_SMALL], V[KSUP_SMALL * KSUP_SMALL], y[KSUP_SMALL], row[KSUP_SMALL], x[KSUP_SMALL];
    uint8_t sup_id[STAB_SUP_POOL];
};
template <bool REAL, class G, bool ALIAS = false>
static __device__ __noinline__ int stability_check(const G &g, const typename G::Node &root, EdgePool &pool, BigScratch *big, int *lock,
                                            const int new_id, int &flags, long long *g_prof_out = nullptr, StabScratch *scr = nullptr) {
    typedef typename G::Node Node;
    constexpr bool real = REAL;  // REAL: load-propagating update of a committed placement; else read-only feasibility check
    constexpr bool alias = REAL && ALIAS;  // object semantics of the reference's load entries; `pool` is an EdgePoolA then
    StabScratch local_scr;  // untouched (no cache footprint) when the caller provides one
    StabScratch &S = scr ? *scr : local_scr;
    StabFrame *fr = S.fr;
    uint8_t *sup_id = S.sup_id;
    double *sup_m = S.sup_m;
    const int root_id = real ? new_id : NODE_NEW;
    int depth = 0;            // number of pushed frames
    int node = root_id, base = 0;
    Stack4 st;
    g.centre(root, st.cx, st.cy, st.cz);
    st.m = root.mass;
    if constexpr (alias) static_cast<EdgePoolA &>(pool).box_st[new_id] = st;  // Box.__init__: thisStack = Stack(centre, mass)

#ifdef PCT_PHASE_TIMERS
    long long sec_[6] = {0, 0, 0, 0, 0, 0}, tq_ = clock64();
#define SEC(i) do { long long n_ = clock64(); sec_[i] += n_ - tq_; tq_ = n_; } while (0)
#define SEC_OUT() do { if (g_prof_out) for (int i_ = 0; i_ < 6; i_++) g_prof_out[i_] = sec_[i_]; } while (0)
    flags += 1 << 16;  // debug: visits in bits 16..23, lstsq solves in bits 24..31 (masked off by the caller)
#define DBG_VISIT() flags += 1 << 16
#define DBG_LS() flags += 1 << 24
#else
#define DBG_VISIT()
#define DBG_LS()
#define SEC(i)
#define SEC_OUT()
#endif
#pragma unroll 1
    for (;;) {
        // ================= ENTER(node, st) =================
        Node cur;
        if (node != root_id) g.node_box(node, cur);
        else cur = root;
        int k = 0, sid0 = 0;
        double r0[4], r[4];
        const int eoff = (node == root_id) ? pool.n : (int)pool.off[node];  // pool position of this node's first edge
        if (node == root_id) {
            // the box being placed / tested: supports are found by scanning every placed box (D:space.py:360-376)
            const int limit = g.n_boxes();
#pragma unroll 1
            for (int t = 0; t < limit; t++) {
                if (!g.support(cur, t, r)) continue;
                if (k >= STAB_SUP_POOL || k >= KSUP_MAX) { flags |= PCT_FLAG_SUPPORT_OVERFLOW; return 0; }
                if (k == 0) { sid0 = t; r0[0] = r[0]; r0[1] = r[1]; r0[2] = r[2]; r0[3] = r[3]; }
                sup_id[base + k] = (uint8_t)t;
                k++;
            }
        } else {
            // a placed box: its supports were recorded (in the same scan order) when it was placed
            k = (int)pool.off[node + 1] - eoff;
            if (base + k > STAB_SUP_POOL) { flags |= PCT_FLAG_SUPPORT_OVERFLOW; return 0; }
#pragma unroll 1
            for (int j = 0; j < k; j++) sup_id[base + j] = pool.lower[eoff + j];
            if (k >= 1) { sid0 = sup_id[base]; g.support(cur, sid0, r0); }
        }
        SEC(0);
        int child = -1;          // >= 0: tail-descend into this support with load (vx,vy,st.cz,vm)
        int skip = EDGE_NIL;     // pool position of the real edge parent->child (replaced by the virtual load)
        double vx = st.cx, vy = st.cy, vm = st.m;
        if (k == 1) {
            const double t1 = r0[1] * 1e-6, t2 = r0[3] * 1e-6;
            const bool fast = (r0[0] + t1 < r0[0] + t2) && (r0[0] + t2 < r0[2] + t1) && (r0[2] + t1 < r0[2] + t2);
            bool ok;
            if (fast) ok = pip_rect(r0[0], r0[1], r0[2], r0[3], t1, t2, st.cx, st.cy);
            else {
                double px[4] = {r0[0] + t1, r0[0] + t2, r0[2] + t1, r0[2] + t2}, py[4] = {r0[1], r0[3], r0[1], r0[3]};
                double hx[8], hy[8];
                const int m = hull_coords(px, py, 4, hx, hy);
                ok = pip_shrunk(hx, hy, 1, m, st.cx, st.cy);
            }
            SEC(1);
            if (!ok) { SEC_OUT(); return 0; }
            if (real) {
                if (node == root_id && !pool_append(pool, sid0)) { flags |= PCT_FLAG_EDGE_OVERFLOW; return 0; }
                pool.load(eoff) = st;
                if constexpr (alias) alias_set_edge(g, static_cast<EdgePoolA &>(pool), eoff, node, sid0, true);  // up_edges[self] = self.thisStack
            }
            child = sid0;  // whole stack goes to the single support
            skip = (node == root_id) ? EDGE_NIL : eoff;
        } else if (k >= 2) {
            // ---------- general case: hull over all contact-rectangle corners ----------
            const bool small = k <= KSUP_SMALL;
            double (*rect)[4] = S.rect;
            double *px = S.px, *py = S.py, *hx = S.hx, *hy = S.hy;
            if (!small) {  // rare: serialise the lanes of this env on the per-env HBM scratch
                while (atomicCAS(lock, 0, 1) != 0) { }
                __threadfence_block();
                rect = big->rect; px = big->px; py = big->py; hx = big->hx; hy = big->hy;
            }
#pragma unroll 1
            for (int s = 0; s < k; s++) g.support(cur, sup_id[base + s], rect[s]);
            bool ok;
            const double *split = nullptr;  // k == 2, placed box: the stored split direction
            const int pv = node == root_id ? 0 : (int)pool.poly_off[node], pm = node == root_id ? 0 : (int)pool.poly_off[node + 1] - pv;
            if (pm > 0 && (pv + pm <= POLY_STAGE || pv >= POLY_STAGE)) {
                // a placed box: its support polygon was stored when it was placed
                const double *xy = pool.poly_at(pv);
                ok = pip_stored(xy, pm - (k == 2), st.cx, st.cy);
                if (k == 2) split = xy + 2 * (pm - 1);
            } else {
                // combine_contact_points order: (x1,y1) (x1,y2) (x2,y1) (x2,y2); perturb x += y*1e-6 (convex_hull.py:43)
#pragma unroll 1
                for (int s = 0; s < k; s++) {
                    const double x1 = rect[s][0], y1 = rect[s][1], x2 = rect[s][2], y2 = rect[s][3];
                    const double t1 = y1 * 1e-6, t2 = y2 * 1e-6;
                    px[4 * s + 0] = x1 + t1; py[4 * s + 0] = y1;
                    px[4 * s + 1] = x1 + t2; py[4 * s + 1] = y2;
                    px[4 * s + 2] = x2 + t1; py[4 * s + 2] = y1;
                    px[4 * s + 3] = x2 + t2; py[4 * s + 3] = y2;
                }
                const int m = hull_coords(px, py, 4 * k, hx, hy);
                ok = pip_shrunk(hx, hy, 1, m, st.cx, st.cy);
                if (real && ok && node == root_id && pool.n_poly + m + (k == 2) <= POLY_MAX) {
                    // the box being placed: remember its shrunk polygon (bottom_whole_contact_area, D:space.py:378-379; same operations as
                    // pip_shrunk) and, with two supports, the split direction behind it
                    double sx = 0, sy = 0;
#pragma unroll 1
                    for (int i = 0; i < m; i++) { sx += hx[i]; sy += hy[i]; }
                    double pcx, pcy;
                    ddiv2(sx, sy, (double)m, pcx, pcy);
#pragma unroll 1
                    for (int i = 0; i < m; i++) {
                        double *v = pool.poly_at(pool.n_poly + i);
                        double d = hx[i] - pcx;
                        v[0] = hx[i] - d * 0.1;
                        d = hy[i] - pcy;
                        v[1] = hy[i] - d * 0.1;
                    }
                    pool.n_poly += m;
                    if (k == 2) {
                        double cx2[2] = {(rect[0][0] + rect[0][2]) * 0.5, (rect[1][0] + rect[1][2]) * 0.5};
                        double cy2[2] = {(rect[0][1] + rect[0][3]) * 0.5, (rect[1][1] + rect[1][3]) * 0.5};
                        double *v = pool.poly_at(pool.n_poly);
                        split2_dir(cx2, cy2, v[0], v[1]);
                        pool.n_poly += 1;
                    }
                }
            }
            SEC(1);
            int whole = 2;
            if (ok) {
                // --- distribution ---
                int direct = -1;
#pragma unroll 1
                for (int s = 0; s < k; s++)
                    if (g.strictly_inside(st.cx, st.cy, rect[s])) { direct = s; break; }
                if (direct >= 0) {
#pragma unroll 1
                    for (int s = 0; s < k; s++) sup_m[base + s] = (s == direct) ? st.m : 0.0;
                } else {
                    whole = 0;
                    // contact-rectangle centres (centre2D, D:space.py:371) reuse px/py (hull no longer needed)
#pragma unroll 1
                    for (int s = 0; s < k; s++) {
                        px[s] = (rect[s][0] + rect[s][2]) * 0.5;  // (x1 + x2) / 2, exact
                        py[s] = (rect[s][1] + rect[s][3]) * 0.5;
                    }
                    if (k == 2) {
                        double lx, ly;
                        if (split) { lx = split[0]; ly = split[1]; }
                        else split2_dir(px, py, lx, ly);
                        sup_m[base + 0] = st.m * fabs(dot2(st.cx - px[1], st.cy - py[1], lx, ly));
                        sup_m[base + 1] = st.m * fabs(dot2(st.cx - px[0], st.cy - py[0], lx, ly));
                    } else {
                        LsWork w;
                        w.R = small ? S.R : big->R; w.V = small ? S.V : big->V; w.y = small ? S.y : big->y;
                        w.row = small ? S.row : big->row; w.x = small ? S.x : big->x; w.ld = small ? KSUP_SMALL : KSUP_MAX;
                        DBG_LS();
                        lstsq_ratios(w, k, px, py, st.cx, st.cy);
#pragma unroll 1
                        for (int s = 0; s < k; s++) sup_m[base + s] = st.m * w.x[s];
                    }
                }
                SEC(2);
                if (real) {
                    // persist the loads: up_edges[self] = Stack(...) for every support, in support order
#pragma unroll 1
                    for (int s = 0; s < k; s++) {
                        Stack4 e = st;
                        if (!whole) { e.cx = px[s]; e.cy = py[s]; }
                        e.m = sup_m[base + s];
                        if (node == root_id && !pool_append(pool, sup_id[base + s])) { flags |= PCT_FLAG_EDGE_OVERFLOW; ok = false; break; }
                        pool.load(eoff + s) = e;
                        // the direct support receives the object itself (space.py:98), every other entry is a fresh Stack(...)
                        if constexpr (alias) alias_set_edge(g, static_cast<EdgePoolA &>(pool), eoff + s, node, sup_id[base + s], whole == 2 && s == direct);
                    }
                }
            }
            if (!small) { __threadfence_block(); atomicExch(lock, 0); }
            SEC(3);
            if (!ok) { SEC_OUT(); return 0; }
            if (depth >= STAB_DEPTH) { flags |= PCT_FLAG_SUPPORT_OVERFLOW; return 0; }
            StabFrame &f = fr[depth++];
            f.st = st; f.node = (uint8_t)node; f.base = (uint8_t)base; f.k = (uint8_t)k; f.i = 0; f.whole = (uint8_t)whole;
            f.eoff = (uint8_t)eoff;
        }
        // ================= pick the next node to enter =================
        int parent = node;
        if (child < 0) {
            // k == 0 (return True) or a frame was just pushed: continue with the top frame's next child
            for (;;) {
                if (depth == 0) { SEC_OUT(); return 1; }
                StabFrame &f = fr[depth - 1];
                if (f.i == f.k) { depth--; continue; }  // all supports passed -> True
                const int s = f.i++;
                child = sup_id[f.base + s];
                parent = f.node;
                skip = (parent == root_id) ? EDGE_NIL : (int)f.eoff + s;
                st = f.st;
                vm = sup_m[f.base + s];
                vx = st.cx; vy = st.cy;
                if (!f.whole) {  // load sits at the centre of this support's contact rectangle with the parent
                    Node par;
                    if (parent != root_id) g.node_box(parent, par);
                    else par = root;
                    g.support(par, child, r);
                    vx = (r[0] + r[2]) * 0.5; vy = (r[1] + r[3]) * 0.5;
                }
                base = f.base + f.k;
                if (s == f.k - 1) { depth--; base = f.base; }  // tail call: the parent frame is finished
                break;
            }
        }
        if constexpr (alias) {  // the support's stack was recomputed eagerly at its last SET_EDGE: calculated_impact reads the field
            st = static_cast<EdgePoolA &>(pool).box_st[child];
            node = child;
            DBG_VISIT();
            continue;
        }
        // ---- calculate_new_com of `child` (D:space.py:51-71) under the load (vx, vy, st.cz, vm) of `parent` ----
        Node sb;
        g.node_box(child, sb);
        double ccx, ccy, ccz, mm = sb.mass;
        g.centre(sb, ccx, ccy, ccz);
        ccx *= mm; ccy *= mm; ccz *= mm;
#pragma unroll 1
        for (int q = pool.first_in[child]; q != EDGE_NIL; q = pool.next[q]) {
            if (!real && q == skip) continue;  // `involved` path member: its real load is replaced by the virtual one
            const Stack4 e = pool.load(q);
            ccx += e.cx * e.m; ccy += e.cy * e.m; ccz += e.cz * e.m;
            mm += e.m;
        }
        if (!real && vm != 0.0) {  // zero-mass virtual loads add +0.0 to every sum: skipped (exact)
            ccx += vx * vm; ccy += vy * vm; ccz += st.cz * vm;
            mm += vm;
        }
        ddiv3(ccx, ccy, ccz, mm, st.cx, st.cy, st.cz); st.m = mm;
        node = child;
        DBG_VISIT();
        SEC(4);
    }
}

// =====================================================================================================================
// stab_virtual: the read-only feasibility check (calculated_impact_virtual, D:space.py:166-267) for a WARP of placements,
// one lane per placement, restructured for SIMT convergence (round 2).
//
// In round 1's thread-per-candidate kernel the DFS of stability_check<false> held most of
// the kernel's warp instructions at 2-5 active lanes — every lane walks its own support DAG, and a visit is either LIGHT (no or
// one support: a rectangle test in registers) or HEAVY (>= 2 supports: hull / stored polygon, load split, frame push), 10x the
// instructions; with both kinds present in nearly every round a warp pays light + heavy per round.  Here the walk is a per-lane state machine with
// two warp-synchronous phases per round: lanes RUN AHEAD through their light visits (diverging only in trip count) until they
// either finish or stand in front of a heavy visit; then all lanes with a heavy visit pending execute it together.  The number
// of heavy phases is the maximum over lanes of the heavy visits on a lane's path, not the number of rounds with any heavy visit.
//
// Semantics, operation order and capacities are those of stability_check<false, G> (same helpers, same FP64 expressions): the
// verdicts are bit-identical, which tests/test_host_emul_stability.py checks on the host build for whole trajectories.
// Every lane of `mask` must call; lanes without work pass has_work = false.  k_root >= 0: the root's supports were found by the
// caller's fused resting-height scan (sup_pack = the first 4 ids, 8 bits each, scan order); k_root < 0: scan here.
#ifdef __CUDA_ARCH__
#define PCT_ANY(mask, p) __any_sync(mask, p)
#else
#define PCT_ANY(mask, p) (p)
#endif
#ifndef PCT_STAT
#define PCT_STAT(i)   // statistics hook of the host build (tests/host_emul/stab_host.cpp)
#endif
#ifndef PCT_PATH_VISIT  // host statistics: cost of a walk in total and along its longest root-to-leaf path (scratch/stats_paths.py)
#define PCT_PATH_VISIT(c)
#define PCT_PATH_PUSH(d)
#define PCT_PATH_POP(d)
#endif

// stab_light: the LIGHT PREFIX of a feasibility walk — visits of nodes with no or one support (81 % of the walks of the BASELINE streams
// consist of nothing else; host statistics, scratch/stats_farout.py): a rectangle test in registers and the centre-of-mass update, no frames,
// no hull, no local arrays, so the kernel that runs it is small, register-light and convergent (lanes differ in trip count only).
// Returns 0 infeasible / 1 feasible / 2 the walk stands in front of a node with >= 2 supports (or the rare single support whose perturbed
// corners are not in the proven order): (node_out, st_out) is where stab_virtual continues.  Same expressions as stab_virtual's light phase.
template <class G>
static __device__ __forceinline__ int stab_light(const G &g, const typename G::Node &root, int k_root, uint32_t sup_pack, const EdgePool &pool,
                                                 int &node_out, Stack4 &st_out) {
    typedef typename G::Node Node;
    int node = NODE_NEW;
    Stack4 st;
    g.centre(root, st.cx, st.cy, st.cz);
    st.cz = 0;
    st.m = root.mass;
#pragma unroll 1
    for (;;) {
        int k, eoff;
        if (node == NODE_NEW) { k = k_root; eoff = pool.n; }
        else { eoff = (int)pool.off[node]; k = (int)pool.off[node + 1] - eoff; }
        if (k == 0) return 1;  // rests on the floor: every support test above passed
        if (k >= 2) { node_out = node; st_out = st; return 2; }
        PCT_STAT(1);
        const int sid0 = (node == NODE_NEW) ? (int)(sup_pack & 0xFFu) : (int)pool.lower[eoff];
        Node cur;
        if (node != NODE_NEW) g.node_box(node, cur);
        else cur = root;
        double r0[4];
        g.support(cur, sid0, r0);
        const double t1 = r0[1] * 1e-6, t2 = r0[3] * 1e-6;
        const bool fast = (r0[0] + t1 < r0[0] + t2) && (r0[0] + t2 < r0[2] + t1) && (r0[2] + t1 < r0[2] + t2);
        if (!fast) { node_out = node; st_out = st; return 2; }
        if (!pip_rect(r0[0], r0[1], r0[2], r0[3], t1, t2, st.cx, st.cy)) return 0;
        // calculate_new_com of the single support under the whole stack (D:space.py:51-71); its real load from `node` is replaced
        const int skip = (node == NODE_NEW) ? EDGE_NIL : eoff;
        Node sb;
        g.node_box(sid0, sb);
        double ccx, ccy, ccz, mm = sb.mass;
        g.centre(sb, ccx, ccy, ccz);
        ccx *= mm; ccy *= mm;  // the z centre of a stack enters no decision (pip tests are 2-D) and a virtual walk stores nothing: not carried
        (void)ccz;
#pragma unroll 1
        for (int q = pool.first_in[sid0]; q != EDGE_NIL; q = pool.next[q]) {
            if (q == skip) continue;
            const Stack4 e = pool.load(q);
            ccx += e.cx * e.m; ccy += e.cy * e.m;
            mm += e.m;
        }
        if (st.m != 0.0) {
            ccx += st.cx * st.m; ccy += st.cy * st.m;
            mm += st.m;
        }
        ddiv2(ccx, ccy, mm, st.cx, st.cy); st.m = mm;
        node = sid0;
    }
}

// start_node != NODE_NEW: continue a walk that stab_light ran as far as its first node with >= 2 supports (its frame stack is empty there:
// every earlier visit was a tail call) — enter `start_node` with the stack *start_st.
template <class G>
static __device__ __noinline__ int stab_virtual(const G &g, const typename G::Node &root, int k_root, uint32_t sup_pack, const EdgePool &pool,
                                                BigScratch *big, int *lock, int &flags, bool has_work, unsigned mask,
                                                int start_node = NODE_NEW, const Stack4 *start_st = nullptr) {
    typedef typename G::Node Node;
    StabFrame fr[STAB_DEPTH];
    uint8_t sup_id[STAB_SUP_POOL];
    double sup_m[STAB_SUP_POOL], sup_x[STAB_SUP_POOL], sup_y[STAB_SUP_POOL];  // load per support; contact-rectangle centres (split loads only)
    int depth = 0, node = NODE_NEW, base = 0;
    Stack4 st;
    g.centre(root, st.cx, st.cy, st.cz);
    st.cz = 0;
    st.m = root.mass;
    if (start_node != NODE_NEW) { node = start_node; st = *start_st; }
    bool active = has_work, need_adv = false;
    int result = 0;
    int child = -1, skip = EDGE_NIL;
    double vx = 0, vy = 0, vm = 0;
    if (active && k_root < 0) {  // supports of the placement itself (D:space.py:360-376), scan order
        int k = 0;
        const int limit = g.n_boxes();
        double r[4];
        sup_pack = 0;
#pragma unroll 1
        for (int t = 0; t < limit; t++) {
            if (!g.support(root, t, r)) continue;
            if (k < 4) sup_pack |= (uint32_t)t << (8 * k);
            k++;
        }
        k_root = k;
    }
#pragma unroll 1
    for (;;) {
        bool heavy = false;
        int k = 0, eoff = 0;
        // ---------------- light phase: run ahead until finished or in front of a node with >= 2 supports ----------------
#pragma unroll 1
        while (active) {
            if (need_adv) {
                if (child < 0) {
                    // the subtree below the last entered node returned True: continue with the top frame's next support
#pragma unroll 1
                    for (;;) {
                        if (depth == 0) { active = false; result = 1; break; }
                        StabFrame &f = fr[depth - 1];
                        if (f.i == f.k) { depth--; continue; }
                        const int s = f.i++;
                        PCT_PATH_POP(depth - 1);
                        child = sup_id[f.base + s];
                        const int parent = f.node;
                        skip = (parent == NODE_NEW) ? EDGE_NIL : (int)f.eoff + s;
                        st = f.st;
                        vm = sup_m[f.base + s];
                        vx = st.cx; vy = st.cy;
                        if (!f.whole) { vx = sup_x[f.base + s]; vy = sup_y[f.base + s]; }  // the load sits at the centre of this support's contact rectangle with the parent
                        base = f.base + f.k;
                        if (s == f.k - 1) { depth--; base = f.base; }  // tail call: the parent frame is finished
                        break;
                    }
                    if (!active) break;
                }
                // calculate_new_com of `child` (D:space.py:51-71) under the virtual load (vx, vy, st.cz, vm)
                Node sb;
                g.node_box(child, sb);
                double ccx, ccy, ccz, mm = sb.mass;
                g.centre(sb, ccx, ccy, ccz);
                ccx *= mm; ccy *= mm;  // z: see stab_light
                (void)ccz;
#pragma unroll 1
                for (int q = pool.first_in[child]; q != EDGE_NIL; q = pool.next[q]) {
                    if (q == skip) continue;  // `involved` path member: its real load is replaced by the virtual one
                    const Stack4 e = pool.load(q);
                    ccx += e.cx * e.m; ccy += e.cy * e.m;
                    mm += e.m;
                }
                if (vm != 0.0) {  // zero-mass virtual loads add +0.0 to every sum: skipped (exact)
                    ccx += vx * vm; ccy += vy * vm;
                    mm += vm;
                }
                ddiv2(ccx, ccy, mm, st.cx, st.cy); st.m = mm;
                node = child;
                need_adv = false;
            }
            // ENTER(node, st): how many supports?
            if (node == NODE_NEW) { k = k_root; eoff = pool.n; }
            else { eoff = (int)pool.off[node]; k = (int)pool.off[node + 1] - eoff; }
            if (k >= 2) { heavy = true; break; }
            child = -1;
            PCT_STAT(k);  // 0 / 1: light visits
            PCT_PATH_VISIT(k ? 1.0 : 0.1);
            if (k == 1) {
                const int sid0 = (node == NODE_NEW) ? (int)(sup_pack & 0xFFu) : (int)pool.lower[eoff];
                Node cur;
                if (node != NODE_NEW) g.node_box(node, cur);
                else cur = root;
                double r0[4];
                g.support(cur, sid0, r0);
                const double t1 = r0[1] * 1e-6, t2 = r0[3] * 1e-6;
                const bool fast = (r0[0] + t1 < r0[0] + t2) && (r0[0] + t2 < r0[2] + t1) && (r0[2] + t1 < r0[2] + t2);
                bool ok;
                if (fast) ok = pip_rect(r0[0], r0[1], r0[2], r0[3], t1, t2, st.cx, st.cy);
                else {
                    double px[4] = {r0[0] + t1, r0[0] + t2, r0[2] + t1, r0[2] + t2}, py[4] = {r0[1], r0[3], r0[1], r0[3]};
                    double hx[8], hy[8];
                    const int m = hull_coords(px, py, 4, hx, hy);
                    ok = pip_shrunk(hx, hy, 1, m, st.cx, st.cy);
                }
                if (!ok) PCT_STAT(node == NODE_NEW ? 17 : 18);  // light visit failed: root / placed box
                if (!ok) { active = false; result = 0; break; }
                child = sid0;  // the whole stack goes to the single support
                skip = (node == NODE_NEW) ? EDGE_NIL : eoff;
                vx = st.cx; vy = st.cy; vm = st.m;
            }
            need_adv = true;
        }
        if (!PCT_ANY(mask, heavy)) break;
        // ---------------- heavy phase: every lane standing in front of a node with >= 2 supports enters it ----------------
        if (heavy) {
            PCT_STAT(node == NODE_NEW ? 2 : 3);  // heavy visits: root / placed box
            PCT_STAT(4 + (k < 8 ? k : 8));       // by number of supports
            PCT_PATH_VISIT(node == NODE_NEW ? 6.0 : 3.5);
            Node cur;
            if (node != NODE_NEW) g.node_box(node, cur);
            else cur = root;
            bool ok = true;
            if (node == NODE_NEW) {
                if (k > KSUP_MAX || k > STAB_SUP_POOL) { flags |= PCT_FLAG_SUPPORT_OVERFLOW; ok = false; }
                else if (k <= 4) {
#pragma unroll 1
                    for (int j = 0; j < k; j++) sup_id[base + j] = (uint8_t)((sup_pack >> (8 * j)) & 0xFFu);
                } else {
                    int kk = 0;
                    const int limit = g.n_boxes();
                    double r[4];
#pragma unroll 1
                    for (int t = 0; t < limit && kk < k; t++)
                        if (g.support(cur, t, r)) sup_id[base + kk++] = (uint8_t)t;
                }
            } else {
                if (base + k > STAB_SUP_POOL) { flags |= PCT_FLAG_SUPPORT_OVERFLOW; ok = false; }
                else {
#pragma unroll 1
                    for (int j = 0; j < k; j++) sup_id[base + j] = pool.lower[eoff + j];
                }
            }
            int whole = 2;
            if (ok) {
                double lrect[KSUP_SMALL][4], lpx[4 * KSUP_SMALL], lpy[4 * KSUP_SMALL], lhx[8 * KSUP_SMALL], lhy[8 * KSUP_SMALL];
                const bool small = k <= KSUP_SMALL;
                double (*rect)[4] = lrect;
                double *px = lpx, *py = lpy, *hx = lhx, *hy = lhy;
                if (!small) {  // rare: serialise the lanes of this env on the per-env HBM scratch
                    while (atomicCAS(lock, 0, 1) != 0) { }
                    __threadfence_block();
                    rect = big->rect; px = big->px; py = big->py; hx = big->hx; hy = big->hy;
                }
#pragma unroll 1
                for (int s = 0; s < k; s++) g.support(cur, sup_id[base + s], rect[s]);
                const double *split = nullptr;  // k == 2, placed box: the stored split direction
                const int pv = node == NODE_NEW ? 0 : (int)pool.poly_off[node], pm = node == NODE_NEW ? 0 : (int)pool.poly_off[node + 1] - pv;
                if (pm > 0 && (pv + pm <= POLY_STAGE || pv >= POLY_STAGE)) {
                    const double *xy = pool.poly_at(pv);  // a placed box: its shrunk support polygon was stored when it was placed
                    ok = pip_stored(xy, pm - (k == 2), st.cx, st.cy);
                    if (k == 2) split = xy + 2 * (pm - 1);
                } else {
#pragma unroll 1
                    for (int s = 0; s < k; s++) {
                        const double x1 = rect[s][0], y1 = rect[s][1], x2 = rect[s][2], y2 = rect[s][3];
                        const double t1 = y1 * 1e-6, t2 = y2 * 1e-6;
                        px[4 * s + 0] = x1 + t1; py[4 * s + 0] = y1;
                        px[4 * s + 1] = x1 + t2; py[4 * s + 1] = y2;
                        px[4 * s + 2] = x2 + t1; py[4 * s + 2] = y1;
                        px[4 * s + 3] = x2 + t2; py[4 * s + 3] = y2;
                    }
                    const int m = hull_coords(px, py, 4 * k, hx, hy);
                    ok = pip_shrunk(hx, hy, 1, m, st.cx, st.cy);
                }
                if (ok) {
                    int direct = -1;
#pragma unroll 1
                    for (int s = 0; s < k; s++)
                        if (g.strictly_inside(st.cx, st.cy, rect[s])) { direct = s; break; }
                    if (direct >= 0) {
#pragma unroll 1
                        for (int s = 0; s < k; s++) sup_m[base + s] = (s == direct) ? st.m : 0.0;
                    } else {
                        whole = 0;
#pragma unroll 1
                        for (int s = 0; s < k; s++) {
                            sup_x[base + s] = px[s] = (rect[s][0] + rect[s][2]) * 0.5;
                            sup_y[base + s] = py[s] = (rect[s][1] + rect[s][3]) * 0.5;
                        }
                        if (k == 2) {
                            double lx, ly;
                            if (split) { lx = split[0]; ly = split[1]; }
                            else split2_dir(px, py, lx, ly);
                            sup_m[base + 0] = st.m * fabs(dot2(st.cx - px[1], st.cy - py[1], lx, ly));
                            sup_m[base + 1] = st.m * fabs(dot2(st.cx - px[0], st.cy - py[0], lx, ly));
                        } else {
                            PCT_STAT(14);
                            PCT_PATH_VISIT(10.0);
                            double lR[KSUP_SMALL * KSUP_SMALL], lV[KSUP_SMALL * KSUP_SMALL], ly_[KSUP_SMALL], lrow[KSUP_SMALL], lx_[KSUP_SMALL];
                            LsWork w;
                            w.R = small ? lR : big->R; w.V = small ? lV : big->V; w.y = small ? ly_ : big->y;
                            w.row = small ? lrow : big->row; w.x = small ? lx_ : big->x; w.ld = small ? KSUP_SMALL : KSUP_MAX;
                            lstsq_ratios(w, k, px, py, st.cx, st.cy);
#pragma unroll 1
                            for (int s = 0; s < k; s++) sup_m[base + s] = st.m * w.x[s];
                        }
                    }
                }
                if (!small) { __threadfence_block(); atomicExch(lock, 0); }
            }
            if (ok && depth >= STAB_DEPTH) { flags |= PCT_FLAG_SUPPORT_OVERFLOW; ok = false; }
            if (!ok) PCT_STAT(node == NODE_NEW ? 15 : 16);  // heavy visit failed: root / placed box
            if (!ok) { active = false; result = 0; }
            else {
                StabFrame &f = fr[depth++];
                PCT_PATH_PUSH(depth - 1);
                f.st = st; f.node = (uint8_t)node; f.base = (uint8_t)base; f.k = (uint8_t)k; f.i = 0; f.whole = (uint8_t)whole;
                f.eoff = (uint8_t)eoff;
                child = -1;
                need_adv = true;
            }
        }
    }
    return result;
}


// ---- fork-join form of the read-only walk (round 2, pct_walk_fork_kernel) -----------------------------------------------------------------------
// calculated_impact_virtual is a conjunction over the support DAG below the placement: a node with k >= 2 supports passes iff its own polygon
// test passes AND every support subtree passes, and a read-only walk has no side effects — so the k subtrees are independent.  stab_piece runs ONE
// chain of the walk: it visits nodes, follows single supports itself (tail calls) and, at a node with k >= 2 supports, keeps the first subtree and
// hands the other k - 1 to `fork` as new pieces; the walk's verdict is the AND over its pieces (the reference's depth-first order only decides
// which failing subtree is seen first).  No frames and no per-depth arrays are left: the state of a piece is (node, stack).  The longest walk of a step
// (what the continuation kernel's duration was) shrinks from the SUM over its visits to its longest root-to-floor path (host statistics,
// scratch/stats_paths.py: 51 -> 34 visit units at the 99.99 % quantile).
// A piece is either "enter `node` with the stack (a, b, c) = (cx, cy, mass)" (kind 0) or "the load (a, b, c) = (x, y, mass) arrives on `node`
// in place of the stored edge `skip`: combine (calculate_new_com), then enter" (kind 1).
// (struct WalkPiece: pct_kernels.h)

template <class G, class Fork>
static __device__ __noinline__ int stab_piece(const G &g, const typename G::Node &root, int k_root, uint32_t sup_pack, const EdgePool &pool,
                                              BigScratch *big, int *lock, int &flags, int node, int kind, int skip, double pa, double pb, double pc,
                                              Fork &fork) {
    typedef typename G::Node Node;
    Stack4 st;
    st.cx = pa; st.cy = pb; st.cz = 0; st.m = pc;
    bool need_com = kind != 0;
    int child = node;
    double vx = pa, vy = pb, vm = pc;
#pragma unroll 1
    for (;;) {
        if (need_com) {
            // calculate_new_com of `child` (D:space.py:51-71) under the virtual load (vx, vy, vm); z: see stab_light
            Node sb;
            g.node_box(child, sb);
            double ccx, ccy, ccz, mm = sb.mass;
            g.centre(sb, ccx, ccy, ccz);
            ccx *= mm; ccy *= mm;
            (void)ccz;
#pragma unroll 1
            for (int q = pool.first_in[child]; q != EDGE_NIL; q = pool.next[q]) {
                if (q == skip) continue;  // `involved` path member: its real load is replaced by the virtual one
                const Stack4 e = pool.load(q);
                ccx += e.cx * e.m; ccy += e.cy * e.m;
                mm += e.m;
            }
            if (vm != 0.0) {  // zero-mass virtual loads add +0.0 to every sum: skipped (exact)
                ccx += vx * vm; ccy += vy * vm;
                mm += vm;
            }
            ddiv2(ccx, ccy, mm, st.cx, st.cy); st.m = mm;
            node = child;
        }
        need_com = true;
        // ENTER(node, st)
        int k, eoff;
        if (node == NODE_NEW) { k = k_root; eoff = pool.n; }
        else { eoff = (int)pool.off[node]; k = (int)pool.off[node + 1] - eoff; }
        if (k == 0) return 1;  // rests on the floor
        Node cur;
        if (node != NODE_NEW) g.node_box(node, cur);
        else cur = root;
        if (k == 1) {
            PCT_STAT(1);
            PCT_PATH_VISIT(1.0);
            const int sid0 = (node == NODE_NEW) ? (int)(sup_pack & 0xFFu) : (int)pool.lower[eoff];
            double r0[4];
            g.support(cur, sid0, r0);
            const double t1 = r0[1] * 1e-6, t2 = r0[3] * 1e-6;
            const bool fast = (r0[0] + t1 < r0[0] + t2) && (r0[0] + t2 < r0[2] + t1) && (r0[2] + t1 < r0[2] + t2);
            bool ok;
            if (fast) ok = pip_rect(r0[0], r0[1], r0[2], r0[3], t1, t2, st.cx, st.cy);
            else {
                double px[4] = {r0[0] + t1, r0[0] + t2, r0[2] + t1, r0[2] + t2}, py[4] = {r0[1], r0[3], r0[1], r0[3]};
                double hx[8], hy[8];
                const int m = hull_coords(px, py, 4, hx, hy);
                ok = pip_shrunk(hx, hy, 1, m, st.cx, st.cy);
            }
            if (!ok) return 0;
            child = sid0;  // the whole stack goes to the single support
            skip = (node == NODE_NEW) ? EDGE_NIL : eoff;
            vx = st.cx; vy = st.cy; vm = st.m;
            continue;
        }
        // ---------------- k >= 2 supports: polygon test, load split, fork ----------------
        PCT_STAT(node == NODE_NEW ? 2 : 3);
        PCT_STAT(4 + (k < 8 ? k : 8));
        PCT_PATH_VISIT(node == NODE_NEW ? 6.0 : 3.5);
        uint8_t sup_id[KSUP_MAX];
        double sup_m[KSUP_MAX];
        if (k > KSUP_MAX) { flags |= PCT_FLAG_SUPPORT_OVERFLOW; return 0; }
        if (node == NODE_NEW) {
            if (k <= 4) {
#pragma unroll 1
                for (int j = 0; j < k; j++) sup_id[j] = (uint8_t)((sup_pack >> (8 * j)) & 0xFFu);
            } else {
                int kk = 0;
                const int limit = g.n_boxes();
                double r[4];
#pragma unroll 1
                for (int t = 0; t < limit && kk < k; t++)
                    if (g.support(cur, t, r)) sup_id[kk++] = (uint8_t)t;
            }
        } else {
#pragma unroll 1
            for (int j = 0; j < k; j++) sup_id[j] = pool.lower[eoff + j];
        }
        int whole = 2;
        bool ok;
        double lrect[KSUP_SMALL][4], lpx[4 * KSUP_SMALL], lpy[4 * KSUP_SMALL], lhx[8 * KSUP_SMALL], lhy[8 * KSUP_SMALL];
        const bool small = k <= KSUP_SMALL;
        double (*rect)[4] = lrect;
        double *px = lpx, *py = lpy, *hx = lhx, *hy = lhy;
        if (!small) {  // rare: serialise the lanes of this env on the per-env HBM scratch
            while (atomicCAS(lock, 0, 1) != 0) { }
            __threadfence_block();
            rect = big->rect; px = big->px; py = big->py; hx = big->hx; hy = big->hy;
        }
#pragma unroll 1
        for (int s = 0; s < k; s++) g.support(cur, sup_id[s], rect[s]);
        const double *split = nullptr;  // k == 2, placed box: the stored split direction
        const int pv = node == NODE_NEW ? 0 : (int)pool.poly_off[node], pm = node == NODE_NEW ? 0 : (int)pool.poly_off[node + 1] - pv;
        if (pm > 0 && (pv + pm <= POLY_STAGE || pv >= POLY_STAGE)) {
            const double *xy = pool.poly_at(pv);  // a placed box: its shrunk support polygon was stored when it was placed
            ok = pip_stored(xy, pm - (k == 2), st.cx, st.cy);
            if (k == 2) split = xy + 2 * (pm - 1);
        } else {
#pragma unroll 1
            for (int s = 0; s < k; s++) {
                const double x1 = rect[s][0], y1 = rect[s][1], x2 = rect[s][2], y2 = rect[s][3];
                const double t1 = y1 * 1e-6, t2 = y2 * 1e-6;
                px[4 * s + 0] = x1 + t1; py[4 * s + 0] = y1;
                px[4 * s + 1] = x1 + t2; py[4 * s + 1] = y2;
                px[4 * s + 2] = x2 + t1; py[4 * s + 2] = y1;
                px[4 * s + 3] = x2 + t2; py[4 * s + 3] = y2;
            }
            const int m = hull_coords(px, py, 4 * k, hx, hy);
            ok = pip_shrunk(hx, hy, 1, m, st.cx, st.cy);
        }
        if (ok) {
            int direct = -1;
#pragma unroll 1
            for (int s = 0; s < k; s++)
                if (g.strictly_inside(st.cx, st.cy, rect[s])) { direct = s; break; }
            if (direct >= 0) {
#pragma unroll 1
                for (int s = 0; s < k; s++) sup_m[s] = (s == direct) ? st.m : 0.0;
            } else {
                whole = 0;
#pragma unroll 1
                for (int s = 0; s < k; s++) {
                    px[s] = (rect[s][0] + rect[s][2]) * 0.5;
                    py[s] = (rect[s][1] + rect[s][3]) * 0.5;
                }
                if (k == 2) {
                    double lx, ly;
                    if (split) { lx = split[0]; ly = split[1]; }
                    else split2_dir(px, py, lx, ly);
                    sup_m[0] = st.m * fabs(dot2(st.cx - px[1], st.cy - py[1], lx, ly));
                    sup_m[1] = st.m * fabs(dot2(st.cx - px[0], st.cy - py[0], lx, ly));
                } else {
                    PCT_STAT(14);
                    PCT_PATH_VISIT(10.0);
                    double lR[KSUP_SMALL * KSUP_SMALL], lV[KSUP_SMALL * KSUP_SMALL], ly_[KSUP_SMALL], lrow[KSUP_SMALL], lx_[KSUP_SMALL];
                    LsWork w;
                    w.R = small ? lR : big->R; w.V = small ? lV : big->V; w.y = small ? ly_ : big->y;
                    w.row = small ? lrow : big->row; w.x = small ? lx_ : big->x; w.ld = small ? KSUP_SMALL : KSUP_MAX;
                    lstsq_ratios(w, k, px, py, st.cx, st.cy);
#pragma unroll 1
                    for (int s = 0; s < k; s++) sup_m[s] = st.m * w.x[s];
                }
            }
            // the subtrees of supports 1 .. k-1 become pieces of their own; support 0 is followed here
#pragma unroll 1
            for (int s = 1; s < k; s++)
                fork((int)sup_id[s], (node == NODE_NEW) ? EDGE_NIL : eoff + s, whole ? st.cx : px[s], whole ? st.cy : py[s], sup_m[s]);
            vx = whole ? st.cx : px[0]; vy = whole ? st.cy : py[0]; vm = sup_m[0];
        }
        if (!small) { __threadfence_block(); atomicExch(lock, 0); }
        if (!ok) return 0;
        child = sup_id[0];
        skip = (node == NODE_NEW) ? EDGE_NIL : eoff;
    }
}


}  // namespace pct
