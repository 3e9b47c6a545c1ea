// TEST INFRASTRUCTURE — device unit library of the stability check's FP64 primitives (tests/test_gpu_geometry_units.py).
// The product headers are included unchanged, so every launcher below runs the product's own function, compiled with the product's
// flags (Makefile), one thread per input.  Launchers take raw device pointers (torch tensors), run on the legacy default stream and
// synchronise: they return the CUDA error code (0 = success).  Two test-local mutants (orient3 / cross_left with their pre-filter
// tolerance set to 0) live here and only here: they show that the near-tie input sets can tell a wrong pre-filter from the product's.
#include <cstdint>
#include <cuda_runtime.h>
#include "pct_stability.cuh"
#include "pct_geom.cuh"
#include "pct_geom_continuous.cuh"
#include "pct_pyhash.cuh"

using namespace pct;

#define GRID(n) dim3((unsigned)(((n) + 127) / 128)), dim3(128)
#define FINISH() do { cudaError_t e_ = cudaGetLastError(); if (e_ != cudaSuccess) return (int)e_; return (int)cudaDeviceSynchronize(); } while (0)

// ---- test-local mutants: the product's pre-filters with tolerance 0 (the float estimate decides whenever the float gap is non-zero) ----
__device__ __noinline__ int orient3_tol0(double ax, double ay, double bx, double by, double cx, double cy) {
    const double d1x = bx - ax, d1y = by - ay, d2x = cx - bx, d2y = cy - by;
    if (d1x != 0 && d2x != 0) {
        if (d1y == 0 && d2y == 0) return 0;
        const float f1 = __fdividef((float)d1y, (float)d1x), f2 = __fdividef((float)d2y, (float)d2x);
        const float gap = f2 - f1;
        if (fabsf(gap) > 0.0f && fabsf(f1) < 1e30f && fabsf(f2) < 1e30f) return gap > 0 ? -1 : 1;
    }
    return orient_of(slope_of(ax, ay, bx, by), slope_of(bx, by, cx, cy));
}
__device__ __noinline__ bool cross_left_tol0(double ix, double iy, double jx, double jy, double lat, double lon) {
    const float xf = (float)ix + __fdividef((float)(lon - iy), (float)(jy - iy)) * (float)(jx - ix);
    const float gap = xf - (float)lat;
    if (fabsf(gap) > 1e-30f) return gap < 0;
    const double t = ddiv(lon - iy, jy - iy);
    const double u = t * (jx - ix);
    return ix + u < lat;
}

// in [n][6] = (ax, ay, bx, by, cx, cy) -> out [n][4] = orient3, orient_of(slope_of, slope_of), branch, mutant; ratio[n] = |float gap| / tol
// branch: 0 exact path, 1 decided by the float pre-filter, 2 horizontal early-out.  The branch is restated here for coverage accounting only.
__global__ void k_orient3(const double *in, int n, int *out, float *ratio) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double *p = in + 6 * i;
    const double ax = p[0], ay = p[1], bx = p[2], by = p[3], cx = p[4], cy = p[5];
    out[4 * i + 0] = orient3(ax, ay, bx, by, cx, cy);
    out[4 * i + 1] = orient_of(slope_of(ax, ay, bx, by), slope_of(bx, by, cx, cy));
    out[4 * i + 3] = orient3_tol0(ax, ay, bx, by, cx, cy);
    const double d1x = bx - ax, d1y = by - ay, d2x = cx - bx, d2y = cy - by;
    int br = 0;
    float rt = -1.0f;
    if (d1x != 0 && d2x != 0) {
        if (d1y == 0 && d2y == 0) br = 2;
        else {
            const float f1 = __fdividef((float)d1y, (float)d1x), f2 = __fdividef((float)d2y, (float)d2x);
            const float gap = f2 - f1, tol = 1e-4f * (fabsf(f1) + fabsf(f2));
            if (fabsf(gap) > tol && fabsf(f1) < 1e30f && fabsf(f2) < 1e30f) br = 1;
            rt = tol > 0 ? fabsf(gap) / tol : -1.0f;
        }
    }
    out[4 * i + 2] = br;
    ratio[i] = rt;
}
extern "C" int gu_orient3(const double *in, int n, int *out, float *ratio) { if (n > 0) k_orient3<<<GRID(n)>>>(in, n, out, ratio); FINISH(); }

// in [n][6] = (ix, iy, jx, jy, lat, lon) -> out [n][3] = cross_left, branch (1: decided by the float estimate), mutant
__global__ void k_cross_left(const double *in, int n, int *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double *p = in + 6 * i;
    out[3 * i + 0] = cross_left(p[0], p[1], p[2], p[3], p[4], p[5]);
    const float xf = (float)p[0] + __fdividef((float)(p[5] - p[1]), (float)(p[3] - p[1])) * (float)(p[2] - p[0]);
    const float scale = fabsf((float)p[0]) + fabsf((float)(p[2] - p[0])) + fabsf((float)p[4]);
    out[3 * i + 1] = fabsf(xf - (float)p[4]) > 1e-4f * scale + 1e-30f;
    out[3 * i + 2] = cross_left_tol0(p[0], p[1], p[2], p[3], p[4], p[5]);
}
extern "C" int gu_cross_left(const double *in, int n, int *out) { if (n > 0) k_cross_left<<<GRID(n)>>>(in, n, out); FINISH(); }

// in [n][6] = (ix, iy, jx, jy, lat, lon) -> pip_edge
__global__ void k_pip_edge(const double *in, int n, int *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double *p = in + 6 * i;
    out[i] = pip_edge(p[0], p[1], p[2], p[3], p[4], p[5]);
}
extern "C" int gu_pip_edge(const double *in, int n, int *out) { if (n > 0) k_pip_edge<<<GRID(n)>>>(in, n, out); FINISH(); }

// in [n][6] = (x1, y1, x2, y2, lat, lon) of one contact rectangle -> out [n][2] = the `fast` precondition of stability_check, pip_rect
// (pip_rect is only called, and only meaningful, where `fast` holds)
__global__ void k_pip_rect(const double *in, int n, int *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double *r0 = in + 6 * i;
    const double t1 = r0[1] * 1e-6, t2 = r0[3] * 1e-6;
    const bool fast = (r0[0] + t1 < r0[0] + t2) && (r0[0] + t2 < r0[2] + t1) && (r0[2] + t1 < r0[2] + t2);
    out[2 * i + 0] = fast;
    out[2 * i + 1] = fast ? pip_rect(r0[0], r0[1], r0[2], r0[3], t1, t2, r0[4], r0[5]) : 0;
}
extern "C" int gu_pip_rect(const double *in, int n, int *out) { if (n > 0) k_pip_rect<<<GRID(n)>>>(in, n, out); FINISH(); }

// hull_coords on already perturbed points: problem i owns px/py[off[i] .. off[i+1]) (sorted in place) and hx/hy[2 off[i] ..); m[i] = hull size
__global__ void k_hull(double *px, double *py, const int *off, int n, double *hx, double *hy, int *m) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int o = off[i], np = off[i + 1] - o;
    m[i] = hull_coords(px + o, py + o, np, hx + 2 * o, hy + 2 * o);
}
extern "C" int gu_hull(double *px, double *py, const int *off, int n, double *hx, double *hy, int *m) {
    if (n > 0) k_hull<<<GRID(n)>>>(px, py, off, n, hx, hy, m);
    FINISH();
}

// pip_shrunk of query q on hull poly[q] (vertices hx/hy[hoff[poly[q]] ..), m[poly[q]] of them)
__global__ void k_pip_shrunk(const double *hx, const double *hy, const int *hoff, const int *m, const int *poly, const double *q, int nq, int *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    const int p = poly[i];
    out[i] = pip_shrunk(hx + hoff[p], hy + hoff[p], 1, m[p], q[2 * i], q[2 * i + 1]);
}
extern "C" int gu_pip_shrunk(const double *hx, const double *hy, const int *hoff, const int *m, const int *poly, const double *q, int nq, int *out) {
    if (nq > 0) k_pip_shrunk<<<GRID(nq)>>>(hx, hy, hoff, m, poly, q, nq, out);
    FINISH();
}

// pip_stored of query q on the stored (x, y interleaved) polygon poly[q]: vertices xy[2 off[p] ..), off[p+1] - off[p] of them
__global__ void k_pip_stored(const double *xy, const int *off, const int *poly, const double *q, int nq, int *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    const int p = poly[i];
    out[i] = pip_stored(xy + 2 * off[p], off[p + 1] - off[p], q[2 * i], q[2 * i + 1]);
}
extern "C" int gu_pip_stored(const double *xy, const int *off, const int *poly, const double *q, int nq, int *out) {
    if (nq > 0) k_pip_stored<<<GRID(nq)>>>(xy, off, poly, q, nq, out);
    FINISH();
}

// in [n][7] = (px0, px1, py0, py1, cx, cy, m): two-support split of stability_check -> out [n][6] = lx, ly (split2_dir), sup_m0, sup_m1,
// dot2(px0, py0, px1, py1) (plain dot2 of the raw operands), and 0
__global__ void k_split2(const double *in, int n, double *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double *p = in + 7 * i;
    const double px[2] = {p[0], p[1]}, py[2] = {p[2], p[3]};
    double lx, ly;
    split2_dir(px, py, lx, ly);
    double *o = out + 6 * i;
    o[0] = lx; o[1] = ly;
    o[2] = p[6] * fabs(dot2(p[4] - px[1], p[5] - py[1], lx, ly));
    o[3] = p[6] * fabs(dot2(p[4] - px[0], p[5] - py[0], lx, ly));
    o[4] = dot2(p[0], p[2], p[1], p[3]);
    o[5] = 0;
}
extern "C" int gu_split2(const double *in, int n, double *out) { if (n > 0) k_split2<<<GRID(n)>>>(in, n, out); FINISH(); }

// lstsq_ratios of system i: k[i] contact-rectangle centres c2x/c2y[off[i] ..), stack centre com[2 i], com[2 i + 1]; the LsWork lives in global
// scratch (LS_STRIDE doubles per system) with the leading dimension stability_check picks: KSUP_SMALL for k <= 8, KSUP_MAX above.  x -> x[off[i] ..)
constexpr int LS_STRIDE = 2 * KSUP_MAX * KSUP_MAX + 3 * KSUP_MAX;
__global__ void k_lstsq(const double *c2x, const double *c2y, const int *off, const double *com, int n, double *scratch, double *x) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int o = off[i], k = off[i + 1] - o;
    double *s = scratch + (size_t)LS_STRIDE * i;
    LsWork w;
    w.ld = k <= KSUP_SMALL ? KSUP_SMALL : KSUP_MAX;
    w.R = s; w.V = s + KSUP_MAX * KSUP_MAX; w.y = s + 2 * KSUP_MAX * KSUP_MAX; w.row = w.y + KSUP_MAX; w.x = w.row + KSUP_MAX;
    lstsq_ratios(w, k, c2x + o, c2y + o, com[2 * i], com[2 * i + 1]);
    for (int j = 0; j < k; j++) x[o + j] = w.x[j];
}
extern "C" int gu_lstsq_stride() { return LS_STRIDE; }
extern "C" int gu_lstsq(const double *c2x, const double *c2y, const int *off, const double *com, int n, double *scratch, double *x) {
    if (n > 0) k_lstsq<<<GRID(n)>>>(c2x, c2y, off, com, n, scratch, x);
    FINISH();
}

__global__ void k_around6(const double *in, int n, double *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = around6(in[i]);
}
extern "C" int gu_around6(const double *in, int n, double *out) { if (n > 0) k_around6<<<GRID(n)>>>(in, n, out); FINISH(); }

__global__ void k_hash(const double *in, int n, unsigned long long *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = hash_double(in[i]);
}
extern "C" int gu_hash_double(const double *in, int n, unsigned long long *out) { if (n > 0) k_hash<<<GRID(n)>>>(in, n, out); FINISH(); }

// The exhaustive proof of around6's division-free quotient, on the device: for every integer a in [lo, hi) take v = a / 1e6.  cnt[0] counts
// the a with rint(v * 1e6) != a (none: the relative error of v * 1e6 is below 0.5 / 2.2e9), cnt[1] those with around6(v) != a / 1e6.
// Positive controls: cnt[2] counts the a where the uncorrected quotient a * 1e-6 differs from a / 1e6 (about 30 %), cnt[3] the operands visited.
__global__ void k_around6_range(long long lo, long long hi, unsigned long long *cnt) {
    unsigned long long bad_rint = 0, bad = 0, bad_q0 = 0, seen = 0;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = lo + blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += stride) {
        const double a = (double)i;
        const double v = ddiv(a, 1e6);
        bad_rint += rint(v * 1e6) != a;
        bad += around6(v) != v;
        bad_q0 += a * 1e-6 != v;
        seen++;
    }
    if (bad_rint) atomicAdd(cnt, bad_rint);
    if (bad) atomicAdd(cnt + 1, bad);
    if (bad_q0) atomicAdd(cnt + 2, bad_q0);
    if (seen) atomicAdd(cnt + 3, seen);
}
extern "C" int gu_around6_range(long long lo, long long hi, unsigned long long *cnt) {
    if (hi > lo) k_around6_range<<<132 * 16, 256>>>(lo, hi, cnt);
    FINISH();
}

// Root test of a DISCRETE placement: query i = (layout, lx, ly, dx, dy) on the boxes of its layout (nbox[layout] of NB_MAX int16 records,
// lx ly lz hx hy hz).  out [n][8] = rest_height, rest_height_supports (mh, k, pack, far_out), the centre's hull test on the supports' contact
// rectangles (pip_shrunk on hull_coords of the perturbed corners, as stability_check builds it; -1 if k == 0 or k > KSUP_MAX), direct support
// (GeomD::strictly_inside: index of the first rectangle, -1 none), k again from GeomD::support.  rects [n][KSUP_MAX][4] = the contact rectangles.
__global__ void k_root_d(const int16_t *boxes, const int *nbox, const int *q, int n, int *out, double *rects, double *scratch) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int lay = q[5 * i], lx = q[5 * i + 1], ly = q[5 * i + 2], dx = q[5 * i + 3], dy = q[5 * i + 4];
    const int16_t (*box)[6] = (const int16_t (*)[6])(boxes + (size_t)lay * NB_MAX * 6);
    const int nb = nbox[lay];
    int k = 0;
    uint32_t pack = 0;
    bool far_out = false;
    const int mh = rest_height_supports(box, nb, lx, ly, lx + dx, ly + dy, k, pack, far_out);
    int *o = out + 8 * i;
    o[0] = rest_height(box, 0, nb, 1, lx, ly, lx + dx, ly + dy);
    o[1] = mh; o[2] = k; o[3] = (int)pack; o[4] = far_out;
    GeomD g{box, nb, nullptr};
    NodeD nd{lx, ly, mh, dx, dy, 1, 1.0};
    double cx, cy, cz;
    g.centre(nd, cx, cy, cz);
    double *rc = rects + (size_t)i * KSUP_MAX * 4;
    int ks = 0, direct = -1;
    for (int t = 0; t < nb && ks < KSUP_MAX; t++) {
        double r[4];
        if (!g.support(nd, t, r)) continue;
        for (int c = 0; c < 4; c++) rc[4 * ks + c] = r[c];
        if (direct < 0 && g.strictly_inside(cx, cy, r)) direct = ks;
        ks++;
    }
    o[6] = direct; o[7] = ks;
    int pip = -1;
    if (ks > 0 && mh > 0) {
        double *px = scratch + (size_t)i * 24 * KSUP_MAX, *py = px + 4 * KSUP_MAX, *hx = py + 4 * KSUP_MAX, *hy = hx + 8 * KSUP_MAX;
        for (int s = 0; s < ks; s++) {
            const double x1 = rc[4 * s], y1 = rc[4 * s + 1], x2 = rc[4 * s + 2], y2 = rc[4 * s + 3];
            const double t1 = y1 * 1e-6, t2 = y2 * 1e-6;
            px[4 * s + 0] = x1 + t1; py[4 * s + 0] = y1;
            px[4 * s + 1] = x1 + t2; py[4 * s + 1] = y2;
            px[4 * s + 2] = x2 + t1; py[4 * s + 2] = y1;
            px[4 * s + 3] = x2 + t2; py[4 * s + 3] = y2;
        }
        const int m = hull_coords(px, py, 4 * ks, hx, hy);
        pip = pip_shrunk(hx, hy, 1, m, cx, cy);
    }
    o[5] = pip;
}
extern "C" int gu_root_d(const int16_t *boxes, const int *nbox, const int *q, int n, int *out, double *rects, double *scratch) {
    if (n > 0) k_root_d<<<GRID(n)>>>(boxes, nbox, q, n, out, rects, scratch);
    FINISH();
}

// Root test of a CONTINUOUS placement: query i = (layout, lx, ly, x, y) on the boxes of its layout (nbox[layout] of NB_MAX double records
// lx ly lz dx dy dz, density 1).  out [n][5] = rest_height_c, rest_height_pre (operands pre-rounded as the candidates kernel does), k (supports by
// GeomC::support at the resting height), the centre's hull test (-1 if k == 0, k > KSUP_MAX or the resting height is the floor), direct support;
// rects [n][KSUP_MAX][4] = the contact rectangles GeomC::support returns.
__global__ void k_root_c(const double *boxes, const int *nbox, const double *q, int n, double *out, double *rects, double *scratch) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int lay = (int)q[5 * i];
    const double lx = q[5 * i + 1], ly = q[5 * i + 2], x = q[5 * i + 3], y = q[5 * i + 4];
    const double (*box)[6] = (const double (*)[6])(boxes + (size_t)lay * NB_MAX * 6);
    const int nb = nbox[lay];
    double *o = out + 5 * i;
    double mh = rest_height_c(box, 0, nb, 1, lx, ly, lx + x, ly + y);
    o[0] = mh;
    double (*rb)[5] = (double (*)[5])(scratch + (size_t)i * 24 * KSUP_MAX);  // NB_MAX * 5 <= 24 * KSUP_MAX
    for (int t = 0; t < nb; t++) {
        const double *b = box[t];
        rb[t][0] = around6(-b[0]); rb[t][1] = around6(-b[1]); rb[t][2] = around6(b[0] + b[3]); rb[t][3] = around6(b[1] + b[4]);
        rb[t][4] = b[2] + b[5];
    }
    o[1] = rest_height_pre(rb, nb, around6(-lx), around6(-ly), around6(lx + x), around6(ly + y));
    if (mh < 0) mh = 0.0;
    GeomC g{box, nullptr, nb};  // support / centre / strictly_inside read no density
    NodeC nd{lx, ly, mh, x, y, 1.0, 1.0};
    double cx, cy, cz;
    g.centre(nd, cx, cy, cz);
    double *rc = rects + (size_t)i * KSUP_MAX * 4;
    int ks = 0, direct = -1;
    for (int t = 0; t < nb && ks < KSUP_MAX; t++) {
        double r[4];
        if (!g.support(nd, t, r)) continue;
        for (int c = 0; c < 4; c++) rc[4 * ks + c] = r[c];
        if (direct < 0 && g.strictly_inside(cx, cy, r)) direct = ks;
        ks++;
    }
    o[2] = ks; o[4] = direct;
    double pip = -1;
    if (ks > 0 && fabs(mh) >= 1e-6) {
        double *px = scratch + (size_t)i * 24 * KSUP_MAX, *py = px + 4 * KSUP_MAX, *hx = py + 4 * KSUP_MAX, *hy = hx + 8 * KSUP_MAX;
        for (int s = 0; s < ks; s++) {
            const double x1 = rc[4 * s], y1 = rc[4 * s + 1], x2 = rc[4 * s + 2], y2 = rc[4 * s + 3];
            const double t1 = y1 * 1e-6, t2 = y2 * 1e-6;
            px[4 * s + 0] = x1 + t1; py[4 * s + 0] = y1;
            px[4 * s + 1] = x1 + t2; py[4 * s + 1] = y2;
            px[4 * s + 2] = x2 + t1; py[4 * s + 2] = y1;
            px[4 * s + 3] = x2 + t2; py[4 * s + 3] = y2;
        }
        const int m = hull_coords(px, py, 4 * ks, hx, hy);
        pip = pip_shrunk(hx, hy, 1, m, cx, cy);
    }
    o[3] = pip;
}
extern "C" int gu_root_c(const double *boxes, const int *nbox, const double *q, int n, double *out, double *rects, double *scratch) {
    if (n > 0) k_root_c<<<GRID(n)>>>(boxes, nbox, q, n, out, rects, scratch);
    FINISH();
}
extern "C" int gu_root_scratch_doubles() { return 24 * KSUP_MAX; }
