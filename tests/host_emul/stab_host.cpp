// TEST INFRASTRUCTURE — a HOST build of the device stability routine (csrc/pct_stability.cuh + pct_geom.cuh, compiled by g++ with the
// few CUDA intrinsics it uses shimmed) so that the `-m "not gpu"` tests can drive the very source the kernels compile against the CPU
// oracle / the reference's records: every real placement (stability_check<true>: load persistence in the edge pool) and every virtual
// feasibility check (stability_check<false>) of whole trajectories.  It mirrors what pct_apply_kernel does around the call
// (csrc/pct_discrete.cu: CSR slot of the new box, resting height, commit of the box and of the pool counters) and nothing else.
// What it does NOT cover: warp-level code, TMA staging, SASS — those are the GPU tests' business.  g++ -ffp-contract=off == nvcc -fmad=false.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>
#include <cstdlib>
using std::max;
using std::min;
static inline float __fdividef(float a, float b) { return a / b; }  // device: approximate; only a pre-filter whose verdict the exact path confirms
static inline int atomicCAS(int *p, int cmp, int val) { int o = *p; if (o == cmp) *p = val; return o; }
static inline int atomicExch(int *p, int v) { int o = *p; *p = v; return o; }
static inline void __threadfence_block() {}
static inline double __longlong_as_double(long long v) { double d; memcpy(&d, &v, 8); return d; }
static long long g_far_out = 0, g_walks = 0;  // statistics of the quick reject (sh_stats)
static long long g_stat[32];
#define PCT_STAT(i) g_stat[(i)]++
static double g_path_cur = 0, g_path_tot = 0, g_path_max = 0, g_path_fr[64];
#define PCT_PATH_VISIT(c) do { g_path_cur += (c); g_path_tot += (c); if (g_path_cur > g_path_max) g_path_max = g_path_cur; } while (0)
#define PCT_PATH_PUSH(d) (g_path_fr[(d)] = g_path_cur)
#define PCT_PATH_POP(d) (g_path_cur = g_path_fr[(d)])
static double g_last_path[3];  // the last continuation walk: total cost, cost of its longest root-to-leaf path, result
static long long g_pieces = 0;
static int g_use_v2 = 0;  // sh_use_v2: route the virtual checks through stab_virtual (the warp-convergent restatement used by the round-2 feasibility kernels)
#include <cuda_runtime.h>
#ifndef __noinline__
#define __noinline__ __attribute__((noinline))
#endif
#include "pct_stability.cuh"
#include "pct_pyhash.cuh"
#include "pct_geom.cuh"
#include "pct_geom_continuous.cuh"
#include "pct_support_graph.h"

using namespace pct;

struct StabHost {
    int setting, W, L, H, nb_holder;
    int n_box, n_edge, n_poly, flags;
    int16_t box[NB_MAX][6];
    double density[NB_MAX];
    uint8_t e_lower[EDGE_MAX + 1], e_next[EDGE_MAX + 1], first_in[NB_MAX], last_in[NB_MAX];
    uint16_t e_off[NB_MAX + 2], poly_off[NB_MAX + 2];
    Stack4 e_st[EDGE_MAX + 1];
    double poly[POLY_MAX][2];
    BigScratch big;
    int lock;
    // ALIAS variant (EdgePoolA): the reference's object semantics of the load entries
    int alias;
    Stack4 box_st[NB_MAX + 1];
    uint8_t e_upper[EDGE_MAX + 1];
    uint32_t e_alias[(EDGE_MAX + 32) / 32];
};

static EdgePool pool_of(StabHost *h) {
    return EdgePool{h->e_lower, h->e_next, h->e_off, h->first_in, h->last_in, h->e_st, h->e_st, h->n_edge, h->poly_off, &h->poly[0][0], &h->poly[0][0], h->n_poly};
}

extern "C" {
StabHost *sh_create(int setting, int W, int L, int H) {
    StabHost *h = new StabHost();
    memset(h, 0, sizeof *h);
    h->setting = setting; h->W = W; h->L = L; h->H = H; h->nb_holder = NB_MAX;
    return h;
}
void sh_set_holder(StabHost *h, int nb) { h->nb_holder = nb; }
void sh_destroy(StabHost *h) { delete h; }
void sh_set_alias(StabHost *h, int on) { h->alias = on; }
void sh_reset(StabHost *h) { h->n_box = 0; h->n_edge = 0; h->n_poly = 0; h->flags = 0; h->lock = 0; }
int sh_flags(StabHost *h) { return h->flags; }
int sh_n_boxes(StabHost *h) { return h->n_box; }

// Space.drop_box_virtual (D:space.py:393-433): feasibility of the oriented item (x, y, z) at (lx, ly); *mh_out = resting height
int sh_virtual(StabHost *h, int x, int y, int z, int lx, int ly, double density, int *mh_out) {
    const int mh = rest_height(h->box, 0, h->n_box, 1, lx, ly, lx + x, ly + y);
    if (mh_out) *mh_out = mh;
    g_last_path[0] = g_last_path[1] = 0;
    if (lx + x > h->W || ly + y > h->L) return 0;
    if (mh + z > h->H) return 0;
    if (h->setting == 2 || mh == 0) return 1;
    GeomD g{h->box, h->n_box, h->setting == 3 ? h->density : nullptr};
    NodeD root{lx, ly, mh, x, y, z, (double)(x * y * z) * density};
    EdgePool pool = pool_of(h);  // the read-only check knows snapshots only, in both semantics (like pct_feas_emit_kernel)
    int fl = 0;
    int ok;
    if (g_use_v2 == 1) {  // as pct_feas_emit_kernel calls it: supports from the fused resting-height scan
        int k; uint32_t pack; bool far_out;
        const int mh2 = rest_height_supports(h->box, h->n_box, lx, ly, lx + x, ly + y, k, pack, far_out);
        if (mh2 != mh) { h->flags |= 1 << 20; return -1; }
        if (far_out) { g_far_out++; return 0; }  // the kernel's integer quick reject
        g_walks++;
        ok = stab_virtual<GeomD>(g, root, k, pack, pool, &h->big, &h->lock, fl, true, 0xffffffffu);
    } else if (g_use_v2 == 3) {  // as the round-2 kernels run it: light prefix (pct_walk_light_kernel), then the continuation (pct_walk_kernel)
        int k; uint32_t pack; bool far_out;
        const int mh2 = rest_height_supports(h->box, h->n_box, lx, ly, lx + x, ly + y, k, pack, far_out);
        if (mh2 != mh) { h->flags |= 1 << 20; return -1; }
        if (far_out) { g_far_out++; return 0; }
        int node = NODE_NEW; Stack4 st{};
        ok = stab_light<GeomD>(g, root, k, pack, pool, node, st);
        if (ok == 2) {
            g_walks++;
            g_path_cur = g_path_tot = g_path_max = 0;
            ok = stab_virtual<GeomD>(g, root, k, pack, pool, &h->big, &h->lock, fl, true, 0xffffffffu, node, &st);
            g_last_path[0] = g_path_tot; g_last_path[1] = g_path_max; g_last_path[2] = ok;
        } else g_last_path[0] = g_last_path[1] = 0;
    } else if (g_use_v2 == 4) {  // fork-join form (pct_walk_fork_kernel): light prefix, then pieces from a queue, verdict = AND over the pieces
        int k; uint32_t pack; bool far_out;
        const int mh2 = rest_height_supports(h->box, h->n_box, lx, ly, lx + x, ly + y, k, pack, far_out);
        if (mh2 != mh) { h->flags |= 1 << 20; return -1; }
        if (far_out) { g_far_out++; return 0; }
        int node = NODE_NEW; Stack4 st{};
        ok = stab_light<GeomD>(g, root, k, pack, pool, node, st);
        if (ok == 2) {
            g_walks++;
            std::vector<WalkPiece> q;
            q.push_back(WalkPiece{0u, (uint8_t)node, (uint8_t)EDGE_NIL, 0, 0, st.cx, st.cy, st.m});
            struct Fork {
                std::vector<WalkPiece> *q;
                void operator()(int child, int skip, double vx, double vy, double vm) { q->push_back(WalkPiece{0u, (uint8_t)child, (uint8_t)skip, 1, 0, vx, vy, vm}); }
            } fork{&q};
            ok = 1;
            double longest = 0, total = 0;
            for (size_t i = 0; i < q.size(); i++) {  // every piece runs (the kernel runs them concurrently)
                const WalkPiece pc = q[i];
                g_path_cur = g_path_tot = g_path_max = 0;
                if (!stab_piece<GeomD>(g, root, k, pack, pool, &h->big, &h->lock, fl, (int)pc.node, (int)pc.kind, (int)pc.skip, pc.a, pc.b, pc.c, fork)) ok = 0;
                total += g_path_tot; if (g_path_tot > longest) longest = g_path_tot;
            }
            g_last_path[0] = total; g_last_path[1] = longest; g_last_path[2] = ok; g_pieces += (long long)q.size();
        }
    } else if (g_use_v2 == 2) ok = stab_virtual<GeomD>(g, root, -1, 0, pool, &h->big, &h->lock, fl, true, 0xffffffffu);
    else ok = stability_check<false, GeomD>(g, root, pool, &h->big, &h->lock, 0, fl) != 0;
    h->flags |= fl;
    return ok;
}
void sh_use_v2(int on) { g_use_v2 = on; }
double sh_around6(double v) { return around6(v); }
long long sh_hash_double(double v, int loop) { return (long long)(loop ? hash_double_loop(v) : hash_double(v)); }  // _Py_HashDouble: integer restatement / frexp loop  // the device's np.around(v, 6) (fast division by 1e6, pct_geom_continuous.cuh)
void sh_stats(long long *out2) { out2[0] = g_far_out; out2[1] = g_walks; }
long long sh_pieces() { return g_pieces; }
void sh_last_path(double *out3) { memcpy(out3, g_last_path, sizeof g_last_path); }
void sh_stats_visits(long long *out32) { memcpy(out32, g_stat, sizeof g_stat); }

// Space.drop_box (D:space.py:347-391) as pct_apply_kernel performs it: 1 = placed, 0 = rejected (the episode ends)
int sh_place(StabHost *h, int x, int y, int z, int lx, int ly, double density) {
    const int n0 = h->n_box;  // may equal the holder size: the kernel (like the reference) runs the check first and rejects the box afterwards
    h->e_off[n0] = (uint16_t)h->n_edge;
    h->poly_off[n0] = (uint16_t)h->n_poly;
    if (n0 < NB_MAX) h->first_in[n0] = EDGE_NIL;
    const int mh = rest_height(h->box, 0, n0, 1, lx, ly, lx + x, ly + y);
    if (lx + x > h->W || ly + y > h->L) return 0;
    if (mh + z > h->H) return 0;
    if (h->setting != 2 && mh != 0) {
        GeomD g{h->box, n0, h->setting == 3 ? h->density : nullptr};
        NodeD root{lx, ly, mh, x, y, z, (double)(x * y * z) * density};
        EdgePoolA pool;
        static_cast<EdgePool &>(pool) = pool_of(h);
        pool.box_st = h->box_st; pool.e_upper = h->e_upper; pool.e_alias = h->e_alias;
        int fl = 0;
        const int res = h->alias ? stability_check<true, GeomD, true>(g, root, pool, &h->big, &h->lock, n0, fl)
                                 : stability_check<true, GeomD>(g, root, pool, &h->big, &h->lock, n0, fl);
        if (h->alias && !res && !getenv("PCT_HOST_EMUL_NO_SYNC")) alias_sync_loads(pool);  // as the ALIAS instantiation of the apply kernel does (switch: sensitivity test)
        h->n_edge = pool.n;
        h->n_poly = pool.n_poly;
        h->flags |= fl;
        if (!res) return 0;
    }
    if (n0 >= h->nb_holder) return 0;  // PCT_FLAG_BOX_OVERFLOW in the kernel (IndexError in the reference, D:space.py:385)
    int16_t *b = h->box[n0];
    b[0] = (int16_t)lx; b[1] = (int16_t)ly; b[2] = (int16_t)mh; b[3] = (int16_t)(lx + x); b[4] = (int16_t)(ly + y); b[5] = (int16_t)(mh + z);
    h->density[n0] = density;
    h->n_box = n0 + 1;
    h->e_off[n0 + 1] = (uint16_t)h->n_edge;
    h->poly_off[n0 + 1] = (uint16_t)h->n_poly;
    return 1;
}
}


// ---- continuous domain (GeomC; what pctc_apply_kernel / pctc_feas_emit_kernel do around the routine, csrc/pct_continuous.cu) ----------
struct StabHostC {
    int setting, nb_holder;
    double W, L, H;
    int n_box, n_edge, n_poly, flags;
    double box[NB_MAX][6];  // lx, ly, lz, x, y, z
    double den[NB_MAX];
    uint8_t e_lower[EDGE_MAX + 1], e_next[EDGE_MAX + 1], first_in[NB_MAX], last_in[NB_MAX];
    uint16_t e_off[NB_MAX + 2], poly_off[NB_MAX + 2];
    Stack4 e_st[EDGE_MAX + 1];
    double poly[POLY_MAX][2];
    BigScratch big;
    int lock, alias;
    Stack4 box_st[NB_MAX + 1];
    uint8_t e_upper[EDGE_MAX + 1];
    uint32_t e_alias[(EDGE_MAX + 32) / 32];
};
static EdgePool pool_of(StabHostC *h) {
    return EdgePool{h->e_lower, h->e_next, h->e_off, h->first_in, h->last_in, h->e_st, h->e_st, h->n_edge, h->poly_off, &h->poly[0][0], &h->poly[0][0], h->n_poly};
}

extern "C" {
StabHostC *shc_create(int setting, double W, double L, double H) {
    StabHostC *h = new StabHostC();
    memset(h, 0, sizeof *h);
    h->setting = setting; h->W = W; h->L = L; h->H = H; h->nb_holder = NB_MAX;
    return h;
}
void shc_set_holder(StabHostC *h, int nb) { h->nb_holder = nb; }
void shc_destroy(StabHostC *h) { delete h; }
void shc_set_alias(StabHostC *h, int on) { h->alias = on; }
void shc_reset(StabHostC *h) { h->n_box = 0; h->n_edge = 0; h->n_poly = 0; h->flags = 0; h->lock = 0; }
int shc_flags(StabHostC *h) { return h->flags; }

// pctc_feas_emit_kernel's feasibility of one candidate tuple (xs, ys, zs, xe, ye, ze)   (C:bin3D.py:134-137, C:space.py:380-425)
int shc_virtual(StabHostC *h, const double t6[6], double density) {
    const double x = t6[3] - t6[0], y = t6[4] - t6[1], z = t6[5] - t6[2], lx = t6[0], ly = t6[1];
    bool chk = !(lx + x - 1e-6 > h->W || ly + y - 1e-6 > h->L) && !(lx + 1e-6 < 0 || ly + 1e-6 < 0);
    double mh = rest_height_c(h->box, 0, h->n_box, 1, lx, ly, lx + x, ly + y);
    if (mh < 0) mh = 0.0;
    if (mh + z - 1e-6 > h->H) chk = false;
    if (!chk) return 0;
    if (h->setting == 2 || fabs(mh) < 1e-6) return 1;
    GeomC g{h->box, h->den, h->n_box};
    NodeC root{lx, ly, mh, x, y, z, x * y * z * density};
    EdgePool pool = pool_of(h);  // the read-only check knows snapshots only, in both semantics (like pct_feas_emit_kernel)
    int fl = 0;
    int ok;
    if (g_use_v2 == 3 || g_use_v2 == 4) {  // as the round-2 continuous kernels run it: supports + quick reject (classification), light prefix, continuation (4: fork-join pieces)
        int k = 0; uint32_t pack = 0; double r[4], X1 = 0, Y1 = 0, X2 = 0, Y2 = 0;
        for (int t = 0; t < h->n_box; t++) {
            if (!g.support(root, t, r)) continue;
            if (k == 0) { X1 = r[0]; Y1 = r[1]; X2 = r[2]; Y2 = r[3]; }
            else { X1 = fmin(X1, r[0]); Y1 = fmin(Y1, r[1]); X2 = fmax(X2, r[2]); Y2 = fmax(Y2, r[3]); }
            if (k < 4) pack |= (uint32_t)t << (8 * k);
            k++;
        }
        const double margin = 2e-6 * (1.0 + fmax(h->W, h->L)), cx = lx + x * 0.5, cy = ly + y * 0.5;
        if (k > 0 && (cx < X1 - margin || cx > X2 + margin || cy < Y1 - margin || cy > Y2 + margin)) { g_far_out++; return 0; }
        int node = NODE_NEW; Stack4 st{};
        ok = stab_light<GeomC>(g, root, k, pack, pool, node, st);
        if (ok == 2 && g_use_v2 == 4) {
            g_walks++;
            std::vector<WalkPiece> q;
            q.push_back(WalkPiece{0u, (uint8_t)node, (uint8_t)EDGE_NIL, 0, 0, st.cx, st.cy, st.m});
            struct Fork {
                std::vector<WalkPiece> *q;
                void operator()(int child, int skip, double vx, double vy, double vm) { q->push_back(WalkPiece{0u, (uint8_t)child, (uint8_t)skip, 1, 0, vx, vy, vm}); }
            } fork{&q};
            ok = 1;
            for (size_t i = 0; i < q.size(); i++) {
                const WalkPiece pc = q[i];
                if (!stab_piece<GeomC>(g, root, k, pack, pool, &h->big, &h->lock, fl, (int)pc.node, (int)pc.kind, (int)pc.skip, pc.a, pc.b, pc.c, fork)) ok = 0;
            }
        } else if (ok == 2) { g_walks++; ok = stab_virtual<GeomC>(g, root, k, pack, pool, &h->big, &h->lock, fl, true, 0xffffffffu, node, &st); }
    } else ok = g_use_v2 ? stab_virtual<GeomC>(g, root, -1, 0, pool, &h->big, &h->lock, fl, true, 0xffffffffu)
                         : (int)(stability_check<false, GeomC>(g, root, pool, &h->big, &h->lock, 0, fl) != 0);
    h->flags |= fl;
    return ok;
}

// pctc_apply_kernel on a 9-float leaf row: LeafNode2Action (C:bin3D.py:151-167) + Space.drop_box (C:space.py:329-376); 1 = placed
int shc_place_row(StabHostC *h, const double a[6], const double nb[3], double density) {
    double lx = 0, ly = 0, x = nb[0], y = nb[1], z = nb[2], s = 0;
    for (int t = 0; t < 6; t++) s += a[t];
    if (s != 0) {
        x = around6(a[3] - a[0]);
        y = around6(a[4] - a[1]);
        int rec[3] = {0, 1, 2}, n = 3;
        for (int i = 0; i < n; i++)
            if (fabs(x - nb[rec[i]]) < 1e-6) { for (int u = i; u < n - 1; u++) rec[u] = rec[u + 1]; n--; break; }
        for (int i = 0; i < n; i++)
            if (fabs(y - nb[rec[i]]) < 1e-6) { for (int u = i; u < n - 1; u++) rec[u] = rec[u + 1]; n--; break; }
        z = nb[rec[0]];
        lx = a[0]; ly = a[1];
    }
    lx = around6(lx); ly = around6(ly);
    const int n0 = h->n_box;
    bool ok = !(lx + x - 1e-6 > h->W || ly + y - 1e-6 > h->L) && !(lx + 1e-6 < 0 || ly + 1e-6 < 0);
    h->e_off[n0] = (uint16_t)h->n_edge; h->poly_off[n0] = (uint16_t)h->n_poly; if (n0 < NB_MAX) h->first_in[n0] = EDGE_NIL;
    if (!ok) return 0;
    double mh = rest_height_c(h->box, 0, n0, 1, lx, ly, lx + x, ly + y);
    const double max_h = mh < 0 ? 0.0 : mh;
    if (max_h + z - 1e-6 > h->H) return 0;
    if (h->setting != 2 && !(fabs(max_h) < 1e-6)) {
        GeomC g{h->box, h->den, n0};
        NodeC root{lx, ly, max_h, x, y, z, x * y * z * density};
        EdgePoolA pool;
        static_cast<EdgePool &>(pool) = pool_of(h);
        pool.box_st = h->box_st; pool.e_upper = h->e_upper; pool.e_alias = h->e_alias;
        int fl = 0;
        const int res = h->alias ? stability_check<true, GeomC, true>(g, root, pool, &h->big, &h->lock, n0, fl)
                                 : stability_check<true, GeomC>(g, root, pool, &h->big, &h->lock, n0, fl);
        if (h->alias && !res && !getenv("PCT_HOST_EMUL_NO_SYNC")) alias_sync_loads(pool);  // as the ALIAS instantiation of the apply kernel does (switch: sensitivity test)
        h->n_edge = pool.n; h->n_poly = pool.n_poly; h->flags |= fl;
        if (!res) return 0;
    }
    if (n0 >= h->nb_holder) return 0;  // PCT_FLAG_BOX_OVERFLOW in the kernel
    double *b = h->box[n0];
    b[0] = lx; b[1] = ly; b[2] = max_h; b[3] = x; b[4] = y; b[5] = z;
    h->den[n0] = density;
    h->n_box = n0 + 1;
    h->e_off[n0 + 1] = (uint16_t)h->n_edge; h->poly_off[n0 + 1] = (uint16_t)h->n_poly;
    return 1;
}
}

// The support graph the pools hold, through the decoder the C ABI runs on the device records (csrc/pct_support_graph.h): 1 = decoded, 0 = finding in err.
// sh_pool_field: address of one pool array (0 e_st, 1 e_next, 2 e_alias), so a test can damage a record and see the decoder / the comparison name it.
template <class H>
static int graph_of(H *h, pct_support_graph *out, char *err, int cap) {
    const GraphRecord r{h->n_box, h->n_edge, h->n_poly, h->e_off, h->poly_off, h->e_lower, h->e_next, h->first_in, h->last_in, h->e_st, &h->poly[0][0],
                        h->alias ? h->box_st : nullptr, h->alias ? h->e_upper : nullptr, h->alias ? h->e_alias : nullptr};
    return decode_support_graph(r, out, err, (size_t)cap) ? 1 : 0;
}
template <class H>
static void *field_of(H *h, int which) { return which == 0 ? (void *)h->e_st : which == 1 ? (void *)h->e_next : (void *)h->e_alias; }
extern "C" {
int sh_support_graph(StabHost *h, pct_support_graph *out, char *err, int cap) { return graph_of(h, out, err, cap); }
int shc_support_graph(StabHostC *h, pct_support_graph *out, char *err, int cap) { return graph_of(h, out, err, cap); }
void *sh_pool_field(StabHost *h, int which) { return field_of(h, which); }
void *shc_pool_field(StabHostC *h, int which) { return field_of(h, which); }
}
