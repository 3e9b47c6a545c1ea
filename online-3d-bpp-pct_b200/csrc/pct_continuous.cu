// Continuous PCT environment (pct_envs/PctContinuous0 in the reference, "C:" below): batched reset / step for sm_90a.
//
// Same three-kernel pipeline as the discrete domain (apply / candidates / feasibility+emit) and the same stability
// routine (pct_stability.cuh) instantiated with a float64 geometry policy that carries the reference's 1e-6
// tolerances and 6-decimal roundings.  This first version keeps the per-env record in HBM (no TMA staging): it is the
// correctness path for BASELINE config 4; the discrete kernels are the tuned ones.
//
// Reference behaviour restated:
//   PackingContinuous.step / reset / cur_observation / get_possible_position / LeafNode2Action   C:bin3D.py:69-207
//   Space.interSect2D / drop_box / drop_box_virtual / check_box                                   C:space.py:305-439
//   Space.interSectEMS3D / GENEMS / Difference / EliminateInscribedEMS / EMSPoint                 C:space.py:441-568
// Parity contract (see oracle/pct_oracle_continuous.c): float64 leaf rows as actions; float32 rows are widened.
#include "pct_common.cuh"
#include "pct_stability.cuh"
#include "pct_kernels.h"
#include "pct_geom_continuous.cuh"
#include "pct_walks.cuh"
#include "pct_continuous.cuh"
#include "pct_cand_c.cuh"
#include "pct_block.cuh"
#include "pct_draw.cuh"

namespace pct {

// around6, NodeC / GeomC (geometry policy of the stability routine), rest_height_c, rest_height_pre: pct_geom_continuous.cuh
// rot_dims_c, cand_tuple, hash_double_call, cand_hash_c, cand_equal and the set emulation (PCTC_CANDIDATES_BODY): pct_cand_c.cuh

__device__ __noinline__ void reset_space_c(CEnv *ev, const CParams &p, int e, int lane) {
    if (lane == 0) {
        CHdr &h = ev->h;
        h.n_box = 0; h.n_ems = 1; h.n_leaf = 0; h.flags = 0; h.n_edge = 0; h.n_poly = 0; h.vol_sum = 0; h.ep_len = 0; h.ep_reward = 0;
        ev->ems[0][0] = 0; ev->ems[0][1] = 0; ev->ems[0][2] = 0; ev->ems[0][3] = p.W; ev->ems[0][4] = p.L; ev->ems[0][5] = p.H;
        if (p.traj_len > 0 && h.draw_pos % p.traj_len) h.draw_pos += p.traj_len - h.draw_pos % p.traj_len;
        draw_item_c(p, e, h);
    }
    __syncwarp();
}

// GENEMS (C:space.py:441-528): same ballot / scan compaction as the discrete kernel, float64 with rounded intersections
constexpr int CE_STAGE = 128;  // intermediate EMS entries staged in shared memory for the inscribed-EMS purge (6 KB per warp)
__device__ __noinline__ int genems_warp_c(CEnv *ev, const int n0, const double loc[6], double lb, int lane, int &flags, double (*stage)[6]) {
    double (*ems)[6] = ev->ems, (*tmp)[6] = ev->ems_tmp;
    const int nch = (n0 + 31) >> 5;
    const double itn[6] = {-loc[0], -loc[1], -loc[2], loc[3], loc[4], loc[5]};
    int off = 0;
#pragma unroll 1
    for (int pass = 0; pass < 2; pass++) {
#pragma unroll 1
        for (int c = 0; c < nch; c++) {
            const int i = c * 32 + lane;
            bool inter = false;
            double it[6], m[6];
            if (i < n0) {
#pragma unroll
                for (int t = 0; t < 6; t++) m[t] = ems[i][t];
#pragma unroll
                for (int t = 0; t < 6; t++) it[t] = around6(fmin(itn[t], t < 3 ? -m[t] : m[t]));
                inter = (it[0] + it[3] > 0) && (it[1] + it[4] > 0) && (it[2] + it[5] > 0);
            }
            if (pass == 0) {  // survivors keep their order
                const bool keep = i < n0 && !inter;
                const uint32_t bm = __ballot_sync(FULL, keep);
                if (keep) {
                    const int p = off + __popc(bm & ((1u << lane) - 1));
#pragma unroll
                    for (int t = 0; t < 6; t++) tmp[p][t] = m[t];
                }
                off += __popc(bm);
            } else {  // children: left, right, front, back, top (Difference, :490-502)
                uint32_t cm = 0;
                const double x3 = -it[0], y3 = -it[1], x4 = it[3], y4 = it[4], z4 = it[5];
                if (inter) {
                    const bool ux = m[3] - m[0] + 1e-6 >= lb, uy = m[4] - m[1] + 1e-6 >= lb, uz = m[5] - m[2] + 1e-6 >= lb;
                    if (x3 - m[0] + 1e-6 >= lb && uy && uz) cm |= 1;
                    if (m[3] - x4 + 1e-6 >= lb && uy && uz) cm |= 2;
                    if (ux && y3 - m[1] + 1e-6 >= lb && uz) cm |= 4;
                    if (ux && m[4] - y4 + 1e-6 >= lb && uz) cm |= 8;
                    if (ux && uy && m[5] - z4 + 1e-6 >= lb) cm |= 16;
                }
                const int cnt = __popc(cm);
                const int incl = warp_incl_scan(cnt, lane);
                int p = off + incl - cnt;
#pragma unroll 1
                for (int ch = 0; ch < 5 && cm; ch++) {
                    if (!(cm & (1u << ch))) continue;
                    double q[6] = {m[0], m[1], m[2], m[3], m[4], m[5]};
                    if (ch == 0) q[3] = x3; else if (ch == 1) q[0] = x4; else if (ch == 2) q[4] = y3; else if (ch == 3) q[1] = y4; else q[2] = z4;
                    if (p < CE_TMP) {
#pragma unroll
                        for (int t = 0; t < 6; t++) tmp[p][t] = q[t];
                    } else flags |= PCT_FLAG_EMS_OVERFLOW;
                    p++;
                }
                off += __shfl_sync(FULL, incl, 31);
            }
        }
    }
    flags = __reduce_or_sync(FULL, flags);
    const int n = off < CE_TMP ? off : CE_TMP;
    __syncwarp();
    // EliminateInscribedEMS (C:space.py:505-528): the O(n^2) containment test read every candidate container b from the env record in global memory
    // (the line with the most stall samples in a profile of this kernel); the intermediate list is staged in shared memory first
    // (lists longer than CE_STAGE entries — not seen on the BASELINE streams — keep reading the record).
    const bool staged = n <= CE_STAGE;
    // Every EMS coordinate is a 6-decimal value (the container's corners or an np.around(.., 6) result), so v -> rint(v * 1e6) is an order-preserving
    // bijection onto integers; for bins up to 1.048575 they fit 20 bits and the six comparisons of a containment test become two 64-bit subtractions on
    // packed fields with guard bits (the discrete kernel's trick).  Any coordinate that is not
    // exactly such a value (checked per entry) sends the whole list through the float64 comparisons.
    constexpr uint64_t GUARD = (1ull << 20) | (1ull << 41) | (1ull << 62);
    uint64_t *pk = (uint64_t *)&stage[0][0];
    bool packed = staged;
    if (packed) {
        bool good = true;
#pragma unroll 1
        for (int i = lane; i < n; i += 32) {
            uint64_t w2[2] = {0, 0};
#pragma unroll
            for (int t = 0; t < 6; t++) {
                const double v = tmp[i][t], k = rint(v * 1e6);
                good = good && k >= 0.0 && k < 1048576.0 && around6(v) == v;
                w2[t / 3] |= (uint64_t)(long long)k << (21 * (t % 3));
            }
            pk[2 * i] = w2[0]; pk[2 * i + 1] = w2[1];
        }
        packed = __all_sync(FULL, good);
        __syncwarp();
    }
    if (staged && !packed)
        for (int t = lane; t < n * 6; t += 32) (&stage[0][0])[t] = (&tmp[0][0])[t];
    __syncwarp();
    const double (*src)[6] = (staged && !packed) ? stage : tmp;
    int w = 0;
    const int nch2 = (n + 31) >> 5;
#pragma unroll 1
    for (int c = 0; c < nch2; c++) {
        const int i = c * 32 + lane;
        bool keep = false;
        double a[6];
        if (i < n) {
#pragma unroll
            for (int t = 0; t < 6; t++) a[t] = src[i][t];
            int hit = 0;
            if (packed) {
                const uint64_t alo = pk[2 * i] | GUARD, ahi = pk[2 * i + 1];
#pragma unroll 4
                for (int j = 0; j < n; j++) {
                    const ulonglong2 b = *(const ulonglong2 *)(pk + 2 * j);
                    hit |= (int)(j != i && (((alo - b.x) & ((b.y | GUARD) - ahi) & GUARD) == GUARD));
                }
            } else {
#pragma unroll 2
                for (int j = 0; j < n; j++) {
                    const double *b = src[j];
                    hit |= (int)(j != i && a[0] >= b[0] && a[1] >= b[1] && a[2] >= b[2] && a[3] <= b[3] && a[4] <= b[4] && a[5] <= b[5]);
                }
            }
            keep = !hit;
        }
        const uint32_t bm = __ballot_sync(FULL, keep);
        if (keep) {
            const int p = w + __popc(bm & ((1u << lane) - 1));
            if (p < CE_MAX) {
#pragma unroll
                for (int t = 0; t < 6; t++) ems[p][t] = a[t];
            }
        }
        w += __popc(bm);
    }
    if (w > CE_MAX) { flags |= PCT_FLAG_EMS_OVERFLOW; w = CE_MAX; }
    __syncwarp();
    return w;
}

// ================= K1: apply =================
// ALIAS variant (the default; PCT_B200_ALIAS=0 selects the snapshot kernels): the reference's object semantics of the load entries (EdgePoolA,
// DESIGN.md section 3 (b)); per-env state through CParams::aux.

// SEL: the selected launch (EnvSel, pct_kernels.h)
template <bool STAB, bool ALIAS = false, bool SEL = false>
__global__ void __launch_bounds__(64) pctc_apply_kernel(const ParamsT<CParams, SEL> p) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int e = blockIdx.x * 2 + warp;
    if constexpr (SEL) e = sel_env(p.sel, p.n_envs, e);
    if (e >= p.n_envs || (SEL && e < 0)) return;
    __shared__ int lock_s[2];
    __shared__ __align__(16) double ems_stage[2][CE_STAGE][6];
    int *lock = &lock_s[warp];
    static_assert(sizeof(StabScratch) <= sizeof(double) * CE_STAGE * 6, "the descent's scratch fits the EMS stage");
    StabScratch *scr = (StabScratch *)&ems_stage[warp][0][0];  // the descent's working arrays: aliased onto the EMS stage, which only GENEMS (after the descent) uses
    CEnv *ev = p.env + e;
    CHdr &h = ev->h;
    if (p.ready) pdl_launch_dependents();
    if (lane == 0) *lock = 0;
    float reward = 0.f;
    int done = 0;
    pct_step_info info{};
    if (p.mode == 0) {
        const int64_t dp = p.keep_draw ? h.draw_pos : 0;
        __syncwarp();
        if (lane == 0) h.draw_pos = dp;
        reset_space_c(ev, p, e, lane);
    } else {
        const double nb0 = h.next_box[0], nb1 = h.next_box[1], nb2 = h.next_box[2], den0 = h.next_den;
        const int n_box0 = h.n_box, n_leaf0 = h.n_leaf, flags0 = h.flags, n_ems0 = h.n_ems;
        __syncwarp();
        // ---- LeafNode2Action (C:bin3D.py:151-167) ----
        double lx = 0, ly = 0, x = nb0, y = nb1, z = nb2;
        {
            double a[6] = {0, 0, 0, 0, 0, 0}, s = 0;
            bool zero = true;
            if (p.leaf_idx) {
                const int k = p.leaf_idx[e];
                if (k >= 0 && k < n_leaf0) {
                    zero = false;
                    for (int t = 0; t < 6; t++) a[t] = ev->leaf[k][t];
                }
            } else {
                for (int t = 0; t < 6; t++) {
                    a[t] = p.action_f64 ? ((const double *)p.actions)[(size_t)e * 9 + t] : (double)((const float *)p.actions)[(size_t)e * 9 + t];
                    s += a[t];
                }
                zero = (s == 0);
            }
            if (!zero) {
                x = around6(a[3] - a[0]);
                y = around6(a[4] - a[1]);
                const double nb[3] = {nb0, nb1, nb2};
                int rec[3] = {0, 1, 2}, n = 3;
                for (int i = 0; i < n; i++)
                    if (fabs(x - nb[rec[i]]) < 1e-6) { for (int u = i; u < n - 1; u++) rec[u] = rec[u + 1]; n--; break; }
                for (int i = 0; i < n; i++)
                    if (fabs(y - nb[rec[i]]) < 1e-6) { for (int u = i; u < n - 1; u++) rec[u] = rec[u + 1]; n--; break; }
                z = nb[rec[0]];
                lx = a[0]; ly = a[1];
            }
        }
        lx = around6(lx); ly = around6(ly);  // C:bin3D.py:173
        // ---- Space.drop_box (C:space.py:329-376) ----
        bool ok = !(lx + x - 1e-6 > p.W || ly + y - 1e-6 > p.L) && !(lx + 1e-6 < 0 || ly + 1e-6 < 0);
        double max_h = 0;
        if (lane == 0) { ev->e_off[n_box0] = (uint16_t)h.n_edge; ev->poly_off[n_box0] = (uint16_t)h.n_poly; if (n_box0 < NB_MAX) ev->first_in[n_box0] = EDGE_NIL; }
        __syncwarp();
        if (ok) {
            double mh = rest_height_c(ev->box, lane, n_box0, 32, lx, ly, lx + x, ly + y);
#pragma unroll
            for (int d = 16; d; d >>= 1) mh = fmax(mh, __shfl_xor_sync(FULL, mh, d));
            max_h = mh < 0 ? 0.0 : mh;
            if (max_h + z - 1e-6 > p.H) ok = false;
            else if (STAB && !(fabs(max_h) < 1e-6)) {
                int res = 0;
                if (lane == 0) {
                    int fl = 0;
                    GeomC g{ev->box, ev->den, n_box0};
                    NodeC root{lx, ly, max_h, x, y, z, x * y * z * den0};
                    if constexpr (ALIAS) {
                        EdgePoolA pool;
                        static_cast<EdgePool &>(pool) = EdgePool{ev->e_lower, ev->e_next, ev->e_off, ev->first_in, ev->last_in, ev->e_st, ev->e_st, h.n_edge,
                                                                 ev->poly_off, &ev->poly[0][0], &ev->poly[0][0], h.n_poly};
                        DEnvAux *ax = p.aux + e;
                        pool.box_st = ax->box_st; pool.e_upper = ax->e_upper; pool.e_alias = ax->e_alias;
                        res = stability_check<true, GeomC, true>(g, root, pool, &ev->big, lock, n_box0, fl, nullptr, scr);
                        if (!res) alias_sync_loads(pool);
                        h.n_edge = pool.n; h.n_poly = pool.n_poly;
                    } else {
                    EdgePool pool{ev->e_lower, ev->e_next, ev->e_off, ev->first_in, ev->last_in, ev->e_st, ev->e_st, h.n_edge,
                                  ev->poly_off, &ev->poly[0][0], &ev->poly[0][0], h.n_poly};
                    res = stability_check<true, GeomC>(g, root, pool, &ev->big, lock, n_box0, fl, nullptr, scr);
                    h.n_edge = pool.n; h.n_poly = pool.n_poly;
                    }
                    h.flags |= fl;
                }
                __syncwarp();
                ok = __shfl_sync(FULL, res, 0) != 0;
            }
            if (ok && n_box0 >= p.nb) { ok = false; if (lane == 0) h.flags |= PCT_FLAG_BOX_OVERFLOW; }
        }
        __syncwarp();
        const double binvol = p.W * p.L * p.H;
        if (ok) {
            if (lane == 0) {
                double *b = ev->box[n_box0];
                b[0] = lx; b[1] = ly; b[2] = max_h; b[3] = x; b[4] = y; b[5] = z;
                ev->den[n_box0] = den0;
                h.n_box = n_box0 + 1;
                h.vol_sum += x * y * z;
                ev->e_off[n_box0 + 1] = (uint16_t)h.n_edge; ev->poly_off[n_box0 + 1] = (uint16_t)h.n_poly;
            }
            __syncwarp();
            int fl = 0;
            const double loc[6] = {lx, ly, max_h, around6(lx + x), around6(ly + y), around6(max_h + z)};  // C:bin3D.py:191-194
            const int n_ems = genems_warp_c(ev, n_ems0, loc, p.low_bound, lane, fl, ems_stage[warp]);
            const double rw = (nb0 * nb1 * nb2) / binvol * 10;
            reward = (float)rw;
            info.counter = n_box0 + 1;
            info.flags = flags0 | fl;
            if (lane == 0) {
                h.n_ems = n_ems; h.flags |= fl; h.ep_len++; h.ep_reward += rw;
                draw_item_c(p, e, h);
            }
            __syncwarp();
        } else {
            done = 1;
            info.counter = n_box0;
            info.flags = h.flags;
            info.ratio = (float)(h.vol_sum / binvol);
            info.ep_reward = (float)h.ep_reward;
            info.ep_len = h.ep_len + 1;
            __syncwarp();
            if (!p.no_auto_reset) reset_space_c(ev, p, e, lane);
        }
    }
    __syncwarp();
    if (lane == 0) {
        if (p.reward) p.reward[e] = reward;
        if (p.done) p.done[e] = (uint8_t)done;
        if (p.info) p.info[e] = info;
        if (p.ready) env_publish(p.ready + e, p.epoch);
    }
}

// ================= K2: candidates in CPython-set order (C:space.py:531-568) =================

template <bool SEL = false>
__global__ void __launch_bounds__(32) pctc_candidates_kernel(const ParamsT<CParams, SEL> p) {
    __shared__ uint32_t tabA[CC_TAB], tabB[512];
    __shared__ uint64_t stg_h[32], rs_h[32];  // staging area kept in the layout; PCTC_CANDIDATES_BODY does not use it
    __shared__ uint32_t rs_c[32];
    __shared__ uint16_t stg_c[32];
    const int lane = threadIdx.x;
    int e = blockIdx.x;
    if constexpr (SEL) {
        e = sel_env(p.sel, p.n_envs, e);
        if (e < 0) return;
    }
    CEnv *ev = p.env + e;
    int fl = 0;
    if (p.ready) {  // overlapped mode: wait for the apply kernel's hand-over of THIS env
        pdl_launch_dependents();
        if (lane == 0 && !env_wait(p.ready + e, p.epoch)) fl = PCT_FLAG_SYNC_TIMEOUT;
        fl = __shfl_sync(FULL, fl, 0);
    }
    const CHdr &h = ev->h;
    const double nb[3] = {h.next_box[0], h.next_box[1], h.next_box[2]};
    const int R = p.setting == 2 ? 6 : 2, n_ems = h.n_ems;
    PCTC_CANDIDATES_BODY
    if (p.walk.walkq) {
        // ---- classify (round 2): drop_box_virtual's bounds / resting height (C:space.py:380-398) on pre-rounded box rectangles, supports + exact
        // quick reject for the placements that rest on boxes; the stability walks of all envs go to one pool (pctc_walk_light / pctc_walk kernels) ----
        __shared__ double rb[NB_MAX][5];
        const int n_box = h.n_box, nl = p.nl;
        const bool stab = p.setting != 2;
        for (int t = lane; t < n_box; t += 32) {
            const double *b = ev->box[t];
            rb[t][0] = around6(-b[0]); rb[t][1] = around6(-b[1]); rb[t][2] = around6(b[0] + b[3]); rb[t][3] = around6(b[1] + b[4]);
            rb[t][4] = b[2] + b[5];
        }
        __syncwarp();
        const uint32_t lt = (1u << lane) - 1;
        const double margin = 2e-6 * (1.0 + fmax(p.W, p.L));  // the support polygon lies inside the contact rectangles' bounding box up to the 1e-6 * y perturbation
        int pos = 0, nf = 0, n_walk = 0;
#pragma unroll 1
        while (pos < cnt && nf < nl) {
            const int c = pos + lane;
            bool feas = false, pend = false;
            int k = 0;
            uint32_t pack = 0;
            uint16_t code = 0;
            double mh = 0;
            if (c < cnt) {
                code = ev->cand[c];
                double t6[6];
                cand_tuple(code, ev->ems, nb, t6);
                const double x = t6[3] - t6[0], y = t6[4] - t6[1], z = t6[5] - t6[2], lx = t6[0], ly = t6[1];
                bool chk = !(lx + x - 1e-6 > p.W || ly + y - 1e-6 > p.L) && !(lx + 1e-6 < 0 || ly + 1e-6 < 0);
                const double c0 = around6(-lx), c1 = around6(-ly), c2 = around6(lx + x), c3 = around6(ly + y);
                mh = rest_height_pre(rb, n_box, c0, c1, c2, c3);
                if (mh < 0) mh = 0.0;
                if (mh + z - 1e-6 > p.H) chk = false;
                if (!chk) feas = false;
                else if (!stab || fabs(mh) < 1e-6) feas = true;
                else {
                    // supports = GeomC::support(root, t): top within 1e-6 of the resting height and a positive rounded intersection (C:space.py:350-359)
                    double X1 = 0, Y1 = 0, X2 = 0, Y2 = 0;
#pragma unroll 1
                    for (int t = 0; t < n_box; t++) {
                        const double *b = rb[t];
                        if (!(fabs(b[4] - mh) < 1e-6)) continue;
                        const double i0 = fmin(c0, b[0]), i1 = fmin(c1, b[1]), i2 = fmin(c2, b[2]), i3 = fmin(c3, b[3]);
                        if (!((i0 + i2 > 0) && (i1 + i3 > 0))) continue;
                        if (k == 0) { X1 = -i0; Y1 = -i1; X2 = i2; Y2 = i3; }
                        else { X1 = fmin(X1, -i0); Y1 = fmin(Y1, -i1); X2 = fmax(X2, i2); Y2 = fmax(Y2, i3); }
                        if (k < 4) pack |= (uint32_t)t << (8 * k);
                        k++;
                    }
                    const double cx = lx + x * 0.5, cy = ly + y * 0.5;
                    const bool far_out = k > 0 && (cx < X1 - margin || cx > X2 + margin || cy < Y1 - margin || cy > Y2 + margin);
                    pend = !far_out;  // centre outside the supports' bounding box: the root test fails (cf. rest_height_supports, pct_geom.cuh)
                }
            }
            const uint32_t fm = __ballot_sync(FULL, feas), pm = __ballot_sync(FULL, pend);
            if (lane == 0) ev->fbits[pos >> 5] = fm;
            nf += __popc(fm);
            n_walk += __popc(pm);
            if (pm) {
                int qb = 0;
                if (lane == 0) qb = atomicAdd(p.walk.walk_ctr, __popc(pm));
                qb = __shfl_sync(FULL, qb, 0);
                if (pend) p.walk.walkq[qb + __popc(pm & lt)] = WalkItemC{(uint32_t)e, pack, (uint16_t)c, code, k, mh};
            }
            pos += 32;
        }
        if (lane == 0) { ev->n_fw = pos >> 5; ev->n_pending = n_walk; }
    }
    if (lane == 0) {
        ev->h.n_cand = cnt;
        if (fl) ev->h.flags |= fl;
        if (p.ready) env_publish(p.ready + p.n_envs + e, p.epoch);
    }
}

// ---- pooled walks (round 2): the walk stage of pct_walks.cuh over the continuous record ----
// the candidate's tuple is rebuilt from its code (cand_tuple); everything else of the walk lives in CEnv
struct CWalkView {
    GeomC g;
    EdgePool pool;
    NodeC root;
    CEnv *ev;
    __device__ __forceinline__ uint32_t *fbits() const { return ev->fbits; }
    __device__ __forceinline__ int32_t *flags() const { return &ev->h.flags; }
    __device__ __forceinline__ int32_t *n_pending() const { return &ev->n_pending; }
    __device__ __forceinline__ BigScratch *big() const { return &ev->big; }
    __device__ __forceinline__ int32_t *lock() const { return &ev->lock; }
};
struct CWalk {
    typedef CParams Params;
    typedef WalkItemC Item;
    typedef GeomC Geom;
    static __device__ __forceinline__ CWalkView view(const CParams &p, const WalkItemC &it, bool has) {
        CEnv *ev = p.env + it.env;
        const CHdr &h = ev->h;
        double t6[6] = {0, 0, 0, 0, 0, 0};
        if (has) {
            const double nb[3] = {h.next_box[0], h.next_box[1], h.next_box[2]};
            cand_tuple(it.code, ev->ems, nb, t6);
        }
        const double x = t6[3] - t6[0], y = t6[4] - t6[1], z = t6[5] - t6[2];
        return CWalkView{GeomC{ev->box, ev->den, has ? h.n_box : 0},
                               EdgePool{ev->e_lower, ev->e_next, ev->e_off, ev->first_in, ev->last_in, ev->e_st, ev->e_st, has ? h.n_edge : 0, ev->poly_off,
                                        &ev->poly[0][0], &ev->poly[0][0], has ? h.n_poly : 0},
                               NodeC{t6[0], t6[1], it.mh, x, y, z, x * y * z * (has ? h.next_den : 1.0)},
                         ev};
    }
    static __device__ __forceinline__ bool tall(const CParams &p, const WalkItemC &it) { return it.mh >= 0.6 * p.H; }
};

__global__ void __launch_bounds__(32 * LIGHT_WARPS, 4) pctc_walk_light_kernel(const CParams p) { walk_light<CWalk>(p); }
__global__ void __launch_bounds__(32 * WALK_WARPS, 8) pctc_walk_kernel(const CParams p) { PCT_WALK_CONT_BODY(CWalk, p) }
__global__ void __launch_bounds__(32 * WALK_WARPS, 8) pctc_walk_fork_kernel(const CParams p) { walk_fork<CWalk>(p); }

template <typename OT, bool SEL = false> __device__ __noinline__ void write_obs_c_delta(const CParams &p, int e, const CEnv *ev, const double (*leaf)[6], int n_leaf, int tid, int nthreads);

// emit (round 2): the first `nl` set feasibility bits in candidate order -> leaf rows, observation; 64 threads per env.
// SEL: the selected launch; block 0 empties the pools whether or not its slot holds an env
template <typename OT, bool SEL = false>
__global__ void __launch_bounds__(64) pctc_emit_kernel(const ParamsT<CParams, SEL> p) {
    __shared__ double leaf[NL_MAX][6];
    __shared__ int s_nleaf;
    const int tid = threadIdx.x, lane = tid & 31, e = slot_env<SEL>(p, blockIdx.x);
    if (SEL && blockIdx.x == 0 && tid == 0) reset_walk_pools(p.walk);
    if (SEL && e < 0) return;  // the whole block
    CEnv *ev = p.env + e;
    const CHdr &h = ev->h;
    const double nb[3] = {h.next_box[0], h.next_box[1], h.next_box[2]};
    if (!SEL && e == 0 && tid == 0) reset_walk_pools(p.walk);
    if (tid == 0) wait_walks(&ev->n_pending, ev);
    __syncthreads();
    if (tid < 32) {
        const int nl = p.nl, nw = ev->n_fw;
        const uint32_t lt = (1u << lane) - 1;
        int base = 0;
#pragma unroll 1
        for (int w = 0; w < nw && base < nl; w++) {
            const uint32_t bits = ev->fbits[w];
            if ((bits >> lane) & 1u) {
                const int kk = base + __popc(bits & lt);
                if (kk < nl) {
                    double t6[6];
                    cand_tuple(ev->cand[w * 32 + lane], ev->ems, nb, t6);
                    for (int t = 0; t < 6; t++) leaf[kk][t] = t6[t];
                }
            }
            base += __popc(bits);
        }
        if (lane == 0) s_nleaf = min(base, nl);
    }
    __syncthreads();
    const int n_leaf = s_nleaf;
    for (int t = tid; t < n_leaf * 6; t += 64) ((double *)ev->leaf)[t] = ((double *)leaf)[t];
    if (tid == 0) {
        ev->h.n_leaf = n_leaf;
        if (p.info) {
            p.info[e].n_leaf = n_leaf; p.info[e].n_cand = h.n_cand; p.info[e].n_ems = h.n_ems; p.info[e].flags |= h.flags;
        }
    }
    // one instance of the delta writer per kernel: with the whole-batch kernel as its only caller, the compiler specialises the call on that
    // kernel's `leaf` array, and a shared instance would change the whole-batch kernel's code
    if (p.delta) write_obs_c_delta<OT, SEL>(p, e, ev, leaf, n_leaf, tid, 64);
    else write_obs_c<OT>(p, e, ev, leaf, n_leaf, tid, 64);
}


// ================= K3: feasibility per candidate + leaf compaction + observation =================
// Delta variant of write_obs_c (cf. write_obs_delta, pct_discrete.cu): the caller hands back the same observation buffer, obs_prev[0] / [1] say how
// many internal / leaf rows of it may be non-zero; only the rows below max(now, prev) and the item row are written.  Same values as write_obs_c.
template <typename OT, bool SEL>
__device__ __noinline__ void write_obs_c_delta(const CParams &p, int e, const CEnv *ev, const double (*leaf)[6], int n_leaf, int tid, int nthreads) {
    OT *obs = (OT *)p.obs + (size_t)e * (size_t)((p.nb + p.nl + 1) * 9);
    int32_t *prev = p.aux[e].obs_prev;
    const int n_box = ev->h.n_box;
    const int pb = min(prev[0], p.nb), pl = min(prev[1], p.nl);
    __syncthreads();  // every thread of the block (= env) has read prev before thread 0 replaces it
    const int wb = max(max(n_box, pb), 1), wl = max(n_leaf, pl);
    double s0 = ev->h.next_box[0], s1 = ev->h.next_box[1], s2 = ev->h.next_box[2];
    if (s1 < s0) { double t = s0; s0 = s1; s1 = t; }
    if (s2 < s1) { double t = s1; s1 = s2; s2 = t; }
    if (s1 < s0) { double t = s0; s0 = s1; s1 = t; }
    const int total = (wb + wl + 1) * 9;
#pragma unroll 1
    for (int f = tid; f < total; f += nthreads) {
        const int r = f / 9, col = f - r * 9;
        double v = 0;
        int row;
        if (r < wb) {
            row = r;
            if (row < n_box) {
                const double *b = ev->box[row];
                if (col < 3) v = b[col];
                else if (col < 6) v = b[col - 3] + b[col];
                else if (col == 8) v = 1;
            } else if (row == 0 && col == 8) v = 1;
        } else if (r < wb + wl) {
            const int k = r - wb;
            row = p.nb + k;
            if (k < n_leaf) {
                if (col < 5) v = leaf[k][col];
                else if (col == 5) v = p.H;
                else if (col == 8) v = 1;
            }
        } else {
            row = p.nb + p.nl;
            if (col == 0) v = ev->h.next_den;
            else if (col == 3) v = s0;
            else if (col == 4) v = s1;
            else if (col == 5) v = s2;
            else if (col == 8) v = 1;
        }
        obs[row * 9 + col] = (OT)v;
    }
    if (tid == 0) { prev[0] = max(n_box, 1); prev[1] = n_leaf; }
}

template <bool PRE>
__device__ __forceinline__ double (*rb_store())[5] {  // the default instantiation owns no such array
    if constexpr (PRE) { __shared__ double rb_s[NB_MAX][5]; return rb_s; }
    else return nullptr;
}

// PRE: resting heights from pre-rounded box rectangles staged in shared memory (rest_height_pre; opt-in, PCT_B200_CONT_PRE=1)
template <typename OT, bool STAB, bool PRE, bool SEL = false>
__global__ void __launch_bounds__(64) pctc_feas_emit_kernel(const ParamsT<CParams, SEL> p) {
    __shared__ double leaf[NL_MAX][6];
    double (*rb)[5] = rb_store<PRE>();
    __shared__ uint32_t wb[2];
    __shared__ int lock;
    const int tid = threadIdx.x, lane = tid & 31;
    int e = blockIdx.x;
    if constexpr (SEL) {
        e = sel_env(p.sel, p.n_envs, e);
        if (e < 0) return;  // the whole block
    }
    CEnv *ev = p.env + e;
    const CHdr &h = ev->h;
    if (tid == 0) {
        lock = 0;
        if (p.ready && !env_wait(p.ready + p.n_envs + e, p.epoch)) atomicOr(&ev->h.flags, PCT_FLAG_SYNC_TIMEOUT);
    }
    __syncthreads();
    const double nb[3] = {h.next_box[0], h.next_box[1], h.next_box[2]};
    const int n_cand = h.n_cand, n_box = h.n_box;
    const double den = h.next_den;
    GeomC g{ev->box, ev->den, n_box};
    EdgePool pool{ev->e_lower, ev->e_next, ev->e_off, ev->first_in, ev->last_in, ev->e_st, ev->e_st, h.n_edge,
                  ev->poly_off, &ev->poly[0][0], &ev->poly[0][0], h.n_poly};
    int fl = 0;
    if (PRE) {
        for (int t = tid; t < n_box; t += 64) {
            const double *b = ev->box[t];
            rb[t][0] = around6(-b[0]); rb[t][1] = around6(-b[1]); rb[t][2] = around6(b[0] + b[3]); rb[t][3] = around6(b[1] + b[4]);
            rb[t][4] = b[2] + b[5];
        }
        __syncthreads();
    }
    // get_possible_position: x = xe - xs ... (C:bin3D.py:134-137), the first `nl` feasible candidates in order
    const int n_leaf = first_feasible<2>(n_cand, p.nl, leaf, wb, [&](int c, double *t6) {
        cand_tuple(ev->cand[c], ev->ems, nb, t6);
        double mh;
        return place_virtual_c<STAB, PRE>(p, g, pool, &ev->big, &lock, t6[3] - t6[0], t6[4] - t6[1], t6[5] - t6[2], t6[0], t6[1], den, mh, fl, rb) != 0;
    });
    fl = __reduce_or_sync(FULL, fl);
    if (fl && lane == 0) atomicOr(&ev->h.flags, fl);
    __syncthreads();
    for (int t = tid; t < n_leaf * 6; t += 64) ((double *)ev->leaf)[t] = ((double *)leaf)[t];
    if (tid == 0) {
        ev->h.n_leaf = n_leaf;
        if (p.info) {
            p.info[e].n_leaf = n_leaf; p.info[e].n_cand = n_cand; p.info[e].n_ems = h.n_ems; p.info[e].flags |= h.flags;
        }
    }
    write_obs_c<OT>(p, e, ev, leaf, n_leaf, tid, 64);
}

__global__ void pctc_policy_random_kernel(const CEnv *env, int n_envs, int64_t env_id_base, uint64_t seed, int64_t t, int32_t *leaf_idx) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_envs) return;
    const int n = env[e].h.n_leaf;
    leaf_idx[e] = n > 0 ? (int32_t)(rnd_u64(seed, (uint64_t)(env_id_base + e), (uint64_t)t) % (uint64_t)n) : 0;
}

// ================= item preview / item override / per-env reset (pct_preview_items / pct_set_items / pct_reset_envs; discrete twins and notes: pct_items.cu) =================
// C0: the preview column of entry 0 (1: pct_buffer_preview_items, as in pct_items.cu)
template <int C0>
__device__ __forceinline__ void preview_entry_c(const CParams &p, const ItemParams &ip) {
    const int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= (int64_t)ip.n * ip.k) return;
    const int r = (int)(t / ip.k), j = (int)(t - (int64_t)r * ip.k) + C0;
    const int e = ip.env ? ip.env[r] : r;
    double *o = ip.out + (size_t)t * 4;
    if (e < 0 || e >= p.n_envs) {  // not an env of this handle: a zero row
        o[0] = 0; o[1] = 0; o[2] = 0; o[3] = 0;
        return;
    }
    CHdr h = p.env[e].h;
    if (j > 0) {
        h.draw_pos += j - 1;
        draw_item_c(p, e, h);
    }
    o[0] = h.next_box[0]; o[1] = h.next_box[1]; o[2] = h.next_box[2]; o[3] = h.next_den;
}

__global__ void __launch_bounds__(256) pctc_preview_kernel(const CParams p, const ItemParams ip) { preview_entry_c<0>(p, ip); }
__global__ void __launch_bounds__(256) pctc_buf_preview_kernel(const CParams p, const ItemParams ip) { preview_entry_c<1>(p, ip); }

// stands in for pctc_apply_kernel: thread t writes item t (t < n) and initialises env t's info record (t < n_envs).
// SEL (pct_set_items_only): thread t writes item t and the info record of its env, nothing else.
template <bool SEL = false>
__global__ void __launch_bounds__(256) pctc_set_items_kernel(const CParams p, const ItemParams ip) {
    const int t = blockIdx.x * 256 + threadIdx.x;
    if (t < ip.n) {
        const int e = ip.env ? ip.env[t] : t;
        if (e >= 0 && e < p.n_envs) {
            const double *it = (const double *)ip.items + (size_t)t * 3;
            CHdr &h = p.env[e].h;
            h.next_box[0] = it[0]; h.next_box[1] = it[1]; h.next_box[2] = it[2];
            if (ip.density) h.next_den = ip.density[t];
            if (SEL && p.info) {
                pct_step_info info{};
                info.counter = h.n_box;
                info.flags = h.flags;
                p.info[e] = info;
            }
        }
    }
    if (!SEL && t < p.n_envs && p.info) {
        const CHdr &h = p.env[t].h;
        pct_step_info info{};
        info.counter = h.n_box;
        info.flags = h.flags;
        p.info[t] = info;
    }
}

// stands in for pctc_apply_kernel (pct_reset_envs): warp w resets env w with reset_space_c if selected, then writes its info record.
// SEL (pct_reset_envs_only): warp w owns slot w of the selection, O(n); unselected envs are not touched.
template <bool SEL = false>
__global__ void __launch_bounds__(256) pctc_reset_envs_kernel(const CParams p, const ResetParams rp) {
    const int w = (blockIdx.x * 256 + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    int e = w;
    bool sel;
    if constexpr (SEL) {
        e = sel_env(EnvSel{rp.env, rp.mask, rp.n}, p.n_envs, w);
        if (e < 0) return;  // the whole warp
        sel = true;
    } else {
        if (e >= p.n_envs) return;  // the whole warp
        sel = rp.mask && rp.mask[e] != 0;
        if (!rp.mask)
            for (int i0 = 0; i0 < rp.n && !sel; i0 += 32) sel = __any_sync(FULL, i0 + lane < rp.n && rp.env[i0 + lane] == e);
    }
    CEnv *ev = p.env + e;
    if (sel) reset_space_c(ev, p, e, lane);
    if (lane == 0 && p.info) {
        pct_step_info info{};
        info.counter = ev->h.n_box;
        info.flags = ev->h.flags;
        p.info[e] = info;
    }
}

// ================= launchers (pct_api.cu builds their CParams from the handle) =================
// number of kernels one reset / step enqueues (for pct_kernel_launches): apply, candidates, [light, walk], emit; round 1's kernels: apply, candidates, feas_emit
int continuous_kernels_per_step(const CParams &p) { return p.walk.walkq && p.setting != 2 ? 5 : 3; }

// SEL: the selected launch of p.sel (p.ready = nullptr): the SEL instantiations over p.sel.slots(n_envs) slots, the walk kernels as they are
template <bool SEL>
static cudaError_t launch_c(const ParamsT<CParams, SEL> &p, int opt, cudaStream_t st, bool apply) {
    const bool stab = p.setting != 2;
    int slots = p.n_envs;
    if constexpr (SEL) slots = p.sel.slots(p.n_envs);
    const int b2 = (slots + 1) / 2;
    if (apply) {
        if (stab && (opt & PCT_OPT_ALIAS)) pctc_apply_kernel<true, true, SEL><<<b2, 64, 0, st>>>(p);
        else if (stab) pctc_apply_kernel<true, false, SEL><<<b2, 64, 0, st>>>(p);
        else pctc_apply_kernel<false, false, SEL><<<b2, 64, 0, st>>>(p);
    }
    // candidates / feas_emit: with p.ready as programmatic dependent launches (their blocks become resident during the previous
    // kernel's tail and wait per env on the hand-over flags), else plain back-to-back launches
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg{};
    cfg.stream = st; cfg.attrs = at; cfg.numAttrs = p.ready ? 1 : 0;
    // delta observation rows (emit kernel): a buffer other than the tracked one may hold anything -> "all rows"
    if (opt & PCT_OPT_FILL_PREV) launch_fill_prev(p.aux, p.n_envs, p.nb, p.nl, st);
    cfg.gridDim = dim3(slots); cfg.blockDim = dim3(32);
    cudaLaunchKernelEx(&cfg, pctc_candidates_kernel<SEL>, p);
    if (p.walk.walkq) {
        if (stab) {
            int n_sm = 0;
            const cudaError_t es = sm_count(&n_sm);
            if (es != cudaSuccess) return es;
            const CParams &pw = p;  // the walks carry their env and size the continuation pool from p.n_envs: the same kernels serve a selection
            pctc_walk_light_kernel<<<n_sm * 4, 32 * LIGHT_WARPS, 0, st>>>(pw);
            if (p.walk.walk_fork) pctc_walk_fork_kernel<<<n_sm * max(1, min(p.walk.walk_blocks, 8)), 32 * WALK_WARPS, 0, st>>>(pw);  // one resident wave
            else pctc_walk_kernel<<<n_sm * 8, 32 * WALK_WARPS, 0, st>>>(pw);  // one resident wave
        }
        cudaLaunchConfig_t c2{};
        c2.stream = st; c2.attrs = at; c2.numAttrs = (stab && !(opt & PCT_OPT_NO_EMIT_PDL)) ? 1 : 0;
        c2.gridDim = dim3(slots); c2.blockDim = dim3(64);
        if (p.obs_f64) cudaLaunchKernelEx(&c2, pctc_emit_kernel<double, SEL>, p);
        else cudaLaunchKernelEx(&c2, pctc_emit_kernel<float, SEL>, p);
        return cudaGetLastError();
    }
    cfg.blockDim = dim3(64);
    if (opt & PCT_OPT_CONT_PRE) {
        if (p.obs_f64) { if (stab) cudaLaunchKernelEx(&cfg, pctc_feas_emit_kernel<double, true, true, SEL>, p); else cudaLaunchKernelEx(&cfg, pctc_feas_emit_kernel<double, false, true, SEL>, p); }
        else { if (stab) cudaLaunchKernelEx(&cfg, pctc_feas_emit_kernel<float, true, true, SEL>, p); else cudaLaunchKernelEx(&cfg, pctc_feas_emit_kernel<float, false, true, SEL>, p); }
    } else {
        if (p.obs_f64) { if (stab) cudaLaunchKernelEx(&cfg, pctc_feas_emit_kernel<double, true, false, SEL>, p); else cudaLaunchKernelEx(&cfg, pctc_feas_emit_kernel<double, false, false, SEL>, p); }
        else { if (stab) cudaLaunchKernelEx(&cfg, pctc_feas_emit_kernel<float, true, false, SEL>, p); else cudaLaunchKernelEx(&cfg, pctc_feas_emit_kernel<float, false, false, SEL>, p); }
    }
    return cudaGetLastError();
}

cudaError_t launch_continuous(const CParams &p, int opt, cudaStream_t st, bool apply, const EnvSel *sel) {
    if (!sel) return launch_c<false>(p, opt, st, apply);
    SelParams<CParams> ps;
    static_cast<CParams &>(ps) = p;
    ps.sel = *sel;
    return launch_c<true>(ps, opt, st, apply);
}

cudaError_t launch_set_items_continuous(const CParams &p, int opt, const ItemParams &ip, cudaStream_t st, const EnvSel *sel) {
    const int n = sel ? ip.n : max(ip.n, p.n_envs);
    if (sel) pctc_set_items_kernel<true><<<(n + 255) / 256, 256, 0, st>>>(p, ip);
    else pctc_set_items_kernel<<<(n + 255) / 256, 256, 0, st>>>(p, ip);
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) return err;
    return launch_continuous(p, opt, st, false, sel);
}

cudaError_t launch_reset_kernel_continuous(const CParams &p, const ResetParams &rp, cudaStream_t st, const EnvSel *sel) {
    const int slots = sel ? sel->slots(p.n_envs) : p.n_envs;
    if (sel) pctc_reset_envs_kernel<true><<<(slots + 7) / 8, 256, 0, st>>>(p, rp);
    else pctc_reset_envs_kernel<<<(slots + 7) / 8, 256, 0, st>>>(p, rp);
    return cudaGetLastError();
}

cudaError_t launch_reset_envs_continuous(const CParams &p, int opt, const ResetParams &rp, cudaStream_t st, const EnvSel *sel) {
    const cudaError_t err = launch_reset_kernel_continuous(p, rp, st, sel);
    if (err != cudaSuccess) return err;
    return launch_continuous(p, opt, st, false, sel);
}

// the apply kernel alone, in plain stream order (pct_buffer_step / pct_buffer_reset); sel: its SEL instantiation (pct_buffer_step_envs)
cudaError_t launch_apply_continuous(const CParams &p, int opt, cudaStream_t st, const EnvSel *sel) {
    if (sel) {
        SelParams<CParams> ps;
        static_cast<CParams &>(ps) = p;
        ps.sel = *sel;
        const int b2 = (sel->slots(p.n_envs) + 1) / 2;
        if (p.setting != 2 && (opt & PCT_OPT_ALIAS)) pctc_apply_kernel<true, true, true><<<b2, 64, 0, st>>>(ps);
        else if (p.setting != 2) pctc_apply_kernel<true, false, true><<<b2, 64, 0, st>>>(ps);
        else pctc_apply_kernel<false, false, true><<<b2, 64, 0, st>>>(ps);
        return cudaGetLastError();
    }
    const int b2 = (p.n_envs + 1) / 2;
    if (p.setting != 2 && (opt & PCT_OPT_ALIAS)) pctc_apply_kernel<true, true><<<b2, 64, 0, st>>>(p);
    else if (p.setting != 2) pctc_apply_kernel<true, false><<<b2, 64, 0, st>>>(p);
    else pctc_apply_kernel<false, false><<<b2, 64, 0, st>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_preview_continuous(const CParams &p, const ItemParams &ip, cudaStream_t st) {
    const int64_t n = (int64_t)ip.n * ip.k;
    pctc_preview_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(p, ip);
    return cudaGetLastError();
}

cudaError_t launch_buffer_preview_continuous(const CParams &p, const ItemParams &ip, cudaStream_t st) {
    const int64_t n = (int64_t)ip.n * ip.k;
    pctc_buf_preview_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(p, ip);
    return cudaGetLastError();
}

cudaError_t launch_policy_random_continuous(const CEnv *env, int n_envs, int64_t env_id_base, uint64_t seed, int64_t t, int32_t *leaf_idx,
                                            cudaStream_t st) {
    pctc_policy_random_kernel<<<(n_envs + 127) / 128, 128, 0, st>>>(env, n_envs, env_id_base, seed, t, leaf_idx);
    return cudaGetLastError();
}

}  // namespace pct

#include "pct_heuristics_continuous.cuh"
