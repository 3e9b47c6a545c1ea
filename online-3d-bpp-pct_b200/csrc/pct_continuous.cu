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
#include "pct_handle.h"
#include "pct_geom_continuous.cuh"
#include "pct_walks.cuh"
#include "pct_continuous.cuh"

namespace pct {

// around6, NodeC / GeomC (geometry policy of the stability routine), rest_height_c, rest_height_pre: pct_geom_continuous.cuh

__device__ __forceinline__ bool rot_dims_c(const double nb[3], int rot, double &sx, double &sy, double &sz) {  // C:space.py:537-559
    switch (rot) {
    case 0: sx = nb[0]; sy = nb[1]; sz = nb[2]; return true;
    case 1: sx = nb[1]; sy = nb[0]; sz = nb[2]; return !(fabs(sx - sy) < 1e-6);
    case 2: sx = nb[0]; sy = nb[2]; sz = nb[1]; return !(fabs(sx - sy) < 1e-6 && fabs(sy - sz) < 1e-6);
    case 3: sx = nb[1]; sy = nb[2]; sz = nb[0]; return !(fabs(sx - sy) < 1e-6 && fabs(sy - sz) < 1e-6);
    case 4: sx = nb[2]; sy = nb[0]; sz = nb[1]; return !(fabs(sx - sy) < 1e-6);
    default: sx = nb[2]; sy = nb[1]; sz = nb[0]; return !(fabs(sx - sy) < 1e-6);
    }
}
// candidate code = ems_idx << 5 | rot << 2 | corner  ->  the 6-tuple the reference adds to its set (C:space.py:563-566)
__device__ __forceinline__ void cand_tuple(uint16_t code, const double (*ems)[6], const double nb[3], double t[6]) {
    const double *m = ems[code >> 5];
    double sx, sy, sz;
    rot_dims_c(nb, (code >> 2) & 7, sx, sy, sz);
    const int q = code & 3;
    if (q & 1) { t[0] = m[3] - sx; t[3] = m[3]; } else { t[0] = m[0]; t[3] = m[0] + sx; }
    if (q & 2) { t[1] = m[4] - sy; t[4] = m[4]; } else { t[1] = m[1]; t[4] = m[1] + sy; }
    t[2] = m[2]; t[5] = m[2] + sz;
}
__device__ __noinline__ uint64_t hash_double_call(double v) { return hash_double(v); }  // one copy of the routine for the three call sites of the candidates kernel
__device__ __noinline__ uint64_t cand_hash_c(const double t[6]) {
    uint64_t l[6];
#pragma unroll 1
    for (int i = 0; i < 6; i++) l[i] = hash_double(t[i]);
    return tuple_hash6(l);
}

__device__ __noinline__ void draw_item_c(const CParams &p, int e, CHdr &h) {
    const uint64_t gid = (uint64_t)(p.env_id_base + e), d = (uint64_t)h.draw_pos;
    if (p.item_mode == 0 && p.sample_dist) {  // C:bin3D.py:103-112
        auto u01 = [&](uint64_t salt) { return (double)(rnd_u64(p.seed ^ salt, gid, d) >> 11) * (1.0 / 9007199254740992.0); };
        auto r3 = [&](double v) { return ddiv(rint(v * 1000.0), 1000.0); };
        h.next_box[0] = r3(p.sample_a + (p.sample_b - p.sample_a) * u01(0x11));
        h.next_box[1] = r3(p.sample_a + (p.sample_b - p.sample_a) * u01(0x22));
        if (p.setting == 2) h.next_box[2] = r3(p.sample_a + (p.sample_b - p.sample_a) * u01(0x33));
        else {
            const double ch[5] = {0.1, 0.2, 0.3, 0.4, 0.5};
            h.next_box[2] = ch[rnd_u64(p.seed ^ 0x44, gid, d) % 5];
        }
        h.next_den = p.setting == 3 ? rnd_density(p.seed, gid, d) : 1.0;
    } else {
        const double *it = p.item_mode == 0 ? p.item_set + (rnd_u64(p.seed, gid, d) % (uint64_t)p.n_items) * 3
                                            : p.stream + ((size_t)e * p.stream_len + (size_t)(d % (uint64_t)p.stream_len)) * 4;
        h.next_box[0] = it[0]; h.next_box[1] = it[1]; h.next_box[2] = it[2];
        h.next_den = p.setting == 3 ? (p.item_mode == 0 ? rnd_density(p.seed, gid, d) : it[3]) : 1.0;
    }
    h.draw_pos++;
}

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

template <bool STAB, bool ALIAS = false>
__global__ void __launch_bounds__(64) pctc_apply_kernel(const CParams p) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int e = blockIdx.x * 2 + warp;
    if (e >= p.n_envs) return;
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
        if (lane == 0) { ev->e_off[n_box0] = (uint16_t)h.n_edge; ev->poly_off[n_box0] = (uint16_t)h.n_poly; ev->first_in[n_box0 < NB_MAX ? n_box0 : 0] = EDGE_NIL; }
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
// Table slots are 32 bits: candidate code | 16-bit tag (the top bits of the tuple hash — CPython compares the stored hash before the keys, setobject.c).
// A probe rejects a non-matching slot on the tag alone; the exact 6-double comparison (tuples rebuilt from the two codes) runs only on a tag match,
// i.e. practically only for true duplicates.  Round 1 rebuilt and compared the tuple of EVERY probed slot and broadcast the six doubles of every
// inserted key through shuffles (a large share of this kernel's instructions went to _Py_HashDouble's frexp loop — now an integer rotation,
// pct_pyhash.cuh — and to shuffles).
__device__ __forceinline__ bool cand_equal(uint16_t a, uint16_t b, const double (*ems)[6], const double nb[3]) {
    double u[6], v[6];
    cand_tuple(a, ems, nb, u);
    cand_tuple(b, ems, nb, v);
    return u[0] == v[0] && u[1] == v[1] && u[2] == v[2] && u[3] == v[3] && u[4] == v[4] && u[5] == v[5];
}

__global__ void __launch_bounds__(32) pctc_candidates_kernel(const CParams p) {
    __shared__ uint32_t tabA[CC_TAB], tabB[512];
    __shared__ uint64_t stg_h[32], rs_h[32];  // staged (hash, code) of the chunk's new keys / of the slots being re-inserted by a resize
    __shared__ uint32_t rs_c[32];
    __shared__ uint16_t stg_c[32];
    const int lane = threadIdx.x, e = blockIdx.x;
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
    constexpr uint32_t EMPTY = 0xFFFFFFFFu;
    uint32_t *tab = tabA;
    uint32_t mask = 7;
    int fill = 0;
    if (lane < 8) tab[lane] = EMPTY;
    __syncwarp();
    const int raw = n_ems * R * 4;
    bool stop = false;
#pragma unroll 1
    for (int base = 0; base < raw && !stop; base += 32) {
        const int r = base + lane;
        bool valid = false;
        uint64_t hash = 0;
        uint16_t code = 0;
        // The four corners of one (EMS, orientation) are four adjacent lanes and their 6-tuples draw on ten distinct coordinates (x: m0, m0 + sx, m3 - sx,
        // m3; y alike; z: m2, m2 + sz): every lane hashes two or three of them (_Py_HashDouble, the expensive part) and the group exchanges the results,
        // instead of six hashes per lane.  Same expressions as cand_tuple, so the same bits.
        uint64_t h0 = 0, h1 = 0, h2 = 0;
        const int q = r & 3;
        if (r < raw) {
            const int er = r >> 2, rot = er % R, ei = er / R;
            double sx, sy, sz;
            if (rot_dims_c(nb, rot, sx, sy, sz)) {
                const double *m = ev->ems[ei];
                if (m[3] - m[0] + 1e-6 >= sx && m[4] - m[1] + 1e-6 >= sy && m[5] - m[2] + 1e-6 >= sz) {
                    valid = true;
                    code = (uint16_t)((ei << 5) | (rot << 2) | q);
                    double v0, v1, v2 = 0;
                    if (q == 0) { v0 = m[0]; v1 = m[0] + sx; v2 = m[2]; }
                    else if (q == 1) { v0 = m[3] - sx; v1 = m[3]; v2 = m[2] + sz; }
                    else if (q == 2) { v0 = m[1]; v1 = m[1] + sy; }
                    else { v0 = m[4] - sy; v1 = m[4]; }
                    h0 = hash_double_call(v0);
                    h1 = hash_double_call(v1);
                    if (q < 2) h2 = hash_double_call(v2);
                }
            }
        }
        {
            const int gb = lane & ~3, lx = gb + (q & 1), ly = gb + 2 + (q >> 1);
            uint64_t l6[6];
            l6[0] = __shfl_sync(FULL, h0, lx); l6[3] = __shfl_sync(FULL, h1, lx);
            l6[1] = __shfl_sync(FULL, h0, ly); l6[4] = __shfl_sync(FULL, h1, ly);
            l6[2] = __shfl_sync(FULL, h2, gb); l6[5] = __shfl_sync(FULL, h2, gb + 1);
            if (valid) hash = tuple_hash6(l6);
        }
        // already present? (read-only probe; present keys sit on their own probe sequence)
        if (valid) {
            const uint32_t tag = (uint32_t)(hash >> 48);
            uint64_t perturb = hash;
            uint32_t i = (uint32_t)hash & mask;
            bool open = true;
            while (open) {
                const int probes = (i + 9 <= mask) ? 9 : 0;
                for (int j = 0; j <= probes; j++) {
                    const uint32_t s = tab[i + j];
                    if (s == EMPTY) { open = false; break; }
                    if ((s >> 16) == tag && cand_equal((uint16_t)s, code, ev->ems, nb)) { open = false; valid = false; break; }
                }
                perturb >>= 5;
                i = (uint32_t)((uint64_t)i * 5 + 1 + perturb) & mask;
            }
        }
        // the new keys of this chunk go through the order-defining insertion in lane (= reference) order: staged in shared memory and inserted by
        // lane 0 with a scalar set_add_entry (3x fewer warp instructions than a warp-uniform probe with shuffles, as in the discrete kernel);
        // an equal tuple staged by an earlier lane of the same chunk is found by the tag + exact comparison like any other present key
        const uint32_t vm = __ballot_sync(FULL, valid);
        const int n_new = __popc(vm);
        if (valid) {
            const int pos = __popc(vm & ((1u << lane) - 1));
            stg_h[pos] = hash;
            stg_c[pos] = code;
        }
        __syncwarp();
        int done = 0;
#pragma unroll 1
        while (done < n_new && !stop) {
            int upto = n_new;
            if (lane == 0) {
#pragma unroll 1
                for (int t = done; t < n_new; t++) {
                    const uint64_t hk = stg_h[t];
                    const uint16_t ck = stg_c[t];
                    const uint32_t tagk = (uint32_t)(hk >> 48);
                    uint64_t perturb = hk;
                    uint32_t i = (uint32_t)hk & mask;
                    int state = 0;
#pragma unroll 1
                    while (!state) {
                        const int probes = (i + 9 <= mask) ? 9 : 0;
#pragma unroll 1
                        for (int j = 0; j <= probes; j++) {
                            const uint32_t sl = tab[i + j];
                            if (sl == EMPTY) { tab[i + j] = (tagk << 16) | ck; state = 1; break; }
                            if ((sl >> 16) == tagk && cand_equal((uint16_t)sl, ck, ev->ems, nb)) { state = 2; break; }
                        }
                        perturb >>= 5;
                        i = (uint32_t)((uint64_t)i * 5 + 1 + perturb) & mask;
                    }
                    if (state == 1 && (uint32_t)(++fill) * 5 >= mask * 3) { upto = t + 1; break; }
                }
            }
            upto = __shfl_sync(FULL, upto, 0);
            fill = __shfl_sync(FULL, fill, 0);
            done = upto;
            __syncwarp();
            if ((uint32_t)fill * 5 >= mask * 3) {
                uint32_t newsize = 8;
                while (newsize <= (uint32_t)fill * 4) newsize <<= 1;
                if (newsize > CC_TAB) { fl |= PCT_FLAG_CAND_OVERFLOW; stop = true; break; }
                uint32_t *nt = (tab == tabA) ? tabB : tabA;
                for (uint32_t t = lane; t < newsize; t += 32) nt[t] = EMPTY;
                __syncwarp();
#pragma unroll 1
                for (uint32_t b2 = 0; b2 <= mask; b2 += 32) {  // set_table_resize: re-insert in slot order (set_insert_clean: no comparisons)
                    const uint32_t sidx = b2 + lane;
                    const uint32_t c2 = sidx <= mask ? tab[sidx] : EMPTY;
                    const uint32_t em = __ballot_sync(FULL, c2 != EMPTY);
                    if (c2 != EMPTY) {
                        double u[6];
                        cand_tuple((uint16_t)c2, ev->ems, nb, u);
                        const int pos = __popc(em & ((1u << lane) - 1));
                        rs_h[pos] = cand_hash_c(u);
                        rs_c[pos] = c2;
                    }
                    __syncwarp();
                    if (lane == 0) {
                        const int m2 = __popc(em);
#pragma unroll 1
                        for (int t = 0; t < m2; t++) {
                            uint64_t pt = rs_h[t];
                            uint32_t ii = (uint32_t)pt & (newsize - 1);
                            bool placed = false;
#pragma unroll 1
                            while (!placed) {
                                const int pr = (ii + 9 <= newsize - 1) ? 9 : 0;
                                for (int j = 0; j <= pr; j++)
                                    if (nt[ii + j] == EMPTY) { nt[ii + j] = rs_c[t]; placed = true; break; }
                                pt >>= 5;
                                ii = (uint32_t)((uint64_t)ii * 5 + 1 + pt) & (newsize - 1);
                            }
                        }
                    }
                    __syncwarp();
                }
                tab = nt;
                mask = newsize - 1;
            }
        }
        __syncwarp();
    }
    __syncwarp();
    int cnt = 0;
#pragma unroll 1
    for (uint32_t b2 = 0; b2 <= mask; b2 += 32) {
        const uint32_t s = b2 + lane;
        const uint32_t c2 = s <= mask ? tab[s] : EMPTY;
        const uint32_t em = __ballot_sync(FULL, c2 != EMPTY);
        if (c2 != EMPTY) ev->cand[cnt + __popc(em & ((1u << lane) - 1))] = (uint16_t)c2;
        cnt += __popc(em);
    }
    __syncwarp();
    if (p.shuffle) {  // scratch: the GENEMS temp list (24 KB, idle between apply kernels): keys at 0, permuted codes at 10 KB
        static_assert(sizeof(ev->ems_tmp) >= 10240 + sizeof(ev->cand), "shuffle scratch fits");
        shuffle_candidates<uint16_t>(ev->cand, cnt, (uint64_t *)ev->ems_tmp, (uint16_t *)((char *)ev->ems_tmp + 10240), p.seed, (uint64_t)(p.env_id_base + e),
                                     (uint64_t)h.draw_pos, lane);
    }
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

template <typename OT> __device__ __noinline__ void write_obs_c_delta(const CParams &p, int e, const CEnv *ev, const double (*leaf)[6], int n_leaf, int tid, int nthreads);

// emit (round 2): the first `nl` set feasibility bits in candidate order -> leaf rows, observation; 64 threads per env
template <typename OT>
__global__ void __launch_bounds__(64) pctc_emit_kernel(const CParams p) {
    __shared__ double leaf[NL_MAX][6];
    __shared__ int s_nleaf;
    const int tid = threadIdx.x, lane = tid & 31, e = blockIdx.x;
    CEnv *ev = p.env + e;
    const CHdr &h = ev->h;
    const double nb[3] = {h.next_box[0], h.next_box[1], h.next_box[2]};
    if (e == 0 && tid == 0) reset_walk_pools(p.walk);
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
    if (p.delta) write_obs_c_delta<OT>(p, e, ev, leaf, n_leaf, tid, 64);
    else write_obs_c<OT>(p, e, ev, leaf, n_leaf, tid, 64);
}


// ================= K3: feasibility per candidate + leaf compaction + observation =================
// Delta variant of write_obs_c (cf. write_obs_delta, pct_discrete.cu): the caller hands back the same observation buffer, obs_prev[0] / [1] say how
// many internal / leaf rows of it may be non-zero; only the rows below max(now, prev) and the item row are written.  Same values as write_obs_c.
template <typename OT>
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
template <typename OT, bool STAB, bool PRE>
__global__ void __launch_bounds__(64) pctc_feas_emit_kernel(const CParams p) {
    __shared__ double leaf[NL_MAX][6];
    double (*rb)[5] = rb_store<PRE>();
    __shared__ uint32_t wb[2];
    __shared__ int lock;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, e = blockIdx.x;
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
    int n_leaf = 0, fl = 0;
    if (PRE) {
        for (int t = tid; t < n_box; t += 64) {
            const double *b = ev->box[t];
            rb[t][0] = around6(-b[0]); rb[t][1] = around6(-b[1]); rb[t][2] = around6(b[0] + b[3]); rb[t][3] = around6(b[1] + b[4]);
            rb[t][4] = b[2] + b[5];
        }
        __syncthreads();
    }
#pragma unroll 1
    for (int base = 0; base < n_cand && n_leaf < p.nl; base += 64) {
        const int c = base + tid;
        bool feas = false;
        double t6[6] = {0, 0, 0, 0, 0, 0};
        if (c < n_cand) {
            cand_tuple(ev->cand[c], ev->ems, nb, t6);
            // get_possible_position: x = xe - xs ... (C:bin3D.py:134-137); drop_box_virtual (C:space.py:380-425)
            const double x = t6[3] - t6[0], y = t6[4] - t6[1], z = t6[5] - t6[2], lx = t6[0], ly = t6[1];
            bool chk = !(lx + x - 1e-6 > p.W || ly + y - 1e-6 > p.L) && !(lx + 1e-6 < 0 || ly + 1e-6 < 0);
            double mh = PRE ? rest_height_pre(rb, n_box, around6(-lx), around6(-ly), around6(lx + x), around6(ly + y))
                            : rest_height_c(ev->box, 0, n_box, 1, lx, ly, lx + x, ly + y);
            if (mh < 0) mh = 0.0;
            if (mh + z - 1e-6 > p.H) chk = false;
            if (!chk) feas = false;
            else if (!STAB || fabs(mh) < 1e-6) feas = true;
            else {
                NodeC root{lx, ly, mh, x, y, z, x * y * z * den};
                feas = stability_check<false, GeomC>(g, root, pool, &ev->big, &lock, 0, fl) != 0;
            }
        }
        const uint32_t fm = __ballot_sync(FULL, feas);
        if (lane == 0) wb[warp] = fm;
        __syncthreads();
        const int before = warp == 1 ? __popc(wb[0]) : 0, total = __popc(wb[0]) + __popc(wb[1]);
        if (feas) {
            const int k = n_leaf + before + __popc(fm & ((1u << lane) - 1));
            if (k < p.nl)
                for (int t = 0; t < 6; t++) leaf[k][t] = t6[t];
        }
        n_leaf += total;
        __syncthreads();
    }
    if (n_leaf > p.nl) n_leaf = p.nl;
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
__global__ void __launch_bounds__(256) pctc_preview_kernel(const CParams p, const ItemParams ip) {
    const int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= (int64_t)ip.n * ip.k) return;
    const int r = (int)(t / ip.k), j = (int)(t - (int64_t)r * ip.k);
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

// stands in for pctc_apply_kernel: thread t writes item t (t < n) and initialises env t's info record (t < n_envs)
__global__ void __launch_bounds__(256) pctc_set_items_kernel(const CParams p, const ItemParams ip) {
    const int t = blockIdx.x * 256 + threadIdx.x;
    if (t < ip.n) {
        const int e = ip.env ? ip.env[t] : t;
        if (e >= 0 && e < p.n_envs) {
            const double *it = (const double *)ip.items + (size_t)t * 3;
            CHdr &h = p.env[e].h;
            h.next_box[0] = it[0]; h.next_box[1] = it[1]; h.next_box[2] = it[2];
            if (ip.density) h.next_den = ip.density[t];
        }
    }
    if (t < p.n_envs && p.info) {
        const CHdr &h = p.env[t].h;
        pct_step_info info{};
        info.counter = h.n_box;
        info.flags = h.flags;
        p.info[t] = info;
    }
}

// stands in for pctc_apply_kernel (pct_reset_envs): warp w resets env w with reset_space_c if selected, then writes its info record
__global__ void __launch_bounds__(256) pctc_reset_envs_kernel(const CParams p, const ResetParams rp) {
    const int e = (blockIdx.x * 256 + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (e >= p.n_envs) return;  // the whole warp
    bool sel = rp.mask && rp.mask[e] != 0;
    if (!rp.mask)
        for (int i0 = 0; i0 < rp.n && !sel; i0 += 32) sel = __any_sync(FULL, i0 + lane < rp.n && rp.env[i0 + lane] == e);
    CEnv *ev = p.env + e;
    if (sel) reset_space_c(ev, p, e, lane);
    if (lane == 0 && p.info) {
        pct_step_info info{};
        info.counter = ev->h.n_box;
        info.flags = ev->h.flags;
        p.info[e] = info;
    }
}

// ================= host side =================
int continuous_create(pct_env_batch *h) {
    cudaError_t e = cudaMalloc(&h->c_state, sizeof(CEnv) * (size_t)h->n_envs);
    if (e == cudaSuccess) e = cudaMemset(h->c_state, 0, sizeof(CEnv) * (size_t)h->n_envs);
    if (e == cudaSuccess) e = cudaMalloc(&h->d_ready, sizeof(int32_t) * 2 * (size_t)h->n_envs);
    if (e == cudaSuccess) e = cudaMemset(h->d_ready, 0, sizeof(int32_t) * 2 * (size_t)h->n_envs);
    if (e == cudaSuccess && !h->k3_block) e = create_walk_pools(h, sizeof(WalkItemC));
    if (e != cudaSuccess) { h->err = std::string("continuous_create: ") + cudaGetErrorString(e); return PCT_ERR_CUDA; }
    return PCT_OK;
}
void continuous_destroy(pct_env_batch *h) { cudaFree(h->c_state); h->c_state = nullptr; }
int64_t continuous_state_bytes() { return (int64_t)sizeof(CEnv); }

// CParams of the whole batch for the kernels that only read the item source (pct_preview_items)
static CParams item_params(const pct_env_batch *h) {
    CParams p{};
    p.env = (CEnv *)h->c_state; p.n_envs = h->n_envs; p.setting = h->cfg.setting;
    p.item_mode = h->item_mode; p.sample_dist = h->cfg.sample_from_distribution;
    p.sample_a = h->cfg.sample_left_bound; p.sample_b = h->cfg.sample_right_bound;
    p.item_set = h->d_item_set; p.n_items = h->n_items; p.stream = h->d_stream; p.stream_len = h->stream_len; p.traj_len = h->traj_len;
    p.seed = h->cfg.seed; p.env_id_base = h->cfg.env_id_base;
    return p;
}

int continuous_preview(pct_env_batch *h, const ItemParams &ip, cudaStream_t st) {
    const int64_t n = (int64_t)ip.n * ip.k;
    pctc_preview_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(item_params(h), ip);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { h->err = std::string("pct_preview_items: ") + cudaGetErrorString(e); return PCT_ERR_CUDA; }
    return PCT_OK;
}

// pre non-null (pct_set_items / pct_reset_envs): its kernel in place of the apply kernel, then the rest of the step's sequence in plain stream order
int continuous_launch(pct_env_batch *h, int mode, const void *actions, int action_f64, const int32_t *leaf_idx, void *obs, float *rew,
                      uint8_t *done, pct_step_info *info, cudaStream_t st, const PreKernel *pre) {
    CParams p{};
    p.env = (CEnv *)h->c_state; p.n_envs = h->n_envs;
    p.W = h->cfg.container_size[0]; p.L = h->cfg.container_size[1]; p.H = h->cfg.container_size[2];
    p.low_bound = h->cfg.size_minimum;
    p.nb = h->cfg.internal_node_holder; p.nl = h->cfg.leaf_node_holder; p.setting = h->cfg.setting;
    p.item_mode = h->item_mode; p.sample_dist = h->cfg.sample_from_distribution;
    p.sample_a = h->cfg.sample_left_bound; p.sample_b = h->cfg.sample_right_bound;
    p.item_set = h->d_item_set; p.n_items = h->n_items; p.stream = h->d_stream; p.stream_len = h->stream_len; p.traj_len = h->traj_len;
    p.seed = h->cfg.seed; p.env_id_base = h->cfg.env_id_base; p.shuffle = h->cfg.shuffle;
    p.actions = actions; p.action_f64 = action_f64; p.leaf_idx = leaf_idx;
    p.obs = obs; p.obs_f64 = h->cfg.obs_dtype == PCT_F64; p.reward = rew; p.done = done; p.info = info;
    p.mode = mode; p.keep_draw = h->did_reset ? 1 : 0; p.no_auto_reset = h->cfg.no_auto_reset;
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing(st, &cap);
    if (h->overlap_cont && h->d_ready && cap == cudaStreamCaptureStatusNone && !pre) { p.ready = h->d_ready; p.epoch = ++h->epoch; }
    const bool stab = p.setting != 2;
    const int b2 = (p.n_envs + 1) / 2;
    if (pre && pre->items) {
        const int n = max(pre->items->n, p.n_envs);
        pctc_set_items_kernel<<<(n + 255) / 256, 256, 0, st>>>(p, *pre->items);
    } else if (pre) {
        pctc_reset_envs_kernel<<<(p.n_envs + 7) / 8, 256, 0, st>>>(p, *pre->reset);
    } else if (stab && h->alias_mode && h->d_aux) {
        p.aux = h->d_aux;
        pctc_apply_kernel<true, true><<<b2, 64, 0, st>>>(p);
    } else if (stab) pctc_apply_kernel<true><<<b2, 64, 0, st>>>(p);
    else pctc_apply_kernel<false><<<b2, 64, 0, st>>>(p);
    // candidates / feas_emit: with p.ready as programmatic dependent launches (their blocks become resident during the previous
    // kernel's tail and wait per env on the hand-over flags), else plain back-to-back launches
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg{};
    cfg.stream = st; cfg.attrs = at; cfg.numAttrs = p.ready ? 1 : 0;
    const bool pooled = h->d_walkq != nullptr;
    if (pooled && h->obs_delta && h->d_aux) {  // delta observation rows (emit kernel): a buffer other than the tracked one may hold anything -> "all rows"
        if (h->fill_pending) launch_fill_prev(h->d_aux, p.n_envs, p.nb, p.nl, st);
        p.aux = h->d_aux;
        p.delta = 1;
    }
    h->fill_pending = false;
    if (pooled) p.walk = walk_pools<WalkItemC>(h, 0, p.n_envs);
    cfg.gridDim = dim3(p.n_envs); cfg.blockDim = dim3(32);
    cudaLaunchKernelEx(&cfg, pctc_candidates_kernel, p);
    if (pooled) {
        if (stab) {
            int n_sm = 0;
            const cudaError_t es = sm_count(&n_sm);
            if (es != cudaSuccess) { h->err = std::string("continuous launch: ") + cudaGetErrorString(es); return PCT_ERR_CUDA; }
            pctc_walk_light_kernel<<<n_sm * 4, 32 * LIGHT_WARPS, 0, st>>>(p);
            if (p.walk.walk_fork) pctc_walk_fork_kernel<<<n_sm * max(1, min(p.walk.walk_blocks, 8)), 32 * WALK_WARPS, 0, st>>>(p);  // one resident wave
            else pctc_walk_kernel<<<n_sm * 8, 32 * WALK_WARPS, 0, st>>>(p);  // one resident wave
        }
        {
            cudaLaunchAttribute at2[1];
            at2[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
            at2[0].val.programmaticStreamSerializationAllowed = 1;
            cudaLaunchConfig_t c2{};
            c2.stream = st; c2.attrs = at2; c2.numAttrs = (stab && cap == cudaStreamCaptureStatusNone) ? 1 : 0;
            c2.gridDim = dim3(p.n_envs); c2.blockDim = dim3(64);
            if (p.obs_f64) cudaLaunchKernelEx(&c2, pctc_emit_kernel<double>, p);
            else cudaLaunchKernelEx(&c2, pctc_emit_kernel<float>, p);
        }
        cudaError_t e2 = cudaGetLastError();
        if (e2 != cudaSuccess) { h->err = std::string("continuous launch: ") + cudaGetErrorString(e2); return PCT_ERR_CUDA; }
        h->launches += stab ? 4 : 2;  // apply, candidates, [light, walk], emit; the caller counts one
        return PCT_OK;
    }
    cfg.blockDim = dim3(64);
    if (h->cont_pre) {
        if (p.obs_f64) { if (stab) cudaLaunchKernelEx(&cfg, pctc_feas_emit_kernel<double, true, true>, p); else cudaLaunchKernelEx(&cfg, pctc_feas_emit_kernel<double, false, true>, p); }
        else { if (stab) cudaLaunchKernelEx(&cfg, pctc_feas_emit_kernel<float, true, true>, p); else cudaLaunchKernelEx(&cfg, pctc_feas_emit_kernel<float, false, true>, p); }
    } else {
        if (p.obs_f64) { if (stab) cudaLaunchKernelEx(&cfg, pctc_feas_emit_kernel<double, true, false>, p); else cudaLaunchKernelEx(&cfg, pctc_feas_emit_kernel<double, false, false>, p); }
        else { if (stab) cudaLaunchKernelEx(&cfg, pctc_feas_emit_kernel<float, true, false>, p); else cudaLaunchKernelEx(&cfg, pctc_feas_emit_kernel<float, false, false>, p); }
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { h->err = std::string("continuous launch: ") + cudaGetErrorString(e); return PCT_ERR_CUDA; }
    h->launches += 2;  // the caller counts one
    return PCT_OK;
}

int continuous_policy_random(pct_env_batch *h, int32_t *leaf_idx, uint64_t seed, int64_t t, cudaStream_t st) {
    pctc_policy_random_kernel<<<(h->n_envs + 127) / 128, 128, 0, st>>>((const CEnv *)h->c_state, h->n_envs, h->cfg.env_id_base, seed, t, leaf_idx);
    return cudaGetLastError() == cudaSuccess ? PCT_OK : PCT_ERR_CUDA;
}

int continuous_get_state(pct_env_batch *h, int env, pct_state_dump *out) {
    CEnv *tmp = (CEnv *)malloc(sizeof(CEnv));
    if (cudaMemcpy(tmp, (CEnv *)h->c_state + env, sizeof(CEnv), cudaMemcpyDeviceToHost) != cudaSuccess) { free(tmp); return PCT_ERR_CUDA; }
    memset(out, 0, sizeof(*out));
    out->n_boxes = tmp->h.n_box; out->n_ems = tmp->h.n_ems; out->n_leaf = tmp->h.n_leaf; out->flags = tmp->h.flags;
    out->draw_pos = tmp->h.draw_pos; out->next_den = tmp->h.next_den;
    for (int i = 0; i < 3; i++) out->next_box[i] = tmp->h.next_box[i];
    for (int i = 0; i < tmp->h.n_box && i < 80; i++) {
        const double *b = tmp->box[i];
        out->boxes[i][0] = b[0]; out->boxes[i][1] = b[1]; out->boxes[i][2] = b[2];
        out->boxes[i][3] = b[0] + b[3]; out->boxes[i][4] = b[1] + b[4]; out->boxes[i][5] = b[2] + b[5];
        out->boxes[i][6] = tmp->den[i];
    }
    for (int i = 0; i < tmp->h.n_ems && i < 256; i++)
        for (int t = 0; t < 6; t++) out->ems[i][t] = tmp->ems[i][t];
    free(tmp);
    return PCT_OK;
}

}  // namespace pct

#include "pct_heuristics_continuous.cuh"
