// Leaf expansion of caller-given items, read-only (pct_expand_items, include/pct_b200.h): for row r and item j, the leaf rows that
// get_possible_position() (D:bin3D.py:100-136, C:bin3D.py) produces for that item on env env[r] in its current state.
//
// One block of EXPAND_THREADS per row, which takes the row's k items in turn.  Per item:
//   warp 0    the ordered candidate list with the candidates kernel's own routines (build_candidates and the EV / EP / CP / FC generators,
//             pct_cand.cuh; PCTC_CANDIDATES_BODY, pct_cand_c.cuh), then the keyed shuffle, into the env's candidate scratch;
//   block     one thread per candidate in EXPAND_THREADS chunks: the placement test and the ordered compaction of the first `nl` feasible
//             candidates of the step's block-mode feasibility kernel (place_virtual_d / _c and first_feasible, pct_block.cuh);
//   out       the leaf rows as the observation carries them, and the info record pct_set_items would write.
// The pooled walk stage is not used: its pools and counters belong to the step.
//
// Nothing the env keeps is written.  Scratch: the transient fields every step writes before it reads them — discrete cold->cand / raw
// (candidate list, generator output, shuffle keys) and cold->big (under the block's lock); continuous ev->cand / ems_tmp / big.  Capacity
// flags raised by an expansion go to its own info record only.  The envs of one launch are distinct (caller's contract): the scratch is per env.
#include "pct_common.cuh"
#include "pct_stability.cuh"
#include "pct_kernels.h"
#include "pct_geom.cuh"
#include "pct_rot.cuh"
#include "pct_cand.cuh"
#include "pct_geom_continuous.cuh"
#include "pct_continuous.cuh"
#include "pct_cand_c.cuh"
#include "pct_block.cuh"

namespace pct {

constexpr int EXPAND_THREADS = 64;

// shared memory of one discrete block: the staged env, the set emulation's tables (the 2048-slot stage included), the leaves
template <typename SlotT>
struct ExpandSmD {
    StageD s;
    SlotT tabA[TAB_A], tabB[TAB_B];
    SetStage stg;
    int16_t leaf[NL_MAX][6];
    RotTab rt;
    int fl, n_cand;
    uint32_t wb[EXPAND_THREADS / 32];
};

// zero rows and a zero record for a row whose env index is outside the handle
template <typename OT>
__device__ __forceinline__ void expand_zero_row(const ExpandParams &x, int nl, size_t row, int tid) {
    OT *out = (OT *)x.leaves + row * (size_t)nl * 9;
    for (size_t f = tid; f < (size_t)x.k * nl * 9; f += EXPAND_THREADS) out[f] = 0;
    if (x.info)
        for (int j = tid; j < x.k; j += EXPAND_THREADS) x.info[row + j] = pct_step_info{};
}

template <typename OT, bool STAB, typename SlotT>
__global__ void __launch_bounds__(EXPAND_THREADS) pct_expand_kernel(const DParams p, const ExpandParams x) {
    constexpr int KB = sizeof(SlotT) == 2 ? 4 : 8;
    __shared__ __align__(16) ExpandSmD<SlotT> s;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, r = blockIdx.x, K = x.k, nl = p.nl;
    const int e = x.env ? x.env[r] : r;
    const size_t row = (size_t)r * K;
    if (e < 0 || e >= p.n_envs) { expand_zero_row<OT>(x, nl, row, tid); return; }
    const DEnvHot *hot = &s.s.hot;
    DEnvCold *cold = p.cold + e;
    StagedD sd = stage_env_d<STAB>(s.s, p, e, false);
    const DHdr &h = hot->h;
    const int n_box = h.n_box, R = p.setting == 2 ? 6 : 2;
    SlotT *const out = (SlotT *)cold->cand;
    const RotTab *rt = &s.rt;
#pragma unroll 1
    for (int j = 0; j < K; j++) {
        const int32_t *it = (const int32_t *)x.items + (row + j) * 3;
        const double den = x.density ? x.density[row + j] : h.next_den;
        if (warp == 0) {
            // ---- the candidates kernel's list for this item (pct_candidates_kernel) ----
            const int nb3[3] = {min(max(it[0], 0), 255), min(max(it[1], 0), 255), min(max(it[2], 0), 255)};  // as pct_set_items clamps
            if (lane == 0) make_rot_tab(nb3, R, s.rt);
            __syncwarp();
            SlotT *cand = nullptr;
            int fl = 0, n_cand = 0;
            if (p.lnes == 0) {
                const CandList<SlotT> cl = build_candidates<SlotT>(hot->ems, h.n_ems, rt, R, s.tabA, s.tabB, s.tabA, &s.stg, lane);
                cand = cl.keys; n_cand = cl.n; fl = cl.flags;
            } else if (p.lnes == 5) {
                const CandList<SlotT> cl = gen_event_point_m<SlotT>(hot, rt, R, p.W, p.L, p.H, s.tabA, s.tabB, s.tabA,
                                                                    cold->raw, out, lane);
                cand = cl.keys; n_cand = cl.n; fl = cl.flags;
            } else {
                uint32_t *raw = cold->raw;
                RawList rl;
                if (p.lnes == 4) rl = gen_full_coord<KB>(hot->box, n_box, rt, R, p.W, p.L, p.H, raw, lane);
                else if (p.lnes == 1) rl = RawList{gen_event_point<KB>(rt, R, p.W, p.L, raw, lane), 0};
                else rl = gen_level_points<KB>(hot->box, n_box, rt, R, p.W, p.L, p.H, p.lnes == 2, raw, lane);
                fl = rl.flags;
                if (rl.n == -2) {  // empty bin under EP / CP: the reference's 2-element list (D:space.py:700-701)
                    if (lane < 2) out[lane] = (SlotT)key_pack<KB>(0, 0, 0, rt->canon[lane]);
                    n_cand = 2;
                    cand = out;
                } else {
                    const CandList<SlotT> cl = build_candidates<SlotT>(hot->ems, h.n_ems, rt, R, s.tabA, s.tabB, s.tabA, &s.stg, lane, raw, rl.n);
                    cand = cl.keys; n_cand = cl.n; fl |= cl.flags;
                }
            }
            if (cand != out)
                for (int t = lane; t < n_cand; t += 32) out[t] = cand[t];
            __syncwarp();
            if (p.shuffle)  // same keys (seed, global env id, draw_pos) and scratch (cold->raw + cold->tab_big) as the candidates kernel
                shuffle_candidates<SlotT>(out, n_cand, (uint64_t *)cold->raw, (SlotT *)((char *)cold->raw + 10240), p.seed, (uint64_t)(p.env_id_base + e),
                                          (uint64_t)h.draw_pos, lane);
            if (lane == 0) { s.n_cand = n_cand; s.fl = fl; }
        }
        __syncthreads();
        // ---- get_possible_position: first `nl` feasible candidates in order (the step's block-mode feasibility kernel) ----
        const int n_cand = s.n_cand;
        int fl = 0;
        const int n_leaf = first_feasible<EXPAND_THREADS / 32>(n_cand, nl, s.leaf, s.wb, [&](int c, int16_t *row) {
            int xs, ys, zs, rot, mh;
            key_unpack<KB>(out[c], xs, ys, zs, rot);
            const int sx = rt->d[rot][0], sy = rt->d[rot][1], sz = rt->d[rot][2];
            const bool feas = place_virtual_d<STAB>(p, sd.g, sd.pool, &cold->big, &s.s.lock, sx, sy, sz, xs, ys, den, mh, fl) != 0;
            row[0] = (int16_t)xs; row[1] = (int16_t)ys; row[2] = (int16_t)zs;
            row[3] = (int16_t)(xs + sx); row[4] = (int16_t)(ys + sy); row[5] = (int16_t)(zs + sz);
            return feas;
        });
        fl = __reduce_or_sync(FULL, fl);
        if (fl && lane == 0) atomicOr(&s.fl, fl);
        __syncthreads();
        // ---- the leaf rows of cur_observation (write_obs) and the record of pct_set_items ----
        OT *o = (OT *)x.leaves + (row + j) * (size_t)nl * 9;
#pragma unroll 1
        for (int f = tid; f < nl * 9; f += EXPAND_THREADS) {
            const int k = f / 9, col = f - k * 9;
            OT v = 0;
            if (k < n_leaf) {
                if (col < 5) v = (OT)s.leaf[k][col];
                else if (col == 5) v = (OT)p.H;
                else if (col == 8) v = 1;
            }
            o[f] = v;
        }
        if (tid == 0 && x.info) {
            pct_step_info info{};
            info.counter = n_box;
            info.flags = h.flags | s.fl;
            info.n_leaf = n_leaf; info.n_cand = n_cand; info.n_ems = h.n_ems;
            x.info[row + j] = info;
        }
        __syncthreads();  // the next item reuses the rotation table, the leaves and the candidate scratch
    }
}

template <typename OT, bool STAB>
__global__ void __launch_bounds__(EXPAND_THREADS) pctc_expand_kernel(const CParams p, const ExpandParams x) {
    __shared__ uint32_t tabA[CC_TAB], tabB[512];
    __shared__ uint64_t stg_h[32], rs_h[32];
    __shared__ uint32_t rs_c[32];
    __shared__ uint16_t stg_c[32];
    __shared__ double leaf[NL_MAX][6];
    __shared__ uint32_t wb[EXPAND_THREADS / 32];
    __shared__ int lock, s_fl, s_cnt;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, r = blockIdx.x, K = x.k, nl = p.nl;
    const int e = x.env ? x.env[r] : r;
    const size_t row = (size_t)r * K;
    if (e < 0 || e >= p.n_envs) { expand_zero_row<OT>(x, nl, row, tid); return; }
    CEnv *ev = p.env + e;
    const CHdr &h = ev->h;
    if (tid == 0) lock = 0;
    const int R = p.setting == 2 ? 6 : 2, n_ems = h.n_ems, n_box = h.n_box;
    GeomC g{ev->box, ev->den, n_box};
    EdgePool pool{ev->e_lower, ev->e_next, ev->e_off, ev->first_in, ev->last_in, ev->e_st, ev->e_st, h.n_edge,
                  ev->poly_off, &ev->poly[0][0], &ev->poly[0][0], h.n_poly};
#pragma unroll 1
    for (int j = 0; j < K; j++) {
        const double *it = (const double *)x.items + (row + j) * 3;
        const double nb[3] = {it[0], it[1], it[2]};
        const double den = x.density ? x.density[row + j] : h.next_den;
        if (warp == 0) {
            int fl = 0;
            PCTC_CANDIDATES_BODY
            if (lane == 0) { s_cnt = cnt; s_fl = fl; }
        }
        __syncthreads();
        // ---- get_possible_position (the step's block-mode feasibility kernel, pctc_feas_emit_kernel) ----
        const int n_cand = s_cnt;
        int fl = 0;
        const int n_leaf = first_feasible<EXPAND_THREADS / 32>(n_cand, nl, leaf, wb, [&](int c, double *t6) {
            cand_tuple(ev->cand[c], ev->ems, nb, t6);
            double mh;
            return place_virtual_c<STAB>(p, g, pool, &ev->big, &lock, t6[3] - t6[0], t6[4] - t6[1], t6[5] - t6[2], t6[0], t6[1], den, mh, fl) != 0;
        });
        fl = __reduce_or_sync(FULL, fl);
        if (fl && lane == 0) atomicOr(&s_fl, fl);
        __syncthreads();
        OT *o = (OT *)x.leaves + (row + j) * (size_t)nl * 9;
#pragma unroll 1
        for (int f = tid; f < nl * 9; f += EXPAND_THREADS) {  // write_obs_c's leaf rows
            const int k = f / 9, col = f - k * 9;
            double v = 0;
            if (k < n_leaf) {
                if (col < 5) v = leaf[k][col];
                else if (col == 5) v = p.H;
                else if (col == 8) v = 1;
            }
            o[f] = (OT)v;
        }
        if (tid == 0 && x.info) {
            pct_step_info info{};
            info.counter = n_box;
            info.flags = h.flags | s_fl;
            info.n_leaf = n_leaf; info.n_cand = n_cand; info.n_ems = n_ems;
            x.info[row + j] = info;
        }
        __syncthreads();
    }
}

template <typename OT>
static void expand_discrete(const DParams &p, const ExpandParams &x, cudaStream_t st) {
    const bool stab = p.setting != 2, small = p.W <= 16 && p.L <= 16 && p.H <= 16;  // the candidate key width of the step (launch_s)
    if (small) {
        if (stab) pct_expand_kernel<OT, true, uint16_t><<<x.n, EXPAND_THREADS, 0, st>>>(p, x);
        else pct_expand_kernel<OT, false, uint16_t><<<x.n, EXPAND_THREADS, 0, st>>>(p, x);
    } else {
        if (stab) pct_expand_kernel<OT, true, uint32_t><<<x.n, EXPAND_THREADS, 0, st>>>(p, x);
        else pct_expand_kernel<OT, false, uint32_t><<<x.n, EXPAND_THREADS, 0, st>>>(p, x);
    }
}

cudaError_t launch_expand_discrete(const DParams &p, const ExpandParams &x, cudaStream_t st) {
    if (p.obs_f64) expand_discrete<double>(p, x, st);
    else expand_discrete<float>(p, x, st);
    return cudaGetLastError();
}

cudaError_t launch_expand_continuous(const CParams &p, const ExpandParams &x, cudaStream_t st) {
    const bool stab = p.setting != 2;
    if (p.obs_f64) {
        if (stab) pctc_expand_kernel<double, true><<<x.n, EXPAND_THREADS, 0, st>>>(p, x);
        else pctc_expand_kernel<double, false><<<x.n, EXPAND_THREADS, 0, st>>>(p, x);
    } else {
        if (stab) pctc_expand_kernel<float, true><<<x.n, EXPAND_THREADS, 0, st>>>(p, x);
        else pctc_expand_kernel<float, false><<<x.n, EXPAND_THREADS, 0, st>>>(p, x);
    }
    return cudaGetLastError();
}

}  // namespace pct
