// Buffered packing (pct_set_buffer / pct_buffer_*, include/pct_b200.h; DESIGN.md section 18): every env holds B items, and one step picks
// the item and its placement by a flat index j * NL + l into the leaf blocks of all B items.
//
// A step is four launches in plain stream order:
//   select   warp / env             decode (j, l); buffer item j becomes the env's current item (as pct_set_items writes it, without an
//                                   expansion) and stored leaf block j the env's leaf list; l goes to the apply kernel's leaf index
//   apply    the step's own kernel  (pct_discrete.cu / pct_continuous.cu, unchanged) placement, reward, done, info, the draw on success,
//                                   the auto-reset
//   refill   thread / env           slot j <- the draw the step consumed; after a reset, slot 0 <- the reset's draw and B - 1 more draws
//   expand   block / (env, slot)    the leaves of the slot's item on the env's new state with the leaf expansion's routines (stage_env_d,
//                                   build_candidates and the generators / PCTC_CANDIDATES_BODY, shuffle_candidates, place_virtual_d / _c,
//                                   first_feasible); the stored leaf block, every observation row of the slot, the record's sums
// The refill is a kernel of its own because the slots' blocks all read the env's final draw position (the shuffle key).  A reset is the apply
// kernel's reset mode followed by refill and expand.
//
// Scratch of the expansion: the slots of one env run in different blocks, so each slot has its own candidate list and generator / shuffle
// scratch (BufSlotD / BufSlotC); the rare many-support visits of all of them share the env's BigScratch under the env's lock (DEnvCold::lock,
// CEnv::lock), as the pooled walks of a step do.  The env record is only read, but for the sums and the sticky flags (atomics).
//
// SEL (pct_buffer_step_envs / pct_buffer_reset_envs): every kernel runs over the slots of an EnvSel (SelParams, pct_kernels.h) and touches
// the selected envs alone; the apply kernel / the reset kernel run in their own SEL instantiations.
//
// Item override (pct_buffer_set_items; DESIGN.md section 21): the set kernel writes the caller's B items of each listed env in the refill
// kernel's place, then the SEL expansion re-expands all B slots of those envs.  Unchanged slots come out bit-identical (same state, same
// draw position, so the same shuffle keys); all of them are re-expanded because the header's n_cand is a sum over the slots.
//
// Heuristic baselines (pct_buffer_heuristic_actions*; DESIGN.md section 22): the plain baselines' selection (heur_select / heur_select_c) in one
// block per (env, slot) on the slot's item, a per-slot result in the slot's scratch, and a pick kernel per env.  pct_buffer_step_rows runs the
// row select kernel in the select kernel's place; apply, refill and expansion are the step's.  In this translation unit, beside the expansion,
// because the selections share the env's BigScratch under the env's lock as the expansion does.
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
#include "pct_draw.cuh"
#include "pct_buf_obs.cuh"
// the heuristic selections of pct_buffer_heuristic_actions*: a block of BUF_THREADS threads per (env, slot)
namespace pct { constexpr int FEAS_THREADS = 64; }
#include "pct_heur_select.cuh"
#include "pct_heur_select_c.cuh"

// 1: one block per env takes its slots in turn (the layout of pct_expand_kernel); 0: one block per (env, slot).  A/B guard of the measurement
// in DESIGN.md section 18, not an option of the library.
#ifndef BUF_SLOTS_INTURN
#define BUF_SLOTS_INTURN 0
#endif

namespace pct {

constexpr int BUF_THREADS = 64;

// flat leaf index -> (slot, leaf index of the slot); outside [0, B * nl): slot 0 with the zero action of a plain step
__device__ __forceinline__ void buf_decode(int d, int B, int nl, int &j, int &l) {
    if (d < 0 || d >= B * nl) { j = 0; l = -1; }
    else { j = d / nl; l = d - j * nl; }
}

// ---- select ----------------------------------------------------------------------------------------------------------------------
template <bool SEL = false>
__global__ void __launch_bounds__(256) pct_buf_select_kernel(const ParamsT<DParams, SEL> p, const BufParams b) {
    const int slot = (blockIdx.x * 256 + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    int e = slot;
    if constexpr (SEL) {
        e = sel_env(p.sel, p.n_envs, slot);
        if (e < 0) return;  // the whole warp
    } else if (e >= p.n_envs) return;  // the whole warp
    int j, l;
    buf_decode(b.flat[e], b.B, p.nl, j, l);
    const size_t s = (size_t)e * b.B + j;
    const int n = b.n_leaf[s];
    const int16_t *src = (const int16_t *)b.leaf + s * NL_MAX * 6;
    int16_t *dst = &p.cold[e].leaf[0][0];
    for (int t = lane; t < n * 6; t += 32) dst[t] = src[t];
    if (lane == 0) {
        DHdr &h = p.hot[e].h;
        const double *it = b.items + s * 4;
        h.next_box[0] = (int)it[0]; h.next_box[1] = (int)it[1]; h.next_box[2] = (int)it[2];  // what draw_item wrote into the header
        h.next_den = it[3];
        h.n_leaf = n;
        b.l[e] = l;
    }
}

template <bool SEL = false>
__global__ void __launch_bounds__(256) pctc_buf_select_kernel(const ParamsT<CParams, SEL> p, const BufParams b) {
    const int slot = (blockIdx.x * 256 + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    int e = slot;
    if constexpr (SEL) {
        e = sel_env(p.sel, p.n_envs, slot);
        if (e < 0) return;
    } else if (e >= p.n_envs) return;
    int j, l;
    buf_decode(b.flat[e], b.B, p.nl, j, l);
    const size_t s = (size_t)e * b.B + j;
    const int n = b.n_leaf[s];
    const double *src = (const double *)b.leaf + s * NL_MAX * 6;
    CEnv *ev = p.env + e;
    double *dst = &ev->leaf[0][0];
    for (int t = lane; t < n * 6; t += 32) dst[t] = src[t];
    if (lane == 0) {
        const double *it = b.items + s * 4;
        ev->h.next_box[0] = it[0]; ev->h.next_box[1] = it[1]; ev->h.next_box[2] = it[2];
        ev->h.next_den = it[3];
        ev->h.n_leaf = n;
        b.l[e] = l;
    }
}

// ---- select by slot and row (pct_buffer_step_rows) ----------------------------------------------------------------------------------
// Warp / env, as the select kernel: slot slots[e] (outside [0, B): slot 0) becomes the env's current item and leaf list.  The caller's row
// goes to the apply kernel as a float64 row in `act` (a float32 row converts exactly, as the apply kernel converts it; outside: the zero
// action), and b.l[e] = slot * NL, a flat index the refill kernel decodes back into the slot.
__device__ __forceinline__ int buf_take_row(const BufParams &b, int e, int nl, const int32_t *slots, const void *rows, int rows_f64, double *act,
                                            int lane) {
    const int s = slots[e];
    const bool in = s >= 0 && s < b.B;
    const int j = in ? s : 0;
    if (lane < 9) {
        const size_t q = (size_t)e * 9 + lane;
        act[q] = !in ? 0.0 : rows_f64 ? ((const double *)rows)[q] : (double)((const float *)rows)[q];
    }
    if (lane == 0) b.l[e] = j * nl;
    return j;
}

__global__ void __launch_bounds__(256) pct_buf_select_rows_kernel(const DParams p, const BufParams b, const int32_t *slots, const void *rows,
                                                                  int rows_f64, double *act) {
    const int e = (blockIdx.x * 256 + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (e >= p.n_envs) return;  // the whole warp
    const int j = buf_take_row(b, e, p.nl, slots, rows, rows_f64, act, lane);
    const size_t s = (size_t)e * b.B + j;
    const int n = b.n_leaf[s];
    const int16_t *src = (const int16_t *)b.leaf + s * NL_MAX * 6;
    int16_t *dst = &p.cold[e].leaf[0][0];
    for (int t = lane; t < n * 6; t += 32) dst[t] = src[t];
    if (lane == 0) {
        DHdr &h = p.hot[e].h;
        const double *it = b.items + s * 4;
        h.next_box[0] = (int)it[0]; h.next_box[1] = (int)it[1]; h.next_box[2] = (int)it[2];
        h.next_den = it[3];
        h.n_leaf = n;
    }
}

__global__ void __launch_bounds__(256) pctc_buf_select_rows_kernel(const CParams p, const BufParams b, const int32_t *slots, const void *rows,
                                                                   int rows_f64, double *act) {
    const int e = (blockIdx.x * 256 + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (e >= p.n_envs) return;
    const int j = buf_take_row(b, e, p.nl, slots, rows, rows_f64, act, lane);
    const size_t s = (size_t)e * b.B + j;
    const int n = b.n_leaf[s];
    const double *src = (const double *)b.leaf + s * NL_MAX * 6;
    CEnv *ev = p.env + e;
    double *dst = &ev->leaf[0][0];
    for (int t = lane; t < n * 6; t += 32) dst[t] = src[t];
    if (lane == 0) {
        const double *it = b.items + s * 4;
        ev->h.next_box[0] = it[0]; ev->h.next_box[1] = it[1]; ev->h.next_box[2] = it[2];
        ev->h.next_den = it[3];
        ev->h.n_leaf = n;
    }
}

// ---- refill ----------------------------------------------------------------------------------------------------------------------
// slot j <- the header's item (the draw the step consumed, or the reset's draw in slot 0 and B - 1 more draws); the header keeps the item it
// had before the extra draws.  Zeroes the header's leaf / candidate counts, which the expansion sums over the slots.
template <typename P, typename Hdr, typename Draw>
__device__ __forceinline__ void buf_refill(const P &p, const BufParams &b, int e, Hdr &h, Draw draw) {
    double *it = b.items + (size_t)e * b.B * 4;
    auto put = [&](int j) {
        it[j * 4 + 0] = (double)h.next_box[0]; it[j * 4 + 1] = (double)h.next_box[1]; it[j * 4 + 2] = (double)h.next_box[2];
        it[j * 4 + 3] = h.next_den;
    };
    if (!b.done || b.done[e]) {
        put(0);
        const Hdr h0 = h;
        for (int j = 1; j < b.B; j++) {
            draw(h);
            put(j);
        }
        const int64_t dp = h.draw_pos;
        h = h0;
        h.draw_pos = dp;
    } else {
        int j, l;
        buf_decode(b.flat[e], b.B, p.nl, j, l);
        put(j);
    }
    h.n_leaf = 0;
    h.n_cand = 0;
}

template <bool SEL = false>
__global__ void __launch_bounds__(128) pct_buf_refill_kernel(const ParamsT<DParams, SEL> p, const BufParams b) {
    int e = blockIdx.x * 128 + threadIdx.x;
    if constexpr (SEL) {
        e = sel_env(p.sel, p.n_envs, e);
        if (e < 0) return;
    } else if (e >= p.n_envs) return;
    DHdr h = p.hot[e].h;
    buf_refill(p, b, e, h, [&](DHdr &hh) { draw_item(p, e, hh); });
    p.hot[e].h = h;
}

template <bool SEL = false>
__global__ void __launch_bounds__(128) pctc_buf_refill_kernel(const ParamsT<CParams, SEL> p, const BufParams b) {
    int e = blockIdx.x * 128 + threadIdx.x;
    if constexpr (SEL) {
        e = sel_env(p.sel, p.n_envs, e);
        if (e < 0) return;
    } else if (e >= p.n_envs) return;
    CHdr h = p.env[e].h;
    buf_refill(p, b, e, h, [&](CHdr &hh) { draw_item_c(p, e, hh); });
    p.env[e].h = h;
}

// ---- set (pct_buffer_set_items) --------------------------------------------------------------------------------------------------
// In the refill kernel's place: slot j of env d_env[i] <- item j of row i, without a draw.  Discrete sizes are truncated and clamped to
// [0, 255] (the range pct_set_items clamps to: no container side is larger); the density is taken as given.  Zeroes the header's leaf /
// candidate counts, which the expansion sums over the slots, and writes the record's fixed fields as pct_set_items_kernel does (counter,
// sticky flags, zeros): the expansion adds its sums and flags.  Thread / selection slot; the row of slot i is row i.
template <typename Hdr>
__device__ __forceinline__ void buf_set(const BufParams &b, int e, const double *row, Hdr &h, bool disc) {
    double *it = b.items + (size_t)e * b.B * 4;
    for (int q = 0; q < b.B * 4; q++) {
        const double v = row[q];
        it[q] = disc && (q & 3) != 3 ? fmin(fmax(trunc(v), 0.0), 255.0) : v;
    }
    h.n_leaf = 0;
    h.n_cand = 0;
    if (b.info) {
        pct_step_info info{};
        info.counter = h.n_box;
        info.flags = h.flags;
        b.info[e] = info;
    }
}

__global__ void __launch_bounds__(128) pct_buf_set_kernel(const SelParams<DParams> p, const BufParams b, const double *rows) {
    const int i = blockIdx.x * 128 + threadIdx.x, e = sel_env(p.sel, p.n_envs, i);
    if (e < 0) return;
    buf_set(b, e, rows + (size_t)i * b.B * 4, p.hot[e].h, true);
}

__global__ void __launch_bounds__(128) pctc_buf_set_kernel(const SelParams<CParams> p, const BufParams b, const double *rows) {
    const int i = blockIdx.x * 128 + threadIdx.x, e = sel_env(p.sel, p.n_envs, i);
    if (e < 0) return;
    buf_set(b, e, rows + (size_t)i * b.B * 4, p.env[e].h, false);
}

// ---- expand ----------------------------------------------------------------------------------------------------------------------
// the slots of block blockIdx.x: (env or selection slot, first slot, end)
__device__ __forceinline__ void buf_slots(int B, int &e, int &j0, int &j1) {
    if (BUF_SLOTS_INTURN) { e = blockIdx.x; j0 = 0; j1 = B; }
    else { e = blockIdx.x / B; j0 = blockIdx.x - e * B; j1 = j0 + 1; }
}

// leaf block j of the observation and the stored block, the item row of slot j, and the slot's share of the record and header sums
template <typename OT, typename LT, typename Hdr>
__device__ __forceinline__ void buf_emit_slot(const BufParams &b, int nb, int nl, double H, int e, int j, OT *obs, const LT (*leaf)[6], int n_leaf,
                                              int n_cand, int fl, int flags_now, int n_ems, const double sz[3], double den, Hdr *gh, int tid) {
    const int B = b.B;
    OT *o = obs + (size_t)(nb + j * nl) * 9;
    BUF_LEAF_ROWS(OT, o, leaf, n_leaf, nl, H, tid, BUF_THREADS)
    LT *dst = (LT *)b.leaf + ((size_t)e * B + j) * NL_MAX * 6;
    for (int t = tid; t < n_leaf * 6; t += BUF_THREADS) dst[t] = (&leaf[0][0])[t];
    buf_item_row<OT>(obs + (size_t)(nb + B * nl + j) * 9, sz, den, tid);
    if (tid == 0) {
        b.n_leaf[(size_t)e * B + j] = n_leaf;
        atomicAdd(&gh->n_leaf, n_leaf);
        atomicAdd(&gh->n_cand, n_cand);
        if (fl) atomicOr(&gh->flags, fl);
        if (b.info) {
            pct_step_info *r = b.info + e;
            atomicAdd(&r->n_leaf, n_leaf);
            atomicAdd(&r->n_cand, n_cand);
            atomicOr(&r->flags, flags_now | fl);
            if (j == 0) r->n_ems = n_ems;
        }
    }
}

template <typename SlotT>
struct BufSmD {
    StageD s;
    SlotT tabA[TAB_A], tabB[TAB_B];
    SetStage stg;
    int16_t leaf[NL_MAX][6];
    RotTab rt;
    int fl, n_cand;
    uint32_t wb[BUF_THREADS / 32];
};

template <typename OT, bool STAB, typename SlotT, bool SEL = false>
__global__ void __launch_bounds__(BUF_THREADS) pct_buf_expand_kernel(const ParamsT<DParams, SEL> p, const BufParams b) {
    constexpr int KB = sizeof(SlotT) == 2 ? 4 : 8;
    __shared__ __align__(16) BufSmD<SlotT> s;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, B = b.B, nl = p.nl, nb = p.nb;
    int e, j0, j1;
    buf_slots(B, e, j0, j1);
    if constexpr (SEL) {
        e = sel_env(p.sel, p.n_envs, e);
        if (e < 0) return;  // the whole block
    }
    DEnvCold *cold = p.cold + e;
    StagedD sd = stage_env_d<STAB>(s.s, p, e, false);
    const DEnvHot *hot = &s.s.hot;
    const DHdr &h = hot->h;
    const int n_box = h.n_box, R = p.setting == 2 ? 6 : 2;
    const RotTab *rt = &s.rt;
    OT *obs = (OT *)b.obs + (size_t)e * (size_t)((nb + B * nl + B) * 9);
    if (j0 == 0) buf_internal_rows_d<OT, BUF_THREADS>(obs, hot, cold, nb, n_box, p.setting, tid);
#pragma unroll 1
    for (int j = j0; j < j1; j++) {
        BufSlotD *sc = (BufSlotD *)b.scratch + (size_t)e * B + j;
        SlotT *const out = (SlotT *)sc->cand;
        const double *itd = b.items + ((size_t)e * B + j) * 4;
        const int nb3[3] = {(int)itd[0], (int)itd[1], (int)itd[2]};
        const double den = itd[3];
        if (warp == 0) {
            // ---- the candidates kernel's list for this item, as pct_expand_kernel builds it ----
            if (lane == 0) make_rot_tab(nb3, R, s.rt);
            __syncwarp();
            SlotT *cand = nullptr;
            int fl = 0, n_cand = 0;
            if (p.lnes == 0) {
                const CandList<SlotT> cl = build_candidates<SlotT>(hot->ems, h.n_ems, rt, R, s.tabA, s.tabB, s.tabA, &s.stg, lane);
                cand = cl.keys; n_cand = cl.n; fl = cl.flags;
            } else if (p.lnes == 5) {
                const CandList<SlotT> cl = gen_event_point_m<SlotT>(hot, rt, R, p.W, p.L, p.H, s.tabA, s.tabB, s.tabA,
                                                                    sc->raw, out, lane);
                cand = cl.keys; n_cand = cl.n; fl = cl.flags;
            } else {
                uint32_t *raw = sc->raw;
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
            if (p.shuffle)  // the step's keys (seed, global env id, draw_pos) on the slot's scratch (raw + tab_big, as the candidates kernel)
                shuffle_candidates<SlotT>(out, n_cand, (uint64_t *)sc->raw, (SlotT *)((char *)sc->raw + 10240), p.seed, (uint64_t)(p.env_id_base + e),
                                          (uint64_t)h.draw_pos, lane);
            if (lane == 0) { s.n_cand = n_cand; s.fl = fl; }
        }
        __syncthreads();
        // ---- get_possible_position: first `nl` feasible candidates in order ----
        const int n_cand = s.n_cand;
        int fl = 0;
        const int n_leaf = first_feasible<BUF_THREADS / 32>(n_cand, nl, s.leaf, s.wb, [&](int c, int16_t *row) {
            int xs, ys, zs, rot, mh;
            key_unpack<KB>(out[c], xs, ys, zs, rot);
            const int sx = rt->d[rot][0], sy = rt->d[rot][1], sz = rt->d[rot][2];
            const bool feas = place_virtual_d<STAB>(p, sd.g, sd.pool, &cold->big, &cold->lock, sx, sy, sz, xs, ys, den, mh, fl) != 0;
            row[0] = (int16_t)xs; row[1] = (int16_t)ys; row[2] = (int16_t)zs;
            row[3] = (int16_t)(xs + sx); row[4] = (int16_t)(ys + sy); row[5] = (int16_t)(zs + sz);
            return feas;
        });
        fl = __reduce_or_sync(FULL, fl);
        if (fl && lane == 0) atomicOr(&s.fl, fl);
        __syncthreads();
        const double sz[3] = {(double)nb3[0], (double)nb3[1], (double)nb3[2]};
        buf_emit_slot<OT, int16_t>(b, nb, nl, (double)p.H, e, j, obs, s.leaf, n_leaf, n_cand, s.fl, h.flags, h.n_ems, sz, den, &p.hot[e].h, tid);
        __syncthreads();  // the next slot reuses the rotation table, the leaves and the flags
    }
}

template <typename OT, bool STAB, bool SEL = false>
__global__ void __launch_bounds__(BUF_THREADS) pctc_buf_expand_kernel(const ParamsT<CParams, SEL> p, const BufParams b) {
    __shared__ uint32_t tabA[CC_TAB], tabB[512];
    __shared__ uint64_t stg_h[32], rs_h[32];
    __shared__ uint32_t rs_c[32];
    __shared__ uint16_t stg_c[32];
    __shared__ double leaf[NL_MAX][6];
    __shared__ uint32_t wb[BUF_THREADS / 32];
    __shared__ int s_fl, s_cnt;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, B = b.B, nl = p.nl, NB = p.nb;
    int e, j0, j1;
    buf_slots(B, e, j0, j1);
    if constexpr (SEL) {
        e = sel_env(p.sel, p.n_envs, e);
        if (e < 0) return;  // the whole block
    }
    CEnv *env = p.env + e;
    const CHdr &h = env->h;
    const int R = p.setting == 2 ? 6 : 2, n_ems = h.n_ems, n_box = h.n_box, flags_now = h.flags;
    GeomC g{env->box, env->den, n_box};
    EdgePool pool{env->e_lower, env->e_next, env->e_off, env->first_in, env->last_in, env->e_st, env->e_st, h.n_edge,
                  env->poly_off, &env->poly[0][0], &env->poly[0][0], h.n_poly};
    OT *obs = (OT *)b.obs + (size_t)e * (size_t)((NB + B * nl + B) * 9);
    if (j0 == 0) buf_internal_rows_c<OT, BUF_THREADS>(obs, env, NB, n_box, tid);
#pragma unroll 1
    for (int j = j0; j < j1; j++) {
        BufSlotC *sc = (BufSlotC *)b.scratch + (size_t)e * B + j;
        // PCTC_CANDIDATES_BODY reads the env's EMS list through `ev` and writes the list and the shuffle scratch through it: here the slot's own
        struct SlotView {
            const double (&ems)[CE_MAX][6];
            uint16_t (&cand)[1232];
            double (&ems_tmp)[265][6];
        } view{env->ems, sc->cand, sc->shuf};
        const SlotView *ev = &view;
        const double *itd = b.items + ((size_t)e * B + j) * 4;
        const double nb[3] = {itd[0], itd[1], itd[2]};
        const double den = itd[3];
        if (warp == 0) {
            int fl = 0;
            PCTC_CANDIDATES_BODY
            if (lane == 0) { s_cnt = cnt; s_fl = fl; }
        }
        __syncthreads();
        const int n_cand = s_cnt;
        int fl = 0;
        const int n_leaf = first_feasible<BUF_THREADS / 32>(n_cand, nl, leaf, wb, [&](int c, double *t6) {
            cand_tuple(sc->cand[c], env->ems, nb, t6);
            double mh;
            return place_virtual_c<STAB>(p, g, pool, &env->big, &env->lock, t6[3] - t6[0], t6[4] - t6[1], t6[5] - t6[2], t6[0], t6[1], den, mh, fl) != 0;
        });
        fl = __reduce_or_sync(FULL, fl);
        if (fl && lane == 0) atomicOr(&s_fl, fl);
        __syncthreads();
        buf_emit_slot<OT, double>(b, NB, nl, p.H, e, j, obs, leaf, n_leaf, n_cand, s_fl, flags_now, n_ems, nb, den, &env->h, tid);
        __syncthreads();
    }
}

// ---- policy and items ------------------------------------------------------------------------------------------------------------
__global__ void pct_buf_policy_random_kernel(const BufParams b, int n_envs, int nl, int64_t env_id_base, uint64_t seed, const int64_t *t_dev,
                                             int32_t *idx) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_envs) return;
    const int32_t *nlf = b.n_leaf + (size_t)e * b.B;
    int total = 0;
    for (int j = 0; j < b.B; j++) total += nlf[j];
    if (total == 0) { idx[e] = 0; return; }
    int k = (int)(rnd_u64(seed, (uint64_t)(env_id_base + e), (uint64_t)*t_dev) % (uint64_t)total), j = 0;
    while (k >= nlf[j]) { k -= nlf[j]; j++; }
    idx[e] = j * nl + k;
}

__global__ void pct_buf_items_kernel(const BufParams b, int n_envs, const int32_t *env, int n, double *out) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (int64_t)n * b.B * 4) return;
    const int r = (int)(t / (b.B * 4)), q = (int)(t - (int64_t)r * b.B * 4);
    const int e = env ? env[r] : r;
    out[t] = (e >= 0 && e < n_envs) ? b.items[(size_t)e * b.B * 4 + q] : 0.0;
}

// ---- launchers -------------------------------------------------------------------------------------------------------------------
// sel non-null: the selected launches (pct_buffer_step_envs / pct_buffer_reset_envs) over sel->slots(n_envs) slots
static unsigned buf_blocks(int slots, int B) { return BUF_SLOTS_INTURN ? (unsigned)slots : (unsigned)slots * (unsigned)B; }

template <typename P>
static SelParams<P> with_sel(const P &p, const EnvSel &sel) {
    SelParams<P> ps;
    static_cast<P &>(ps) = p;
    ps.sel = sel;
    return ps;
}

cudaError_t launch_buffer_select_discrete(const DParams &p, const BufParams &b, cudaStream_t st, const EnvSel *sel) {
    if (sel) pct_buf_select_kernel<true><<<(sel->slots(p.n_envs) + 7) / 8, 256, 0, st>>>(with_sel(p, *sel), b);
    else pct_buf_select_kernel<<<(p.n_envs + 7) / 8, 256, 0, st>>>(p, b);
    return cudaGetLastError();
}

cudaError_t launch_buffer_select_continuous(const CParams &p, const BufParams &b, cudaStream_t st, const EnvSel *sel) {
    if (sel) pctc_buf_select_kernel<true><<<(sel->slots(p.n_envs) + 7) / 8, 256, 0, st>>>(with_sel(p, *sel), b);
    else pctc_buf_select_kernel<<<(p.n_envs + 7) / 8, 256, 0, st>>>(p, b);
    return cudaGetLastError();
}

cudaError_t launch_buffer_select_rows_discrete(const DParams &p, const BufParams &b, const int32_t *slots, const void *rows, int rows_f64, double *act,
                                               cudaStream_t st) {
    pct_buf_select_rows_kernel<<<(p.n_envs + 7) / 8, 256, 0, st>>>(p, b, slots, rows, rows_f64, act);
    return cudaGetLastError();
}

cudaError_t launch_buffer_select_rows_continuous(const CParams &p, const BufParams &b, const int32_t *slots, const void *rows, int rows_f64,
                                                 double *act, cudaStream_t st) {
    pctc_buf_select_rows_kernel<<<(p.n_envs + 7) / 8, 256, 0, st>>>(p, b, slots, rows, rows_f64, act);
    return cudaGetLastError();
}

template <typename OT, bool STAB, bool SEL>
static void expand_d(const ParamsT<DParams, SEL> &p, const BufParams &b, cudaStream_t st, unsigned g) {
    const bool small = p.W <= 16 && p.L <= 16 && p.H <= 16;  // the candidate key width of the step (launch_s)
    if (small) pct_buf_expand_kernel<OT, STAB, uint16_t, SEL><<<g, BUF_THREADS, 0, st>>>(p, b);
    else pct_buf_expand_kernel<OT, STAB, uint32_t, SEL><<<g, BUF_THREADS, 0, st>>>(p, b);
}

// the expansion of every slot of `slots` envs / selection slots; the refill or the set kernel has run before it
template <bool SEL>
static void expand_slots_d(const ParamsT<DParams, SEL> &p, const BufParams &b, cudaStream_t st, int slots) {
    const bool stab = p.setting != 2;
    const unsigned g = buf_blocks(slots, b.B);
    if (p.obs_f64) { if (stab) expand_d<double, true, SEL>(p, b, st, g); else expand_d<double, false, SEL>(p, b, st, g); }
    else { if (stab) expand_d<float, true, SEL>(p, b, st, g); else expand_d<float, false, SEL>(p, b, st, g); }
}

template <bool SEL>
static void buffer_expand_d(const ParamsT<DParams, SEL> &p, const BufParams &b, cudaStream_t st, int slots) {
    pct_buf_refill_kernel<SEL><<<(slots + 127) / 128, 128, 0, st>>>(p, b);
    expand_slots_d<SEL>(p, b, st, slots);
}

cudaError_t launch_buffer_expand_discrete(const DParams &p, const BufParams &b, cudaStream_t st, const EnvSel *sel) {
    if (sel) buffer_expand_d<true>(with_sel(p, *sel), b, st, sel->slots(p.n_envs));
    else buffer_expand_d<false>(p, b, st, p.n_envs);
    return cudaGetLastError();
}

template <bool SEL>
static void expand_slots_c(const ParamsT<CParams, SEL> &p, const BufParams &b, cudaStream_t st, int slots) {
    const bool stab = p.setting != 2;
    const unsigned g = buf_blocks(slots, b.B);
    if (p.obs_f64) {
        if (stab) pctc_buf_expand_kernel<double, true, SEL><<<g, BUF_THREADS, 0, st>>>(p, b);
        else pctc_buf_expand_kernel<double, false, SEL><<<g, BUF_THREADS, 0, st>>>(p, b);
    } else {
        if (stab) pctc_buf_expand_kernel<float, true, SEL><<<g, BUF_THREADS, 0, st>>>(p, b);
        else pctc_buf_expand_kernel<float, false, SEL><<<g, BUF_THREADS, 0, st>>>(p, b);
    }
}

template <bool SEL>
static void buffer_expand_c(const ParamsT<CParams, SEL> &p, const BufParams &b, cudaStream_t st, int slots) {
    pctc_buf_refill_kernel<SEL><<<(slots + 127) / 128, 128, 0, st>>>(p, b);
    expand_slots_c<SEL>(p, b, st, slots);
}

cudaError_t launch_buffer_expand_continuous(const CParams &p, const BufParams &b, cudaStream_t st, const EnvSel *sel) {
    if (sel) buffer_expand_c<true>(with_sel(p, *sel), b, st, sel->slots(p.n_envs));
    else buffer_expand_c<false>(p, b, st, p.n_envs);
    return cudaGetLastError();
}

cudaError_t launch_buffer_set_discrete(const DParams &p, const BufParams &b, const double *rows, cudaStream_t st, const EnvSel &sel) {
    const SelParams<DParams> ps = with_sel(p, sel);
    pct_buf_set_kernel<<<(sel.n + 127) / 128, 128, 0, st>>>(ps, b, rows);
    expand_slots_d<true>(ps, b, st, sel.n);
    return cudaGetLastError();
}

cudaError_t launch_buffer_set_continuous(const CParams &p, const BufParams &b, const double *rows, cudaStream_t st, const EnvSel &sel) {
    const SelParams<CParams> ps = with_sel(p, sel);
    pctc_buf_set_kernel<<<(sel.n + 127) / 128, 128, 0, st>>>(ps, b, rows);
    expand_slots_c<true>(ps, b, st, sel.n);
    return cudaGetLastError();
}

// ---- buffered envs (pct_buffer_heuristic_actions; DESIGN.md section 22) ------------------------------------------------------------
// One block per (env, slot), as pct_buf_expand_kernel: the selection for the slot's item on the env's state, written to the slot's BufHeurD.
template <bool STAB, bool BIG>
__global__ void __launch_bounds__(FEAS_THREADS, 4) pct_buf_heuristic_kernel(const DParams p, const HParams hp, const BufParams b) {
    const int e = blockIdx.x / b.B;
    const size_t s = (size_t)blockIdx.x;
    const HeurPick r = heur_select<STAB, BIG>(p, hp, e, b.items + s * 4, &p.cold[e].lock);
    if (threadIdx.x == 0) {
        BufHeurD *o = (BufHeurD *)((BufSlotD *)b.scratch + s)->raw;
        const int K = hp.code == PCT_H_MACS ? 4 : 1, R = p.setting == 2 ? 6 : 2;
        o->score = r.score;
        o->found = r.found;
        o->rank = hp.code <= PCT_H_MACS ? r.c / (R * K) : 0;
        o->lx = r.best.lx; o->ly = r.best.ly; o->sx = r.best.sx; o->sy = r.best.sy;
    }
}

// Thread / env: the slot by the rules of DESIGN.md section 22 (best score in the heuristic's direction, OnlineBPH the lowest EMS rank, ties to
// the lowest slot; RANDOM a uniform draw among the slots with a placement), its row, and LSAH's footprint of the chosen placement.  No slot
// with a placement: slot 0 and the "no placement" row.
__global__ void __launch_bounds__(128) pct_buf_heuristic_pick_kernel(const DParams p, const HParams hp, const BufParams b, int32_t *slots) {
    const int e = blockIdx.x * 128 + threadIdx.x;
    if (e >= p.n_envs) return;
    const int code = hp.code, B = b.B;
    const BufSlotD *sc = (const BufSlotD *)b.scratch + (size_t)e * B;
    auto res = [&](int j) -> const BufHeurD & { return *(const BufHeurD *)sc[j].raw; };
    int pick = -1;
    if (code == PCT_H_RANDOM) {
        int m = 0;
        for (int j = 0; j < B; j++) m += res(j).found != 0;
        if (m > 0) {
            int k = (int)(rnd_u64(hp.seed ^ BUF_SLOT_SALT, (uint64_t)(p.env_id_base + e), (uint64_t)hp.t) % (uint64_t)m);
            for (pick = 0; !res(pick).found || k-- > 0; pick++) {}
        }
    } else {
        for (int j = 0; j < B; j++) {
            const BufHeurD &r = res(j);
            if (!r.found) continue;
            bool take = pick < 0;
            if (!take) {
                const BufHeurD &q = res(pick);
                if (code == PCT_H_ONLINEBPH) take = r.rank < q.rank;
                else if (code == PCT_H_BR || code == PCT_H_MACS) take = r.score > q.score;
                else take = r.score < q.score;
            }
            if (take) pick = j;
        }
    }
    slots[e] = pick < 0 ? 0 : pick;
    const BufHeurD &r = res(pick < 0 ? 0 : pick);
    heur_row(hp.rows + (size_t)e * 9, pick >= 0, r.lx, r.ly, r.sx, r.sy);
    if (pick >= 0 && code == PCT_H_LSAH) {
        int32_t *s = hp.hstate + (size_t)e * 4;
        const bool fresh = p.hot[e].h.n_box == 0;
        lsah_note(s, fresh ? 0 : s[0], fresh ? 0 : s[1], fresh ? p.W : s[2], fresh ? p.L : s[3], r.lx, r.ly, r.sx, r.sy);
    }
}

cudaError_t launch_buffer_heuristic_discrete(const DParams &p, const HParams &hp, const BufParams &b, int32_t *slots, cudaStream_t st) {
    const unsigned g = (unsigned)p.n_envs * (unsigned)b.B;
    if (heur_big(p, hp.code)) {
        const size_t smem = heur_big_smem(p.W, p.L, p.setting == 2 ? 6 : 2);
        if (p.setting == 2) pct_buf_heuristic_kernel<false, true><<<g, FEAS_THREADS, smem, st>>>(p, hp, b);
        else pct_buf_heuristic_kernel<true, true><<<g, FEAS_THREADS, smem, st>>>(p, hp, b);
    } else if (p.setting == 2) pct_buf_heuristic_kernel<false, false><<<g, FEAS_THREADS, 0, st>>>(p, hp, b);
    else pct_buf_heuristic_kernel<true, false><<<g, FEAS_THREADS, 0, st>>>(p, hp, b);
    pct_buf_heuristic_pick_kernel<<<(p.n_envs + 127) / 128, 128, 0, st>>>(p, hp, b, slots);
    return cudaGetLastError();
}


// ---- buffered envs (pct_buffer_heuristic_actions_f64; DESIGN.md section 22): as pct_buf_heuristic_kernel / pct_buf_heuristic_pick_kernel ----
template <bool STAB>
__global__ void __launch_bounds__(64, STAB ? 8 : 12) pctc_buf_heuristic_kernel(const CParams p, const HParamsC hp, const BufParams b) {
    const int e = blockIdx.x / b.B;
    const size_t s = (size_t)blockIdx.x;
    const HeurPickC r = heur_select_c<STAB>(p, hp, e, b.items + s * 4, &p.env[e].lock);
    if (threadIdx.x == 0) {
        BufHeurC *o = (BufHeurC *)&((BufSlotC *)b.scratch + s)->shuf[0][0];
        o->score = r.score;
        o->found = r.found;
        o->rank = r.c / (p.setting == 2 ? 6 : 2);
        o->lx = r.best.lx; o->ly = r.best.ly; o->sx = r.best.sx; o->sy = r.best.sy;
    }
}

__global__ void __launch_bounds__(128) pctc_buf_heuristic_pick_kernel(const CParams p, const HParamsC hp, const BufParams b, int32_t *slots) {
    const int e = blockIdx.x * 128 + threadIdx.x;
    if (e >= p.n_envs) return;
    const int code = hp.code, B = b.B;
    const BufSlotC *sc = (const BufSlotC *)b.scratch + (size_t)e * B;
    auto res = [&](int j) -> const BufHeurC & { return *(const BufHeurC *)&sc[j].shuf[0][0]; };
    int pick = -1;
    for (int j = 0; j < B; j++) {
        const BufHeurC &r = res(j);
        if (!r.found) continue;
        bool take = pick < 0;
        if (!take) {
            const BufHeurC &q = res(pick);
            if (code == PCT_H_ONLINEBPH) take = r.rank < q.rank;
            else if (code == PCT_H_BR) take = r.score > q.score;
            else take = r.score < q.score;
        }
        if (take) pick = j;
    }
    slots[e] = pick < 0 ? 0 : pick;
    const BufHeurC &r = res(pick < 0 ? 0 : pick);
    heur_row_c(hp.rows + (size_t)e * 9, pick >= 0, p.W, r.lx, r.ly, r.sx, r.sy);
    if (pick >= 0 && code == PCT_H_LSAH) {
        double *s = hp.hstate + (size_t)e * 4;
        const bool fresh = p.env[e].h.n_box == 0;
        lsah_note_c(s, fresh ? 0 : s[0], fresh ? 0 : s[1], fresh ? p.W : s[2], fresh ? p.L : s[3], r.lx, r.ly, r.sx, r.sy);
    }
}

cudaError_t launch_buffer_heuristic_continuous(const CParams &p, const HParamsC &hp, const BufParams &b, int32_t *slots, cudaStream_t st) {
    const unsigned g = (unsigned)p.n_envs * (unsigned)b.B;
    if (p.setting == 2) pctc_buf_heuristic_kernel<false><<<g, 64, 0, st>>>(p, hp, b);
    else pctc_buf_heuristic_kernel<true><<<g, 64, 0, st>>>(p, hp, b);
    pctc_buf_heuristic_pick_kernel<<<(p.n_envs + 127) / 128, 128, 0, st>>>(p, hp, b, slots);
    return cudaGetLastError();
}

// the dynamic shared memory limit of the BIG instantiations, as prepare_heuristic_big raises the plain kernel's (pct_create of a discrete handle
// with W or L > 32; idempotent), so that launch_buffer_heuristic_discrete only enqueues
cudaError_t prepare_buffer_heuristic_big() {
    const int smem = (int)heur_big_smem(255, 255, 6);
    cudaError_t e = cudaFuncSetAttribute(pct_buf_heuristic_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(pct_buf_heuristic_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    return e;
}

cudaError_t launch_buffer_items(const BufParams &b, int n_envs, const int32_t *env, int n, double *out, cudaStream_t st) {
    const int64_t total = (int64_t)n * b.B * 4;
    pct_buf_items_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(b, n_envs, env, n, out);
    return cudaGetLastError();
}

cudaError_t launch_buffer_policy_random(const BufParams &b, int n_envs, int nl, int64_t env_id_base, uint64_t seed, const int64_t *t_dev,
                                        int32_t *idx, cudaStream_t st) {
    pct_buf_policy_random_kernel<<<(n_envs + 127) / 128, 128, 0, st>>>(b, n_envs, nl, env_id_base, seed, t_dev, idx);
    return cudaGetLastError();
}

}  // namespace pct
