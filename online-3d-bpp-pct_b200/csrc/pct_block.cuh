// The read-only placement test of each domain and the pieces every block-per-env kernel around it shares: the staged discrete env
// record and the ordered compaction of the first `nl` feasible candidates.  Callers: the step's block-mode feasibility kernels
// (pct_feas_emit_kernel, pctc_feas_emit_kernel), the leaf expansion (pct_expand.cu), the batched queries (pct_query.cuh,
// pctc_query_kernel) and the heuristic baselines (pct_heuristics*.cuh).  A fix to the placement rule lands here, once per domain.
#pragma once
#include "pct_common.cuh"
#include "pct_kernels.h"
#include "pct_stability.cuh"
#include "pct_geom.cuh"
#include "pct_geom_continuous.cuh"
#include "pct_continuous.cuh"

namespace pct {

// Space.drop_box_virtual(dims, (lx, ly), False, density, setting, returnH=True) + check_box (D:space.py:393-454) of ONE placement of an env
// whose boxes g holds: bounds, resting height, the height test, then the read-only stability check.  mh is the resting height, reported
// whatever the verdict.  Raised capacity flags are ORed into `fl`; prof: phase timers of the stability check (-DPCT_PHASE_TIMERS builds).
template <bool STAB>
__device__ __forceinline__ int place_virtual_d(const DParams &p, const GeomD &g, EdgePool &pool, BigScratch *big, int *lock, int sx, int sy, int sz,
                                               int lx, int ly, double den, int &mh, int &fl, long long *prof = nullptr) {
    mh = rest_height(g.box, 0, g.n, 1, lx, ly, lx + sx, ly + sy);
    if (lx + sx > p.W || ly + sy > p.L) return 0;
    if (mh + sz > p.H) return 0;
    if (!STAB || mh == 0) return 1;
    NodeD root{lx, ly, mh, sx, sy, sz, (double)(sx * sy * sz) * den};
    return stability_check<false, GeomD>(g, root, pool, big, lock, 0, fl, prof) != 0;
}

// The same for the continuous env (C:space.py:380-439), with the reference's 1e-6 tolerances.  mh is interSect2D's max_h (C:space.py:391).
// PRE: the resting height from the pre-rounded box rectangles rb (rest_height_pre; the step's feasibility kernel under PCT_B200_CONT_PRE).
template <bool STAB, bool PRE = false>
__device__ __forceinline__ int place_virtual_c(const CParams &p, const GeomC &g, EdgePool &pool, BigScratch *big, int *lock, double sx, double sy,
                                               double sz, double lx, double ly, double den, double &mh, int &fl, const double (*rb)[5] = nullptr) {
    bool chk = !(lx + sx - 1e-6 > p.W || ly + sy - 1e-6 > p.L) && !(lx + 1e-6 < 0 || ly + 1e-6 < 0);
    mh = PRE ? rest_height_pre(rb, g.n, around6(-lx), around6(-ly), around6(lx + sx), around6(ly + sy))
             : rest_height_c(g.box, 0, g.n, 1, lx, ly, lx + sx, ly + sy);
    if (mh < 0) mh = 0.0;
    if (mh + sz - 1e-6 > p.H) chk = false;
    if (!chk) return 0;
    if (!STAB || fabs(mh) < 1e-6) return 1;
    NodeC root{lx, ly, mh, sx, sy, sz, sx * sy * sz * den};
    return stability_check<false, GeomC>(g, root, pool, big, lock, 0, fl) != 0;
}

// A discrete env record staged in shared memory: the record (TMA bulk copy), the first load edges and polygon vertices the stability
// check reads through EdgePool, the mbarrier of the copies and the lock of the env's `big` scratch.
struct StageD {
    DEnvHot hot;
    alignas(16) Stack4 st[EDGE_STAGE];
    alignas(16) double poly[POLY_STAGE * 2];
    uint64_t mbar;
    int lock;
};

// What the placement test reads of a staged env: its boxes (and setting-3 densities) and its load edges.
struct StagedD {
    GeomD g;
    EdgePool pool;
};

// Stages env e into s: phase 0 of the mbarrier copies the record; phase 1 the edges and vertices (stability settings, only when the env
// has load edges).  handover: first wait for the candidates kernel's hand-over of the env (the step's overlapped launches, p.ready).
// Every thread of the block calls it; thread 0 may write other shared variables before the call, the first barrier inside publishes them.
template <bool STAB>
__device__ __forceinline__ StagedD stage_env_d(StageD &s, const DParams &p, int e, bool handover) {
    const int tid = threadIdx.x;
    DEnvHot *ghot = p.hot + e;
    DEnvCold *cold = p.cold + e;
    if (tid == 0) {
        s.lock = 0;
        mbar_init(&s.mbar, 1);
        fence_proxy_async();
    }
    __syncthreads();
    if (tid == 0) {
        if (handover && p.ready) {
            if (!env_wait(p.ready + p.n_envs + e, p.epoch)) atomicOr(&ghot->h.flags, PCT_FLAG_SYNC_TIMEOUT);
            fence_proxy_async_all();
        }
        mbar_expect_tx(&s.mbar, (uint32_t)sizeof(DEnvHot));
        tma_load_1d(&s.hot, ghot, (uint32_t)sizeof(DEnvHot), &s.mbar);
    }
    mbar_wait(&s.mbar, 0);
    __syncthreads();  // every thread must have observed phase 0 before the barrier is re-armed
    const DHdr &h = s.hot.h;
    if (STAB && h.n_edge > 0) {
        const uint32_t bytes = (uint32_t)min(h.n_edge, EDGE_STAGE) * (uint32_t)sizeof(Stack4);
        const uint32_t pbytes = (uint32_t)min(h.n_poly, POLY_STAGE) * 16u;
        if (tid == 0) {
            mbar_expect_tx(&s.mbar, bytes + pbytes);
            tma_load_1d(s.st, cold->e_st, bytes, &s.mbar);
            if (pbytes) tma_load_1d(s.poly, cold->poly, pbytes, &s.mbar);
        }
        mbar_wait(&s.mbar, 1);
    }
    return StagedD{GeomD{s.hot.box, h.n_box, p.setting == 3 ? cold->density : nullptr},
                   EdgePool{s.hot.e_lower, s.hot.e_next, s.hot.e_off, s.hot.first_in, s.hot.last_in, cold->e_st, s.st, h.n_edge,
                            s.hot.poly_off, &cold->poly[0][0], s.poly, h.n_poly}};
}

// get_possible_position's cut (D:bin3D.py:100-136, C:bin3D.py): the first `nl` feasible of candidates 0 .. n_cand-1, in candidate order.
// One thread per candidate in chunks of the block (WARPS warps, every thread calls it); test(c, row) returns whether candidate c is
// feasible and fills its leaf row, which goes to leaf[k] when it is the k-th feasible one.  wb: WARPS words of shared memory.  Returns
// the number of leaves.
template <int WARPS, typename T, typename Test>
__device__ __forceinline__ int first_feasible(int n_cand, int nl, T (*leaf)[6], uint32_t *wb, Test test) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    int n_leaf = 0;
#pragma unroll 1
    for (int base = 0; base < n_cand && n_leaf < nl; base += 32 * WARPS) {
        const int c = base + tid;
        T row[6] = {0, 0, 0, 0, 0, 0};
        const bool feas = c < n_cand && test(c, row);
        const uint32_t fm = __ballot_sync(FULL, feas);
        if (lane == 0) wb[warp] = fm;
        __syncthreads();
        int before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < WARPS; w++) {
            const int cnt = __popc(wb[w]);
            if (w < warp) before += cnt;
            total += cnt;
        }
        if (feas) {
            const int k = n_leaf + before + __popc(fm & ((1u << lane) - 1));
            if (k < nl)
                for (int t = 0; t < 6; t++) leaf[k][t] = row[t];
        }
        n_leaf += total;
        __syncthreads();
    }
    return n_leaf > nl ? nl : n_leaf;
}

}  // namespace pct
