// Heuristic baselines on the CONTINUOUS env: LSAH, OnlineBPH and BR — the three heuristic.py allows there
// (tools.py:217-218; heuristic.py LASH :138-226, OnlineBPH :364-424, BR :500-577 over pct_envs.PctContinuous0).
//
// Same scheme as pct_heuristics.cuh: a block of 64 threads owns one env, every thread evaluates one (EMS, orientation)
// placement of the current 64-chunk with the placement test of the leaf expansion (place_virtual_c, pct_block.cuh: bounds with
// the 1e-6 tolerances, interSect2D rest height, virtual stability), and thread 0 folds the chunk in enumeration order so that
// ties resolve as in the sequential reference.  All scores are float64 and written with the reference's operand order
// (the translation unit is compiled with -fmad=false), so `score < bestScore` / `score == bestScore` decide identically.
// Output: a float64 ACTION ROW per env, [lx, ly, 0, lx+x, ly+y, 0, 0, 0, 1], which LeafNode2Action (C:bin3D.py:151-167)
// decodes back into the chosen orientation (item sizes carry <= 6 decimals, so round(xe - xs, 6) returns x itself).
// "No feasible placement" (the baselines then end the episode without stepping): the continuous LeafNode2Action never
// raises, so the row is [W+1, 0, 0, W+1, 0, 0, 0, 0, 1] — Space.drop_box rejects it on its bounds test (C:space.py:336)
// and pct_step ends the episode with the same counter / ratio.
//
// Included at the end of pct_continuous.cu (same translation unit: it reuses GeomC / CEnv).
#pragma once
#include "pct_heur_select_c.cuh"

namespace pct {

// 8 / 12 blocks per SM: 128 / 80 registers.  Without the bound the instantiation without a stability test takes 86 registers (11 blocks
// per SM) and its selection is about 10 % slower on the H100 (scratch/heur_bench_cont.py, setting 2: LSAH 0.127 -> 0.140 ms at 4096 envs)
template <bool STAB>
__global__ void __launch_bounds__(64, STAB ? 8 : 12) pctc_heuristic_kernel(const CParams p, const HParamsC hp) {
    const int e = blockIdx.x;
    const HeurPickC r = heur_select_c<STAB>(p, hp, e, nullptr, nullptr);
    if (threadIdx.x == 0) {
        heur_row_c(hp.rows + (size_t)e * 9, r.found, p.W, r.best.lx, r.best.ly, r.best.sx, r.best.sy);
        if (r.found && hp.code == PCT_H_LSAH)
            lsah_note_c(hp.hstate + (size_t)e * 4, r.maxX, r.maxY, r.minX, r.minY, r.best.lx, r.best.ly, r.best.sx, r.best.sy);
    }
}

// Batched placement queries (pct_query_placements_f64): a block of 64 threads owns one row (k placements of one env, read in
// place like pctc_heuristic_kernel does), one thread per placement of the current 64-chunk, answered by place_virtual_c
// (pct_block.cuh); pct_query_placement_f64 asks one row of one placement here.  Nothing is written back to the env.  Envs
// within one launch are distinct (caller's contract): stability_check uses the env's `big` scratch under the block's lock.
template <bool STAB>
__global__ void __launch_bounds__(64) pctc_query_kernel(const CParams p, const QParams q) {
    __shared__ int lock;
    const int tid = threadIdx.x, r = blockIdx.x, K = q.k;
    const int e = q.env ? q.env[r] : r;
    const size_t row = (size_t)r * K;
    double *rest = (double *)q.rest;
    if (e < 0 || e >= p.n_envs) {  // not an env of this handle: infeasible, rest height 0
        for (int j = tid; j < K; j += 64) {
            if (q.feasible) q.feasible[row + j] = 0;
            if (rest) rest[row + j] = 0.0;
        }
        return;
    }
    CEnv *ev = p.env + e;
    const CHdr &h = ev->h;
    if (tid == 0) lock = 0;
    __syncthreads();
    const int n_box = h.n_box;
    GeomC g{ev->box, ev->den, n_box};
    EdgePool pool{ev->e_lower, ev->e_next, ev->e_off, ev->first_in, ev->last_in, ev->e_st, ev->e_st, h.n_edge,
                  ev->poly_off, &ev->poly[0][0], &ev->poly[0][0], h.n_poly};
    int fl = 0;  // not ORed into the env: a query leaves the env as it was
    const double *qv = (const double *)q.q;
#pragma unroll 1
    for (int base = 0; base < K; base += 64) {
        const int j = base + tid;
        if (j >= K) break;
        const double *x = qv + (row + j) * 5;
        const double den = q.density ? q.density[row + j] : h.next_den;
        double mh;
        const int feas = place_virtual_c<STAB>(p, g, pool, &ev->big, &lock, x[0], x[1], x[2], x[3], x[4], den, mh, fl);
        if (q.feasible) q.feasible[row + j] = (uint8_t)feas;
        if (rest) rest[row + j] = mh;
    }
}

cudaError_t launch_heuristic_continuous(const CParams &p, const HParamsC &hp, cudaStream_t st) {
    if (p.setting == 2) pctc_heuristic_kernel<false><<<p.n_envs, 64, 0, st>>>(p, hp);
    else pctc_heuristic_kernel<true><<<p.n_envs, 64, 0, st>>>(p, hp);
    return cudaGetLastError();
}

cudaError_t launch_queries_continuous(const CParams &p, const QParams &q, cudaStream_t st) {
    if (p.setting == 2) pctc_query_kernel<false><<<q.n, 64, 0, st>>>(p, q);
    else pctc_query_kernel<true><<<q.n, 64, 0, st>>>(p, q);
    return cudaGetLastError();
}

}  // namespace pct
