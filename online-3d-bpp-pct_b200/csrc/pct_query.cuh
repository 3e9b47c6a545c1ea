// Batched placement queries and height maps of the discrete env (pct_query_placements / pct_height_maps, include/pct_b200.h).
//
// Queries: a block of FEAS_THREADS owns one row (n_rows x k placements of one env).  It stages the env (stage_env_d,
// pct_block.cuh) and gives each placement of the current FEAS_THREADS-chunk its own thread, which answers it with the
// placement test of every discrete kernel, place_virtual_d.  pct_query_placement asks one row of one placement here.  Nothing
// is written back to the env: capacity flags raised by stability_check stay in the thread.  Envs within one launch are
// distinct (caller's contract), because stability_check uses the env's `big` scratch under the block's lock.
//
// Height maps: a block per env stages the placed boxes and gives each cell its own thread, with the Space.plain expression
// of pct_heuristic_kernel; the map goes straight to global memory, so the container has no side limit here.
//
// Included at the end of pct_discrete.cu (same translation unit: it reuses FEAS_THREADS and rest_height).
#pragma once

namespace pct {

constexpr int HMAP_THREADS = 128;

template <bool STAB>
__global__ void __launch_bounds__(FEAS_THREADS, 4) pct_query_kernel(const DParams p, const QParams q) {
    __shared__ __align__(16) StageD sm;
    const int tid = threadIdx.x, r = blockIdx.x, K = q.k;
    const int e = q.env ? q.env[r] : r;
    const size_t row = (size_t)r * K;
    int32_t *rest = (int32_t *)q.rest;
    if (e < 0 || e >= p.n_envs) {  // not an env of this handle: infeasible, rest height 0
        for (int j = tid; j < K; j += FEAS_THREADS) {
            if (q.feasible) q.feasible[row + j] = 0;
            if (rest) rest[row + j] = 0;
        }
        return;
    }
    StagedD sd = stage_env_d<STAB>(sm, p, e, false);
    const double next_den = sm.hot.h.next_den;
    int fl = 0;  // not ORed into the env: a query leaves the env as it was
    const int32_t *qv = (const int32_t *)q.q;
#pragma unroll 1
    for (int base = 0; base < K; base += FEAS_THREADS) {
        const int j = base + tid;
        if (j >= K) break;
        const int32_t *x = qv + (row + j) * 5;
        const int sx = x[0], sy = x[1], sz = x[2], lx = x[3], ly = x[4];
        const double den = q.density ? q.density[row + j] : next_den;
        int feas = 0, mh = 0;  // a position outside [0, W) x [0, L) or a zero footprint: infeasible, rest height 0
        if (lx >= 0 && ly >= 0 && lx < p.W && ly < p.L && sx > 0 && sy > 0)
            feas = place_virtual_d<STAB>(p, sd.g, sd.pool, &p.cold[e].big, &sm.lock, sx, sy, sz, lx, ly, den, mh, fl);
        if (q.feasible) q.feasible[row + j] = (uint8_t)feas;
        if (rest) rest[row + j] = mh;
    }
}

cudaError_t launch_queries_discrete(const DParams &p, const QParams &q, cudaStream_t st) {
    if (p.setting == 2) pct_query_kernel<false><<<q.n, FEAS_THREADS, 0, st>>>(p, q);
    else pct_query_kernel<true><<<q.n, FEAS_THREADS, 0, st>>>(p, q);
    return cudaGetLastError();
}

__global__ void __launch_bounds__(HMAP_THREADS) pct_height_map_kernel(const DEnvHot *hot, int n_envs, const int32_t *env, int W, int L, int32_t *out) {
    __shared__ __align__(16) int16_t box[NB_MAX][6];
    const int tid = threadIdx.x, r = blockIdx.x, cells = W * L;
    const int e = env ? env[r] : r;
    int32_t *o = out + (size_t)r * cells;
    if (e < 0 || e >= n_envs) {  // not an env of this handle: a zero map
        for (int c = tid; c < cells; c += HMAP_THREADS) o[c] = 0;
        return;
    }
    const DEnvHot *gh = hot + e;
    const int n_box = min(gh->h.n_box, NB_MAX);
    const int nv = (n_box * 12 + 15) / 16;  // the box array starts 16-byte aligned behind the header
    for (int v = tid; v < nv; v += HMAP_THREADS) ((int4 *)box)[v] = ((const int4 *)gh->box)[v];
    __syncthreads();
    for (int c = tid; c < cells; c += HMAP_THREADS) {  // Space.plain (D:space.py:316-326): per cell the highest top among the boxes covering it
        const int i = c / L, j = c - i * L;
        o[c] = rest_height(box, 0, n_box, 1, i, j, i + 1, j + 1);
    }
}

cudaError_t launch_height_maps(const DParams &p, const int32_t *env, int n, int32_t *out, cudaStream_t st) {
    pct_height_map_kernel<<<n, HMAP_THREADS, 0, st>>>(p.hot, p.n_envs, env, p.W, p.L, out);
    return cudaGetLastError();
}

}  // namespace pct
