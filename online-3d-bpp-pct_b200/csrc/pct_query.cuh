// Batched placement queries and height maps of the discrete env (pct_query_placements / pct_height_maps, include/pct_b200.h).
//
// Queries: a block of FEAS_THREADS owns one row (n_rows x k placements of one env).  It stages the env exactly like
// pct_heuristic_kernel (TMA bulk copy of DEnvHot, then the first load edges and polygon vertices when the setting has a
// stability test) and gives each placement of the current FEAS_THREADS-chunk its own thread, which answers it with
// query_placement_d — the code of the single query, so every answer is that of pct_query_placement.  Nothing is written
// back to the env: capacity flags raised by stability_check stay in the thread, as in the single query.  Envs within one
// launch are distinct (caller's contract), because stability_check uses the env's `big` scratch under the block's lock.
//
// Height maps: a block per env stages the placed boxes and gives each cell its own thread, with the Space.plain expression
// of pct_heuristic_kernel; the map goes straight to global memory, so the container has no side limit here.
//
// Included at the end of pct_discrete.cu (same translation unit: it reuses GeomD / rest_height / the staging layout).
#pragma once

namespace pct {

constexpr int HMAP_THREADS = 128;

template <bool STAB>
__global__ void __launch_bounds__(FEAS_THREADS, 4) pct_query_kernel(const DParams p, const QParams q) {
    __shared__ __align__(16) unsigned char sm[K3_SMEM];
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
    DEnvHot *hot = (DEnvHot *)sm;
    uint64_t *mbar = (uint64_t *)(sm + sizeof(DEnvHot) + NL_MAX * 12);
    int *lock = (int *)(mbar + 1);
    Stack4 *st_sm = (Stack4 *)(sm + sizeof(DEnvHot) + NL_MAX * 12 + 64);
    double *poly_sm = (double *)(st_sm + EDGE_STAGE);
    DEnvHot *ghot = p.hot + e;
    DEnvCold *cold = p.cold + e;
    if (tid == 0) {
        *lock = 0;
        mbar_init(mbar, 1);
        fence_proxy_async();
    }
    __syncthreads();
    if (tid == 0) {
        mbar_expect_tx(mbar, (uint32_t)sizeof(DEnvHot));
        tma_load_1d(hot, ghot, (uint32_t)sizeof(DEnvHot), mbar);
    }
    mbar_wait(mbar, 0);
    __syncthreads();
    const DHdr &h = hot->h;
    if (STAB && h.n_edge > 0) {
        const uint32_t bytes = (uint32_t)min(h.n_edge, EDGE_STAGE) * (uint32_t)sizeof(Stack4);
        const uint32_t pbytes = (uint32_t)min(h.n_poly, POLY_STAGE) * 16u;
        if (tid == 0) {
            mbar_expect_tx(mbar, bytes + pbytes);
            tma_load_1d(st_sm, cold->e_st, bytes, mbar);
            if (pbytes) tma_load_1d(poly_sm, cold->poly, pbytes, mbar);
        }
        mbar_wait(mbar, 1);
    }
    const int n_box = h.n_box;
    GeomD g{hot->box, n_box, p.setting == 3 ? cold->density : nullptr};
    EdgePool pool{hot->e_lower, hot->e_next, hot->e_off, hot->first_in, hot->last_in, cold->e_st, st_sm, h.n_edge,
                  hot->poly_off, &cold->poly[0][0], poly_sm, h.n_poly};
    int fl = 0;  // not ORed into the env: a query leaves the env as it was
    const int32_t *qv = (const int32_t *)q.q;
#pragma unroll 1
    for (int base = 0; base < K; base += FEAS_THREADS) {
        const int j = base + tid;
        if (j >= K) break;
        const int32_t *x = qv + (row + j) * 5;
        const double den = q.density ? q.density[row + j] : h.next_den;
        int mh;
        const int feas = query_placement_d<STAB>(hot, n_box, g, pool, &cold->big, lock, p.W, p.L, p.H, x[0], x[1], x[2], x[3], x[4], den, mh, fl);
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
