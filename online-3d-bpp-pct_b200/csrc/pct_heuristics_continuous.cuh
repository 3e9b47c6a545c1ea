// Heuristic baselines on the CONTINUOUS env: LSAH, OnlineBPH and BR — the three heuristic.py allows there
// (tools.py:217-218; heuristic.py LASH :138-226, OnlineBPH :364-424, BR :500-577 over pct_envs.PctContinuous0).
//
// Same scheme as pct_heuristics.cuh: a block of 64 threads owns one env, every thread evaluates one (EMS, orientation)
// placement of the current 64-chunk with the feasibility code of the leaf expansion (pctc_feas_emit_kernel: bounds with the
// 1e-6 tolerances, interSect2D rest height, virtual stability), and thread 0 folds the chunk in enumeration order so that
// ties resolve as in the sequential reference.  All scores are float64 and written with the reference's operand order
// (the translation unit is compiled with -fmad=false), so `score < bestScore` / `score == bestScore` decide identically.
// Output: a float64 ACTION ROW per env, [lx, ly, 0, lx+x, ly+y, 0, 0, 0, 1], which LeafNode2Action (C:bin3D.py:151-167)
// decodes back into the chosen orientation (item sizes carry <= 6 decimals, so round(xe - xs, 6) returns x itself).
// "No feasible placement" (the baselines then end the episode without stepping): the continuous LeafNode2Action never
// raises, so the row is [W+1, 0, 0, W+1, 0, 0, 0, 0, 1] — Space.drop_box rejects it on its bounds test (C:space.py:336)
// and pct_step ends the episode with the same counter / ratio.
//
// Included at the end of pct_continuous.cu (same translation unit: it reuses GeomC / rest_height_c / CEnv).
#pragma once

namespace pct {

// `x, y, z = next_box`, `y, x, z = ...`, `z, x, y = ...`, `z, y, x = ...`, `x, z, y = ...`, `y, z, x = ...` (heuristic.py:176-187)
__device__ __forceinline__ void heur_rot_c(const double nb[3], int rot, double &x, double &y, double &z) {
    switch (rot) {
        case 0: x = nb[0]; y = nb[1]; z = nb[2]; break;
        case 1: x = nb[1]; y = nb[0]; z = nb[2]; break;
        case 2: x = nb[1]; y = nb[2]; z = nb[0]; break;
        case 3: x = nb[2]; y = nb[1]; z = nb[0]; break;
        case 4: x = nb[0]; y = nb[2]; z = nb[1]; break;
        default: x = nb[2]; y = nb[0]; z = nb[1]; break;
    }
}

struct HCandC { double sx, sy, sz, lx, ly, ex, ey, ez; bool valid; };

// Space.drop_box_virtual(dims, (lx, ly), False, density, setting, returnH=True) + check_box (C:space.py:380-439) of ONE placement:
// for the batched queries (pctc_query_kernel).  It is the PCT_H_QUERY_ branch below, expression for expression; that branch keeps
// its own inline copy because routing it through this function changes the register allocation of pctc_heuristic_kernel, and
// tests/test_gpu_queries.py pins the two paths to each other.  mh is interSect2D's max_h (C:space.py:391), reported whatever the
// verdict.  Raised capacity flags go to `fl` (the callers do not OR them into the env).
template <bool STAB>
__device__ __forceinline__ int query_placement_c(const CParams &p, const double (*box)[6], int n_box, const GeomC &g, EdgePool &pool, BigScratch *big,
                                                 int *lock, double sx, double sy, double sz, double lx, double ly, double den, double &mh, int &fl) {
    bool chk = !(lx + sx - 1e-6 > p.W || ly + sy - 1e-6 > p.L) && !(lx + 1e-6 < 0 || ly + 1e-6 < 0);
    mh = rest_height_c(box, 0, n_box, 1, lx, ly, lx + sx, ly + sy);
    if (mh < 0) mh = 0.0;
    if (mh + sz - 1e-6 > p.H) chk = false;
    int feas;
    if (!chk) feas = 0;
    else if (!STAB || fabs(mh) < 1e-6) feas = 1;
    else {
        NodeC root{lx, ly, mh, sx, sy, sz, sx * sy * sz * den};
        feas = stability_check<false, GeomC>(g, root, pool, big, lock, 0, fl) != 0;
    }
    return feas;
}

// enumeration index -> placement: EMS (list order; OnlineBPH: deep-bottom-left order) x orientation, at the EMS origin
__device__ __forceinline__ HCandC heur_decode_c(int code, int c, const double (*ems)[6], const uint16_t *ord, const double nb[3], int R) {
    HCandC k;
    const int i = c / R, rot = c - i * R;
    const double *e = ems[code == PCT_H_ONLINEBPH ? ord[i] : i];
    heur_rot_c(nb, rot, k.sx, k.sy, k.sz);
    k.ex = e[3] - e[0]; k.ey = e[4] - e[1]; k.ez = e[5] - e[2];
    k.valid = code == PCT_H_ONLINEBPH || (k.ex >= k.sx && k.ey >= k.sy && k.ez >= k.sz);  // heuristic.py:189 / :540 (no tolerance)
    k.lx = e[0]; k.ly = e[1];
    return k;
}

template <bool STAB>
__global__ void __launch_bounds__(64) pctc_heuristic_kernel(const CParams p, const HParamsC hp) {
    __shared__ uint16_t ord[CE_MAX];
    __shared__ int c_feas[64];
    __shared__ double c_score[64];
    __shared__ int lock, stop;
    const int tid = threadIdx.x, lane = tid & 31, code = hp.code;
    const int e = code == PCT_H_QUERY_ ? hp.q_env : blockIdx.x;
    CEnv *ev = p.env + e;
    const CHdr &h = ev->h;
    if (tid == 0) { lock = 0; stop = 0; }
    const double nb[3] = {h.next_box[0], h.next_box[1], h.next_box[2]};
    const int n_ems = h.n_ems, n_box = h.n_box, R = p.setting == 2 ? 6 : 2;
    const double den = code == PCT_H_QUERY_ ? hp.q_den : h.next_den;
    if (code == PCT_H_ONLINEBPH) {  // sorted(EMS, key=(z, y, x)) — stable (heuristic.py:383-384); all-zero rows are skipped (:395-396)
        for (int i = tid; i < n_ems; i += 64) {
            const double *a = ev->ems[i];
            int rank = 0;
            for (int j = 0; j < n_ems; j++) {
                const double *b = ev->ems[j];
                const bool less = b[2] != a[2] ? b[2] < a[2] : b[1] != a[1] ? b[1] < a[1] : b[0] != a[0] ? b[0] < a[0] : j < i;
                rank += less;
            }
            ord[rank] = (uint16_t)i;
        }
    }
    __syncthreads();
    GeomC g{ev->box, ev->den, n_box};
    EdgePool pool{ev->e_lower, ev->e_next, ev->e_off, ev->first_in, ev->last_in, ev->e_st, ev->e_st, h.n_edge,
                  ev->poly_off, &ev->poly[0][0], &ev->poly[0][0], h.n_poly};
    int fl = 0;
    if (code == PCT_H_QUERY_) {  // one Space.drop_box_virtual(..., returnH=True) call (C:space.py:380-425) for the single-env facade
        if (tid == 0) {
            const double sx = hp.q[0], sy = hp.q[1], sz = hp.q[2], lx = hp.q[3], ly = hp.q[4];
            bool chk = !(lx + sx - 1e-6 > p.W || ly + sy - 1e-6 > p.L) && !(lx + 1e-6 < 0 || ly + 1e-6 < 0);
            double mh = rest_height_c(ev->box, 0, n_box, 1, lx, ly, lx + sx, ly + sy);
            if (mh < 0) mh = 0.0;
            if (mh + sz - 1e-6 > p.H) chk = false;
            int feas;
            if (!chk) feas = 0;
            else if (!STAB || fabs(mh) < 1e-6) feas = 1;
            else {
                NodeC root{lx, ly, mh, sx, sy, sz, sx * sy * sz * den};
                feas = stability_check<false, GeomC>(g, root, pool, &ev->big, &lock, 0, fl) != 0;
            }
            hp.q_out[0] = (double)feas;
            hp.q_out[1] = mh;
        }
        return;
    }
    const int n_c = n_ems * R;
    // LSAH footprint state (heuristic.py:146-147, 217-220); a fresh episode (no box placed yet) starts from the empty footprint
    double maxX = 0, maxY = 0, minX = p.W, minY = p.L;
    if (code == PCT_H_LSAH && n_box > 0) {
        const double *s = hp.hstate + (size_t)e * 4;
        maxX = s[0]; maxY = s[1]; minX = s[2]; minY = s[3];
    }
    // incumbent (thread 0)
    bool found = false;
    HCandC best{};
    double best_score = code == PCT_H_LSAH ? p.W * p.L + p.L * p.H + p.H * p.W : -1e10;  // heuristic.py:163 / :527
#pragma unroll 1
    for (int base = 0; base < n_c; base += 64) {
        const int c = base + tid;
        int feas = 0;
        double mh = 0, score = 0;
        if (c < n_c) {
            const HCandC k = heur_decode_c(code, c, ev->ems, ord, nb, R);
            if (k.valid) {
                // Space.drop_box_virtual + check_box (C:space.py:380-439), as in pctc_feas_emit_kernel
                bool chk = !(k.lx + k.sx - 1e-6 > p.W || k.ly + k.sy - 1e-6 > p.L) && !(k.lx + 1e-6 < 0 || k.ly + 1e-6 < 0);
                mh = rest_height_c(ev->box, 0, n_box, 1, k.lx, k.ly, k.lx + k.sx, k.ly + k.sy);
                if (mh < 0) mh = 0.0;
                if (mh + k.sz - 1e-6 > p.H) chk = false;
                if (!chk) feas = 0;
                else if (!STAB || fabs(mh) < 1e-6) feas = 1;
                else {
                    NodeC root{k.lx, k.ly, mh, k.sx, k.sy, k.sz, k.sx * k.sy * k.sz * den};
                    feas = stability_check<false, GeomC>(g, root, pool, &ev->big, &lock, 0, fl) != 0;
                }
            }
            if (feas) {
                if (code == PCT_H_LSAH) {  // heuristic.py:196-200
                    const double ex = fmax(k.lx + k.sx, maxX) - fmin(k.lx, minX), ey = fmax(k.ly + k.sy, maxY) - fmin(k.ly, minY);
                    const double top = mh + k.sz;
                    score = ex * ey + top * ey + top * ex;
                } else if (code == PCT_H_BR) {  // eval_ems (heuristic.py:501-513): s = 0; s += volume; s += len(valid); [s += 10]
                    int fits = 0;
                    for (int t = 0; t < p.n_items; t++) {
                        const double *it = p.item_set + 3 * t;
                        fits += k.ex >= it[0] && k.ey >= it[1] && k.ez >= it[2];
                    }
                    score = k.ex * k.ey * k.ez + (double)fits;
                    if (fits == p.n_items) score += 10.0;
                }
            }
        }
        c_feas[tid] = feas;
        c_score[tid] = score;
        __syncthreads();
        if (tid == 0) {
            const int lim = min(64, n_c - base);
            for (int j = 0; j < lim; j++) {
                if (!c_feas[j]) continue;
                const HCandC k = heur_decode_c(code, base + j, ev->ems, ord, nb, R);
                const double s = c_score[j];
                bool take = false;
                if (code == PCT_H_ONLINEBPH) { take = true; stop = 1; }
                else if (code == PCT_H_BR) take = s > best_score;
                else {
                    if (s < best_score) take = true;
                    else if (s == best_score && found)  // the incumbent's EMS slack is measured with THIS orientation's dims (:211-212)
                        take = fmin(fmin(k.ex - k.sx, k.ey - k.sy), k.ez - k.sz) < fmin(fmin(best.ex - k.sx, best.ey - k.sy), best.ez - k.sz);
                }
                if (take) { found = true; best = k; best_score = s; }
                if (stop) break;
            }
        }
        __syncthreads();
        if (stop) break;
    }
    fl = __reduce_or_sync(FULL, fl);
    if (fl && lane == 0) atomicOr(&ev->h.flags, fl);
    if (tid == 0) {
        double *row = hp.rows + (size_t)e * 9;
        if (found) {
            row[0] = best.lx; row[1] = best.ly; row[2] = 0;
            row[3] = best.lx + best.sx; row[4] = best.ly + best.sy; row[5] = 0;
            if (code == PCT_H_LSAH) {  // heuristic.py:217-220
                double *s = hp.hstate + (size_t)e * 4;
                s[0] = fmax(maxX, best.lx + best.sx); s[1] = fmax(maxY, best.ly + best.sy);
                s[2] = fmin(minX, best.lx); s[3] = fmin(minY, best.ly);
            }
        } else {  // out of the container: Space.drop_box returns False, the episode ends (see the header comment)
            row[0] = p.W + 1.0; row[1] = 0; row[2] = 0; row[3] = p.W + 1.0; row[4] = 0; row[5] = 0;
        }
        row[6] = 0; row[7] = 0; row[8] = 1;
    }
}

// Batched placement queries (pct_query_placements_f64): a block of 64 threads owns one row (k placements of one env, read in
// place like pctc_heuristic_kernel does), one thread per placement of the current 64-chunk, answered by query_placement_c.  Nothing
// is written back to the env.  Envs within one launch are distinct (caller's contract): stability_check uses the env's `big`
// scratch under the block's lock.
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
        const int feas = query_placement_c<STAB>(p, ev->box, n_box, g, pool, &ev->big, &lock, x[0], x[1], x[2], x[3], x[4], den, mh, fl);
        if (q.feasible) q.feasible[row + j] = (uint8_t)feas;
        if (rest) rest[row + j] = mh;
    }
}

static CParams state_params_c(pct_env_batch *h) {
    CParams p{};
    p.env = (CEnv *)h->c_state; p.n_envs = h->n_envs;
    p.W = h->cfg.container_size[0]; p.L = h->cfg.container_size[1]; p.H = h->cfg.container_size[2];
    p.low_bound = h->cfg.size_minimum;
    p.nb = h->cfg.internal_node_holder; p.nl = h->cfg.leaf_node_holder; p.setting = h->cfg.setting;
    p.item_set = h->d_item_set; p.n_items = h->n_items;
    return p;
}

int continuous_query(pct_env_batch *h, int env, const double q[5], double density, double *d_out, cudaStream_t st) {
    const CParams p = state_params_c(h);
    HParamsC hp{};
    hp.code = PCT_H_QUERY_; hp.q_env = env; hp.q_den = density; hp.q_out = d_out;
    for (int i = 0; i < 5; i++) hp.q[i] = q[i];
    if (p.setting == 2) pctc_heuristic_kernel<false><<<1, 64, 0, st>>>(p, hp);
    else pctc_heuristic_kernel<true><<<1, 64, 0, st>>>(p, hp);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { h->err = std::string("continuous query launch: ") + cudaGetErrorString(e); return PCT_ERR_CUDA; }
    return PCT_OK;
}

int continuous_queries(pct_env_batch *h, const QParams &q, cudaStream_t st) {
    const CParams p = state_params_c(h);
    if (p.setting == 2) pctc_query_kernel<false><<<q.n, 64, 0, st>>>(p, q);
    else pctc_query_kernel<true><<<q.n, 64, 0, st>>>(p, q);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { h->err = std::string("continuous queries launch: ") + cudaGetErrorString(e); return PCT_ERR_CUDA; }
    return PCT_OK;
}

int continuous_heuristic(pct_env_batch *h, int code, double *rows, double *hstate, cudaStream_t st) {
    const CParams p = state_params_c(h);
    HParamsC hp{};
    hp.code = code; hp.rows = rows; hp.hstate = hstate;
    if (p.setting == 2) pctc_heuristic_kernel<false><<<p.n_envs, 64, 0, st>>>(p, hp);
    else pctc_heuristic_kernel<true><<<p.n_envs, 64, 0, st>>>(p, hp);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { h->err = std::string("continuous heuristic launch: ") + cudaGetErrorString(e); return PCT_ERR_CUDA; }
    return PCT_OK;
}

}  // namespace pct
