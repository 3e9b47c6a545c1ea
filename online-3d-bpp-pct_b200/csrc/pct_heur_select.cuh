// The placement selection of the discrete heuristic baselines for one env and one item (heur_select), shared by the plain kernel
// (pct_heuristics.cuh, pct_discrete.cu) and the buffered one (pct_buffer.cu), and the helpers around it.  The including translation unit
// defines FEAS_THREADS, the block size of the selection.
#pragma once


namespace pct {

constexpr int HM_CELLS_MAX = 1024;   // height map staged in shared memory (HM, MACS): W * L <= 1024
constexpr int HC_MAX = 6144;         // RANDOM: feasibility bitmap capacity (grid x rotations)

// Large-container instantiation (BIG = true: HM, MACS and RANDOM when W or L > 32).  The height map, the RANDOM bitmap and MACS's
// histogram rows then live in dynamic shared memory sized from W * L: the int16 map (padded to 16 bytes), then either the bitmap
// (one bit per grid candidate, ceil(W * L * R / 32) words) or the histogram rows (byte j of thread t at j * FEAS_THREADS + t); only
// one of the two is used by a launch.  At 255 x 255, R = 6 this is 130064 + 48768 bytes next to the static staging.
__host__ __device__ constexpr size_t heur_big_map_bytes(int W, int L) { return ((size_t)W * L * 2 + 15) / 16 * 16; }
__host__ __device__ constexpr size_t heur_big_smem(int W, int L, int R) {
    const size_t bitmap = ((size_t)W * L * R + 31) / 32 * 4, rows = (size_t)FEAS_THREADS * L;
    return heur_big_map_bytes(W, L) + (bitmap > rows ? bitmap : rows);
}


// `x, y, z = next_box`, `y, x, z = ...`, `z, x, y = ...`, `z, y, x = ...`, `x, z, y = ...`, `y, z, x = ...` (heuristic.py:176-187):
// which entry of next_box becomes x / y / z.  (Not the EMSPoint rotation table.)
__device__ __forceinline__ void heur_rot(const int nb[3], int rot, int &x, int &y, int &z) {
    switch (rot) {
        case 0: x = nb[0]; y = nb[1]; z = nb[2]; break;
        case 1: x = nb[1]; y = nb[0]; z = nb[2]; break;
        case 2: x = nb[1]; y = nb[2]; z = nb[0]; break;
        case 3: x = nb[2]; y = nb[1]; z = nb[0]; break;
        case 4: x = nb[0]; y = nb[2]; z = nb[1]; break;
        default: x = nb[2]; y = nb[0]; z = nb[1]; break;
    }
}

struct HCand { int sx, sy, sz, lx, ly, ex, ey, ez; bool valid; };

// enumeration index -> placement.  EMS family: ems (list order; OnlineBPH: deep-bottom-left order) x rot [x corner];
// grid family: lx x ly x rot with the loop bounds of the UNROTATED item (heuristic.py:253-254).
__device__ __forceinline__ HCand heur_decode(int code, int c, const int16_t (*ems)[6], const uint8_t *ord, const int nb[3], int R, int ny) {
    HCand k;
    k.ex = k.ey = k.ez = 0;
    if (code <= PCT_H_MACS) {
        const int K = code == PCT_H_MACS ? 4 : 1;
        const int i = c / (R * K), rot = (c / K) % R, corner = c % K;
        const int16_t *e = ems[code == PCT_H_ONLINEBPH ? ord[i] : i];
        heur_rot(nb, rot, k.sx, k.sy, k.sz);
        k.ex = e[3] - e[0]; k.ey = e[4] - e[1]; k.ez = e[5] - e[2];
        k.valid = code == PCT_H_ONLINEBPH || (k.ex >= k.sx && k.ey >= k.sy && k.ez >= k.sz);
        k.lx = (corner & 1) ? e[3] - k.sx : e[0];
        k.ly = (corner & 2) ? e[4] - k.sy : e[1];
    } else {
        const int per = ny * R;
        k.lx = c / per;
        k.ly = (c / R) % ny;
        heur_rot(nb, c % R, k.sx, k.sy, k.sz);
        k.valid = true;
    }
    return k;
}

// calc_maximal_usable_spaces (heuristic.py:12-45) of the container after the placement, summed over the levels below
// the rest height.  The reference tracks a voxel grid (boxes and the space under them are non-zero, :47-52); a voxel
// (i, j, k) of it is non-zero exactly when k < height map(i, j), so "free at level k" is `height map after <= k`.
// BIG: the row is this thread's column of the histogram rows in dynamic shared memory (values <= W <= 255 fit a byte).
template <bool BIG>
__device__ __noinline__ long long macs_score(const int16_t *hm, int W, int L, const HCand &k, int mh) {
    long long score = 0;
    const int top = mh + k.sz;
    for (int lev = 0; lev < mh; lev++) {
        uint8_t hist_l[BIG ? 1 : 32];  // histogram row i: free cells from row i towards row W-1
        extern __shared__ __align__(16) unsigned char heur_dyn[];
        uint8_t *const hist_s = heur_dyn + heur_big_map_bytes(W, L) + threadIdx.x;
        auto hist = [&](int j) -> uint8_t & { return BIG ? hist_s[j * FEAS_THREADS] : hist_l[j]; };
        for (int j = 0; j < L; j++) hist(j) = 0;
        int best = 0;
        for (int i = W - 1; i >= 0; i--) {
            for (int j = 0; j < L; j++) {
                const bool in = i >= k.lx && i < k.lx + k.sx && j >= k.ly && j < k.ly + k.sy;
                const bool fr = (in ? top : (int)hm[i * L + j]) <= lev;
                hist(j) = fr ? (uint8_t)(hist(j) + 1) : (uint8_t)0;
            }
            for (int j = 0; j < L; j++) {
                const int v = hist(j);
                if (v == 0 || (j > 0 && v == hist(j - 1))) continue;
                int j2 = j, j1 = j;
                while (j2 != L - 1 && !(hist(j2 + 1) < v)) j2++;
                while (j1 != 0 && !(hist(j1 - 1) < v)) j1--;
                best = max(best, v * (j2 - j1 + 1));
            }
        }
        score += best;
    }
    return score;
}

// What the selection for one item found (thread 0's values): the chosen placement, its score, its enumeration index, and the LSAH footprint the
// scores were taken against
struct HeurPick {
    bool found;
    HCand best;
    long long score;
    int c;
    int maxX, maxY, minX, minY;
};

// The selection of one env's placement for one item, run by a block of FEAS_THREADS threads: the body of pct_heuristic_kernel (item nullptr:
// the header's next_box / next_den; lock nullptr: the block's own lock on the env's BigScratch) and of pct_buf_heuristic_kernel (item: the
// slot's [x, y, z, density]; lock: the env's, which the blocks of the env's other slots share).  ORs the placement tests' flags into the env.
// BIG (see heur_big_smem): launched with the dynamic shared memory of the container, for HM / MACS / RANDOM only.
template <bool STAB, bool BIG>
__device__ __forceinline__ HeurPick heur_select(const DParams &p, const HParams &hp, int e, const double *item, int32_t *lock) {
    __shared__ __align__(16) StageD sm;
    __shared__ int16_t hm_s[BIG ? 1 : HM_CELLS_MAX];
    __shared__ uint8_t ord[E_MAX];
    __shared__ int c_feas[FEAS_THREADS];
    __shared__ long long c_score[FEAS_THREADS];
    __shared__ uint32_t fbits_s[BIG ? 1 : HC_MAX / 32];
    __shared__ int hm_sum, stop;
    extern __shared__ __align__(16) unsigned char heur_dyn[];
    int16_t *const hm = BIG ? (int16_t *)heur_dyn : hm_s;
    uint32_t *const fbits = BIG ? (uint32_t *)(heur_dyn + heur_big_map_bytes(p.W, p.L)) : fbits_s;
    const int tid = threadIdx.x, lane = tid & 31;
    const int code = hp.code;
    const DEnvHot *hot = &sm.hot;
    DEnvHot *ghot = p.hot + e;
    if (tid == 0) {
        hm_sum = 0;
        stop = 0;
    }
    StagedD sd = stage_env_d<STAB>(sm, p, e, false);
    const DHdr &h = hot->h;
    const int W = p.W, L = p.L, n_box = h.n_box, n_ems = h.n_ems;
    const int nb[3] = {item ? (int)item[0] : h.next_box[0], item ? (int)item[1] : h.next_box[1], item ? (int)item[2] : h.next_box[2]};
    const int R = p.setting == 2 ? 6 : 2;
    const double den = item ? item[3] : h.next_den;
    const bool need_map = code == PCT_H_HM || code == PCT_H_MACS;
    if (need_map) {  // Space.plain (D:space.py:316-326): per cell the highest top among the boxes covering it
        int part = 0;
        for (int c = tid; c < W * L; c += FEAS_THREADS) {
            const int i = c / L, j = c - i * L;
            const int v = rest_height(hot->box, 0, n_box, 1, i, j, i + 1, j + 1);
            hm[c] = (int16_t)v;
            part += v;
        }
        atomicAdd(&hm_sum, part);
    }
    if (code == PCT_H_ONLINEBPH) {  // sorted(EMS, key=(z, y, x)) — stable (heuristic.py:383-384)
        for (int i = tid; i < n_ems; i += FEAS_THREADS) {
            const int16_t *a = hot->ems[i];
            int rank = 0;
            for (int j = 0; j < n_ems; j++) {
                const int16_t *b = hot->ems[j];
                const bool less = b[2] != a[2] ? b[2] < a[2] : b[1] != a[1] ? b[1] < a[1] : b[0] != a[0] ? b[0] < a[0] : j < i;
                rank += less;
            }
            ord[rank] = (uint8_t)i;
        }
    }
    __syncthreads();
    int fl = 0;
    int ny = 1, n_c;
    if (code <= PCT_H_MACS) n_c = n_ems * R * (code == PCT_H_MACS ? 4 : 1);
    else {
        const int nx = W - nb[0] + 1;
        ny = L - nb[1] + 1;
        n_c = (nx > 0 && ny > 0) ? nx * ny * R : 0;
        if (ny < 1) ny = 1;
    }
    if (code == PCT_H_RANDOM) {
        if (!BIG && n_c > HC_MAX) n_c = HC_MAX;  // BIG: the bitmap holds every grid candidate
        for (int w = tid; w < (BIG ? (n_c + 31) / 32 : HC_MAX / 32); w += FEAS_THREADS) fbits[w] = 0;
        __syncthreads();
    }
    // LSAH footprint state; a fresh episode (no box placed yet) starts from the empty footprint
    int maxX = 0, maxY = 0, minX = W, minY = L;
    if (code == PCT_H_LSAH && n_box > 0) {
        const int32_t *s = hp.hstate + (size_t)e * 4;
        maxX = s[0]; maxY = s[1]; minX = s[2]; minY = s[3];
    }
    // incumbent (thread 0)
    bool found = false;
    HCand best{};
    int best_c = 0;
    long long best_score = code == PCT_H_LSAH ? (long long)W * L + (long long)L * p.H + (long long)p.H * W
                         : (code == PCT_H_BR || code == PCT_H_MACS) ? -10000000000ll : 10000000000ll;
    int n_feas = 0;
#pragma unroll 1
    for (int base = 0; base < n_c; base += FEAS_THREADS) {
        const int c = base + tid;
        int feas = 0, mh = 0;
        long long score = 0;
        if (c < n_c) {
            const HCand k = heur_decode(code, c, hot->ems, ord, nb, R, ny);
            if (k.valid) feas = place_virtual_d<STAB>(p, sd.g, sd.pool, &p.cold[e].big, lock ? lock : &sm.lock, k.sx, k.sy, k.sz, k.lx, k.ly, den, mh, fl);
            if (feas) {
                const int top = mh + k.sz;
                if (code == PCT_H_LSAH) {  // heuristic.py:196-200
                    const long long ex = max(k.lx + k.sx, maxX) - min(k.lx, minX), ey = max(k.ly + k.sy, maxY) - min(k.ly, minY);
                    score = ex * ey + (long long)top * ey + (long long)top * ex;
                } else if (code == PCT_H_BR) {  // eval_ems (heuristic.py:501-513)
                    int fits = 0;
                    for (int t = 0; t < p.n_items; t++) {
                        const double *it = p.item_set + 3 * t;
                        fits += (double)k.ex >= it[0] && (double)k.ey >= it[1] && (double)k.ez >= it[2];
                    }
                    score = (long long)k.ex * k.ey * k.ez + fits + (fits == p.n_items ? 10 : 0);
                } else if (code == PCT_H_MACS) {
                    score = macs_score<BIG>(hm, W, L, k, mh);
                } else if (code == PCT_H_DBL) {  // heuristic.py:482
                    score = k.lx + k.ly + 100ll * mh;
                } else if (code == PCT_H_HM) {  // heuristic.py:281: 100 * np.sum(height map after the placement)
                    int foot = 0;
                    for (int i = k.lx; i < k.lx + k.sx; i++)
                        for (int j = k.ly; j < k.ly + k.sy; j++) foot += hm[i * L + j];
                    score = k.lx + k.ly + 100ll * (hm_sum - foot + k.sx * k.sy * top);
                }
            }
        }
        c_feas[tid] = feas;
        c_score[tid] = score;
        if (code == PCT_H_RANDOM && feas) atomicOr(&fbits[c >> 5], 1u << (c & 31));
        __syncthreads();
        if (tid == 0 && code != PCT_H_RANDOM) {
            const int lim = min(FEAS_THREADS, n_c - base);
            for (int j = 0; j < lim; j++) {
                if (!c_feas[j]) continue;
                const HCand k = heur_decode(code, base + j, hot->ems, ord, nb, R, ny);
                const long long s = c_score[j];
                bool take = false;
                if (code == PCT_H_ONLINEBPH) { take = true; stop = 1; }
                else if (code == PCT_H_BR || code == PCT_H_MACS) take = s > best_score;
                else if (code == PCT_H_LSAH) {
                    if (s < best_score) take = true;
                    else if (s == best_score && found)  // the incumbent's EMS slack is measured with THIS orientation's dims (:211-212)
                        take = min(min(k.ex - k.sx, k.ey - k.sy), k.ez - k.sz) < min(min(best.ex - k.sx, best.ey - k.sy), best.ez - k.sz);
                } else take = s < best_score;
                if (take) { found = true; best = k; best_score = s; best_c = base + j; }
                if (stop) break;
            }
        }
        __syncthreads();
        if (stop) break;
    }
    fl = __reduce_or_sync(FULL, fl);
    if (fl && lane == 0) atomicOr(&ghot->h.flags, fl);
    if (code == PCT_H_RANDOM) {  // uniform over the feasible placements in enumeration order (heuristic.py:346-349)
        __syncthreads();
        if (tid == 0) {
            for (int w = 0; w < (n_c + 31) / 32; w++) n_feas += __popc(fbits[w]);
            if (n_feas > 0) {
                int kth = (int)(rnd_u64(hp.seed, (uint64_t)(p.env_id_base + e), (uint64_t)hp.t) % (uint64_t)n_feas);
                for (int w = 0; w < (n_c + 31) / 32 && !found; w++) {
                    const int cnt = __popc(fbits[w]);
                    if (kth >= cnt) { kth -= cnt; continue; }
                    uint32_t m = fbits[w];
                    while (kth--) m &= m - 1;
                    best_c = w * 32 + __ffs(m) - 1;
                    best = heur_decode(code, best_c, hot->ems, ord, nb, R, ny);
                    found = true;
                }
            }
        }
    }
    return HeurPick{found, best, best_score, best_c, maxX, maxY, minX, minY};
}

// the action row of a placement: [lx, ly, 0, lx+x, ly+y, 0, 0, 0, 1]; without one, extent 0, which matches no item (LeafNode2Action raises in
// the reference, pct_step ends the episode)
__device__ __forceinline__ void heur_row(float *row, bool found, int lx, int ly, int sx, int sy) {
    if (found) {
        row[0] = (float)lx; row[1] = (float)ly; row[2] = 0.f;
        row[3] = (float)(lx + sx); row[4] = (float)(ly + sy); row[5] = 0.f;
    } else {
        row[0] = 1.f; row[1] = 0.f; row[2] = 0.f; row[3] = 1.f; row[4] = 0.f; row[5] = 0.f;
    }
    row[6] = 0.f; row[7] = 0.f; row[8] = 1.f;
}

// LSAH footprint after the chosen placement (heuristic.py:217-220)
__device__ __forceinline__ void lsah_note(int32_t *s, int maxX, int maxY, int minX, int minY, int lx, int ly, int sx, int sy) {
    s[0] = max(maxX, lx + sx); s[1] = max(maxY, ly + sy);
    s[2] = min(minX, lx); s[3] = min(minY, ly);
}

}  // namespace pct
