// The placement selection of the continuous heuristic baselines for one env and one item (heur_select_c), shared by the plain kernel
// (pct_heuristics_continuous.cuh, pct_continuous.cu) and the buffered one (pct_buffer.cu), and the helpers around it.
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

// The selection of one env's placement for one item (thread 0's values), run by a block of 64 threads: the body of pctc_heuristic_kernel (item
// nullptr: the header's next_box / next_den; lock nullptr: the block's own lock on the env's BigScratch) and of pctc_buf_heuristic_kernel (item:
// the slot's [x, y, z, density]; lock: the env's, which the blocks of the env's other slots share).  ORs the placement tests' flags into the env.
struct HeurPickC {
    bool found;
    HCandC best;
    double score;
    int c;
    double maxX, maxY, minX, minY;
};

template <bool STAB>
__device__ __forceinline__ HeurPickC heur_select_c(const CParams &p, const HParamsC &hp, int e, const double *item, int32_t *glock) {
    __shared__ uint16_t ord[CE_MAX];
    __shared__ int c_feas[64];
    __shared__ double c_score[64];
    __shared__ int lock, stop;
    const int tid = threadIdx.x, lane = tid & 31, code = hp.code;
    CEnv *ev = p.env + e;
    const CHdr &h = ev->h;
    if (tid == 0) { lock = 0; stop = 0; }
    const double nb[3] = {item ? item[0] : h.next_box[0], item ? item[1] : h.next_box[1], item ? item[2] : h.next_box[2]};
    const int n_ems = h.n_ems, n_box = h.n_box, R = p.setting == 2 ? 6 : 2;
    const double den = item ? item[3] : h.next_den;
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
    int best_c = 0;
    double best_score = code == PCT_H_LSAH ? p.W * p.L + p.L * p.H + p.H * p.W : -1e10;  // heuristic.py:163 / :527
#pragma unroll 1
    for (int base = 0; base < n_c; base += 64) {
        const int c = base + tid;
        int feas = 0;
        double mh = 0, score = 0;
        if (c < n_c) {
            const HCandC k = heur_decode_c(code, c, ev->ems, ord, nb, R);
            if (k.valid) feas = place_virtual_c<STAB>(p, g, pool, &ev->big, glock ? glock : &lock, k.sx, k.sy, k.sz, k.lx, k.ly, den, mh, fl);
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
                if (take) { found = true; best = k; best_score = s; best_c = base + j; }
                if (stop) break;
            }
        }
        __syncthreads();
        if (stop) break;
    }
    fl = __reduce_or_sync(FULL, fl);
    if (fl && lane == 0) atomicOr(&ev->h.flags, fl);
    return HeurPickC{found, best, best_score, best_c, maxX, maxY, minX, minY};
}

// the float64 action row of a placement, [lx, ly, 0, lx+x, ly+y, 0, 0, 0, 1]; without one, a row out of the container (see the header comment)
__device__ __forceinline__ void heur_row_c(double *row, bool found, double W, double lx, double ly, double sx, double sy) {
    if (found) {
        row[0] = lx; row[1] = ly; row[2] = 0;
        row[3] = lx + sx; row[4] = ly + sy; row[5] = 0;
    } else {
        row[0] = W + 1.0; row[1] = 0; row[2] = 0; row[3] = W + 1.0; row[4] = 0; row[5] = 0;
    }
    row[6] = 0; row[7] = 0; row[8] = 1;
}

// LSAH footprint after the chosen placement (heuristic.py:217-220)
__device__ __forceinline__ void lsah_note_c(double *s, double maxX, double maxY, double minX, double minY, double lx, double ly, double sx, double sy) {
    s[0] = fmax(maxX, lx + sx); s[1] = fmax(maxY, ly + sy);
    s[2] = fmin(minX, lx); s[3] = fmin(minY, ly);
}

}  // namespace pct
