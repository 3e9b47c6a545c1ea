// Internal: per-env record and launch parameters of the continuous domain, and its observation row writer: shared by the step kernels
// (pct_continuous.cu) and the snapshot / restore kernels (pct_snapshot.cu).
#pragma once
#include "pct_kernels.h"

namespace pct {

constexpr int CE_MAX = 256;     // EMS capacity (reference preallocates 1000, C:space.py:276)
constexpr int CE_TMP = 512;     // intermediate list inside GENEMS
constexpr int CC_TAB = 2048;    // set-emulation table (<= 1228 distinct candidates)

struct CHdr {
    int32_t n_box, n_ems, n_leaf, flags;
    int64_t draw_pos;
    double ep_reward;
    double next_box[3];
    double next_den;
    double vol_sum;
    int32_t ep_len, n_cand, n_edge, n_poly;
};
struct alignas(16) CEnv {
    CHdr h;
    double box[NB_MAX][6];      // lx,ly,lz,x,y,z
    double den[NB_MAX];
    double ems[CE_MAX][6];
    double ems_tmp[CE_TMP][6];
    uint16_t e_off[NB_MAX + 2], poly_off[NB_MAX + 2];
    uint8_t e_lower[EDGE_MAX + 1], e_next[EDGE_MAX + 1], first_in[NB_MAX], last_in[NB_MAX];
    Stack4 e_st[EDGE_MAX + 1];
    double poly[POLY_MAX][2];
    double leaf[NL_MAX][6];
    uint16_t cand[1232];
    BigScratch big;
    uint32_t fbits[FBITS_WORDS];  // feasibility bits of the current observation's candidates (classification at the end of K2, pooled walks, emit kernel)
    int32_t n_fw, lock, n_pending, pad_;  // n_pending: stability walks still running (classification sets, walk kernels decrement, emit kernel polls)
};

// one pooled stability walk of the continuous domain (cf. WalkItem): the candidate's tuple is rebuilt from `code` (cand_tuple)
struct WalkItemC {
    uint32_t env, pack;
    uint16_t c, code;
    int32_t k;
    double mh;
};
static_assert(sizeof(WalkItemC) == 24, "queue entry");

struct CParams {
    CEnv *env;
    int n_envs;
    double W, L, H, low_bound;
    int nb, nl, setting;
    int item_mode, sample_dist;
    double sample_a, sample_b;
    const double *item_set;
    int n_items;
    const double *stream;
    int stream_len, traj_len;
    uint64_t seed;
    int64_t env_id_base;
    const void *actions;
    int action_f64;
    const int32_t *leaf_idx;
    void *obs;
    int obs_f64;
    float *reward;
    uint8_t *done;
    pct_step_info *info;
    int mode, keep_draw, no_auto_reset;
    int32_t *ready;  // overlapped launch mode: per-env hand-over flags [2 * n_envs] (see pct_common.cuh), nullptr = off
    int32_t epoch;
    int shuffle;     // pct_config::shuffle: keyed permutation of the ordered candidate list (shuffle_candidates)
    WalkPools<WalkItemC> walk;  // pooled stability walks (round 2, pct_walks.cuh); walk.walkq nullptr: round 1's block kernel does everything
    int32_t delta;   // delta observation rows (DEnvAux::obs_prev), emit kernel only
    DEnvAux *aux;    // per-env state of the ALIAS apply kernel (EdgePoolA arrays), nullptr with PCT_B200_ALIAS=0 / setting 2
};
static_assert(sizeof(WalkPools<WalkItemC>) == 72 && offsetof(CParams, walk) == 232 && offsetof(CParams, delta) == 304 && sizeof(CParams) == 320,
              "walk pools at the byte offsets of the fields they replaced");

template <typename OT>
__device__ __noinline__ void write_obs_c(const CParams &p, int e, const CEnv *ev, const double (*leaf)[6], int n_leaf, int tid, int nthreads) {
    OT *obs = (OT *)p.obs + (size_t)e * (size_t)((p.nb + p.nl + 1) * 9);
    const int n_box = ev->h.n_box, total = (p.nb + p.nl + 1) * 9;
    double s0 = ev->h.next_box[0], s1 = ev->h.next_box[1], s2 = ev->h.next_box[2];
    if (s1 < s0) { double t = s0; s0 = s1; s1 = t; }
    if (s2 < s1) { double t = s1; s1 = s2; s2 = t; }
    if (s1 < s0) { double t = s0; s0 = s1; s1 = t; }
#pragma unroll 1
    for (int f = tid; f < total; f += nthreads) {
        const int row = f / 9, col = f - row * 9;
        double v = 0;
        if (row < p.nb) {
            if (row < n_box) {  // C:space.py:372-373  [lx,ly,lz,lx+x,ly+y,lz+z,0,0,1]
                const double *b = ev->box[row];
                if (col < 3) v = b[col];
                else if (col < 6) v = b[col - 3] + b[col];
                else if (col == 8) v = 1;
            } else if (row == 0 && col == 8) v = 1;
        } else if (row < p.nb + p.nl) {
            const int k = row - p.nb;
            if (k < n_leaf) {
                if (col < 5) v = leaf[k][col];
                else if (col == 5) v = p.H;
                else if (col == 8) v = 1;
            }
        } else {
            if (col == 0) v = ev->h.next_den;
            else if (col == 3) v = s0;
            else if (col == 4) v = s1;
            else if (col == 5) v = s2;
            else if (col == 8) v = 1;
        }
        obs[f] = (OT)v;
    }
}

}  // namespace pct
