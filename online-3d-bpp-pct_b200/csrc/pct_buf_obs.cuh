// Rows of the buffered observation ((NB + B * NL + B) rows per env, include/pct_b200.h): written by the buffered expansion (pct_buffer.cu)
// and by the buffered restore (pct_snapshot.cu).  NT: threads of the calling block.
#pragma once
#include "pct_kernels.h"
#include "pct_continuous.cuh"

namespace pct {

// the internal-node rows of write_obs
template <typename OT, int NT>
__device__ __forceinline__ void buf_internal_rows_d(OT *obs, const DEnvHot *hot, const DEnvCold *cold, int nb, int n_box, int setting, int tid) {
#pragma unroll 1
    for (int f = tid; f < nb * 9; f += NT) {
        const int row = f / 9, col = f - row * 9;
        OT v = 0;
        if (row < n_box) {
            if (col < 6) v = (OT)hot->box[row][col];
            else if (col == 6) v = setting == 3 ? (OT)cold->density[row] : (OT)1;
            else if (col == 8) v = 1;
        } else if (row == 0 && col == 8) v = 1;
        obs[f] = v;
    }
}

// the internal-node rows of write_obs_c
template <typename OT, int NT>
__device__ __forceinline__ void buf_internal_rows_c(OT *obs, const CEnv *env, int nb, int n_box, int tid) {
#pragma unroll 1
    for (int f = tid; f < nb * 9; f += NT) {
        const int row = f / 9, col = f - row * 9;
        double v = 0;
        if (row < n_box) {
            const double *bx = env->box[row];
            if (col < 3) v = bx[col];
            else if (col < 6) v = bx[col - 3] + bx[col];
            else if (col == 8) v = 1;
        } else if (row == 0 && col == 8) v = 1;
        obs[f] = (OT)v;
    }
}

// the nl leaf rows of one slot's block at `o` (the leaf rows of cur_observation, write_obs / write_obs_c) from the n_leaf rows of `leaf`, NT
// threads.  A macro, not a function: as an inlined function it changed the code of the continuous expansion kernel around it.
#define BUF_LEAF_ROWS(OT, o, leaf, n_leaf, nl, H, tid, NT)                  \
    _Pragma("unroll 1") for (int f = (tid); f < (nl) * 9; f += (NT)) {      \
        const int k = f / 9, col = f - k * 9;                               \
        OT v = 0;                                                           \
        if (k < (n_leaf)) {                                                 \
            if (col < 5) v = (OT)(leaf)[k][col];                            \
            else if (col == 5) v = (OT)(H);                                 \
            else if (col == 8) v = 1;                                       \
        }                                                                   \
        (o)[f] = v;                                                         \
    }

// the item row of one slot, as pct_set_items writes it (sizes in ascending order); threads tid < 9
template <typename OT>
__device__ __forceinline__ void buf_item_row(OT *row, const double sz[3], double den, int tid) {
    if (tid < 9) {
        double s0 = sz[0], s1 = sz[1], s2 = sz[2];
        if (s1 < s0) { double t = s0; s0 = s1; s1 = t; }
        if (s2 < s1) { double t = s1; s1 = s2; s2 = t; }
        if (s1 < s0) { double t = s0; s0 = s1; s1 = t; }
        const int col = tid;
        OT v = 0;
        if (col == 0) v = (OT)den;
        else if (col == 3) v = (OT)s0;
        else if (col == 4) v = (OT)s1;
        else if (col == 5) v = (OT)s2;
        else if (col == 8) v = 1;
        row[col] = v;
    }
}

}  // namespace pct
