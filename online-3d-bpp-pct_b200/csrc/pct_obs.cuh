// Observation rows of the discrete domain (include/pct_b200.h layout): written by the step kernels (pct_discrete.cu) and by the restore
// kernel (pct_snapshot.cu).
#pragma once
#include "pct_kernels.h"

namespace pct {

// PART: 0 = the whole observation (round 1's block kernel), 1 = internal-node rows + item row (written by the candidates kernel since round 2: they
// are final after the apply kernel, and on the zero-copy host path their PCIe traffic then overlaps the walk kernels), 2 = leaf rows (emit kernel).
template <typename OT, int PART = 0>
__device__ __noinline__ void write_obs(const DParams &p, int e, const DEnvHot *hot, const DEnvCold *cold, const int16_t (*leaf)[6], int n_leaf,
                                       int tid, int nthreads) {
    OT *obs = (OT *)p.obs + (size_t)e * (size_t)((p.nb + p.nl + 1) * 9);
    const int n_box = hot->h.n_box;
    int s0 = hot->h.next_box[0], s1 = hot->h.next_box[1], s2 = hot->h.next_box[2];
    if (s1 < s0) { int t = s0; s0 = s1; s1 = t; }
    if (s2 < s1) { int t = s1; s1 = s2; s2 = t; }
    if (s1 < s0) { int t = s0; s0 = s1; s1 = t; }
    const OT den = (OT)hot->h.next_den;
    const bool s3 = p.setting == 3;
    const int r_lo = PART == 2 ? p.nb : 0, r_hi = PART == 1 ? p.nb : (PART == 2 ? p.nb + p.nl : p.nb + p.nl + 1);
    const int f_lo = r_lo * 9, f_hi = r_hi * 9;
#pragma unroll 4
    for (int f = f_lo + tid; f < f_hi + (PART == 1 ? 9 : 0); f += nthreads) {
        int row = f / 9;
        const int col = f - row * 9;
        if (PART == 1 && row >= p.nb) row = p.nb + p.nl;  // the 9 extra elements of PART 1 are the item row
        OT v = 0;
        if (row < p.nb) {
            if (row < n_box) {
                if (col < 6) v = (OT)hot->box[row][col];
                else if (col == 6) v = s3 ? (OT)cold->density[row] : (OT)1;
                else if (col == 8) v = 1;
            } else if (row == 0 && col == 8) v = 1;  // D:space.py:294-295
        } else if (row < p.nb + p.nl) {
            const int k = row - p.nb;
            if (k < n_leaf) {
                if (col < 5) v = (OT)leaf[k][col];
                else if (col == 5) v = (OT)p.H;  // D:bin3D.py:128 — bin height, not ze
                else if (col == 8) v = 1;
            }
        } else {
            if (col == 0) v = den;
            else if (col == 3) v = (OT)s0;
            else if (col == 4) v = (OT)s1;
            else if (col == 5) v = (OT)s2;
            else if (col == 8) v = 1;
        }
        obs[row * 9 + col] = v;
    }
}

}  // namespace pct
