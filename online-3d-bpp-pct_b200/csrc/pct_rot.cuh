// Rotation table and canonical candidate keys of the discrete candidate list: shared by the step kernels (pct_discrete.cu, included at the
// place the definitions stood, so their code is unchanged) and the leaf expansion of caller-given items (pct_expand.cu).
#pragma once
#include "pct_common.cuh"
#include "pct_kernels.h"

namespace pct {

struct RotTab {   // per env/item: oriented dims of the R rotations (D:space.py:540-562), validity, canonical index
    uint8_t d[6][3];
    uint8_t valid, canon[6];
};

__device__ __forceinline__ void make_rot_tab(const int nb[3], int R, RotTab &rt) {
    const int perm[6][3] = {{0, 1, 2}, {1, 0, 2}, {0, 2, 1}, {1, 2, 0}, {2, 0, 1}, {2, 1, 0}};
    rt.valid = 0;
#pragma unroll
    for (int r = 0; r < 6; r++) {
        const int sx = nb[perm[r][0]], sy = nb[perm[r][1]], sz = nb[perm[r][2]];
        rt.d[r][0] = (uint8_t)sx; rt.d[r][1] = (uint8_t)sy; rt.d[r][2] = (uint8_t)sz;
        bool v = r < R;
        if (r == 1 || r == 4 || r == 5) v = v && sx != sy;
        if (r == 2 || r == 3) v = v && !(sx == sy && sy == sz);
        if (v) rt.valid |= 1 << r;
        int c = r;
        for (int q = r - 1; q >= 0; q--)
            if (rt.d[q][0] == sx && rt.d[q][1] == sy && rt.d[q][2] == sz) c = q;
        rt.canon[r] = (uint8_t)c;
    }
}

template <int BITS>
__device__ __forceinline__ uint32_t key_pack(int xs, int ys, int zs, int rot) {
    return (uint32_t)xs | ((uint32_t)ys << BITS) | ((uint32_t)zs << (2 * BITS)) | ((uint32_t)rot << (3 * BITS));
}
template <int BITS>
__device__ __forceinline__ void key_unpack(uint32_t k, int &xs, int &ys, int &zs, int &rot) {
    constexpr uint32_t M = (1u << BITS) - 1;
    xs = k & M; ys = (k >> BITS) & M; zs = (k >> (2 * BITS)) & M; rot = (k >> (3 * BITS)) & 7;
}
template <int BITS>
__device__ __noinline__ uint64_t key_hash(uint32_t k, const RotTab *rt) {
    int xs, ys, zs, rot;
    key_unpack<BITS>(k, xs, ys, zs, rot);
    const uint64_t l[6] = {(uint64_t)xs, (uint64_t)ys, (uint64_t)zs, (uint64_t)(xs + rt->d[rot][0]), (uint64_t)(ys + rt->d[rot][1]),
                           (uint64_t)(zs + rt->d[rot][2])};
    return tuple_hash6(l);
}

}  // namespace pct
