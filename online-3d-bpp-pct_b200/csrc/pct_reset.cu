// Per-env reset of the discrete env (pct_reset_envs, include/pct_b200.h).
//
// pct_reset_envs_kernel stands in for the apply kernel of a step, as pct_set_items_kernel does for the item override (pct_items.cu).
// The selected envs get reset_space, the apply kernel's auto-reset of a finished env; every env's info record is initialised the way
// the apply kernel does for a successful step (counter, sticky flags, zeros).  The rest of the step's pipeline (candidates, walks,
// emit) then re-expands every env of the batch (launch_discrete with apply = false).  The selected form (pct_reset_envs_only) resets, records and
// re-expands the selected envs alone.
//
// A translation unit of its own (see pct_draw.cuh): in pct_items.cu, reset_space's call of draw_item changed the code of the preview
// kernel, the other caller of draw_item there.
#include "pct_common.cuh"
#include "pct_kernels.h"
#include "pct_draw.cuh"

namespace pct {

constexpr int RESET_THREADS = 256;

// warp w owns env w: it looks the env up in the mask or the list, resets it if selected (reset_space is warp-collective), then writes
// its info record from the header it has just written.  One owner per env, so the record never races with a reset, and an index
// outside [0, n_envs) matches no warp.  The list is scanned 32 entries at a time, up to the first match.
// SEL (pct_reset_envs_only): warp w owns slot w of the selection (EnvSel), O(n) instead of O(n_envs x n); unselected envs are not touched.
template <bool SEL = false>
__global__ void __launch_bounds__(RESET_THREADS) pct_reset_envs_kernel(const DParams p, const ResetParams rp) {
    const int w = (blockIdx.x * RESET_THREADS + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    int e = w;
    bool sel;
    if constexpr (SEL) {
        e = sel_env(EnvSel{rp.env, rp.mask, rp.n}, p.n_envs, w);
        if (e < 0) return;  // the whole warp
        sel = true;
    } else {
        if (e >= p.n_envs) return;  // the whole warp
        sel = rp.mask && rp.mask[e] != 0;
        if (!rp.mask)
            for (int i0 = 0; i0 < rp.n && !sel; i0 += 32) sel = __any_sync(FULL, i0 + lane < rp.n && rp.env[i0 + lane] == e);
    }
    DEnvHot *hot = p.hot + e;
    if (sel) reset_space(hot, p, e, lane);
    if (lane == 0 && p.info) {
        pct_step_info info{};
        info.counter = hot->h.n_box;
        info.flags = hot->h.flags;
        p.info[e] = info;
    }
}

cudaError_t launch_reset_kernel_discrete(const DParams &p, const ResetParams &rp, cudaStream_t st, const EnvSel *sel) {
    constexpr int envs_per_block = RESET_THREADS / 32;
    const int slots = sel ? sel->slots(p.n_envs) : p.n_envs;
    if (sel) pct_reset_envs_kernel<true><<<(slots + envs_per_block - 1) / envs_per_block, RESET_THREADS, 0, st>>>(p, rp);
    else pct_reset_envs_kernel<<<(slots + envs_per_block - 1) / envs_per_block, RESET_THREADS, 0, st>>>(p, rp);
    return cudaGetLastError();
}

cudaError_t launch_reset_envs_discrete(const DParams &p, const ResetParams &rp, cudaStream_t st, const EnvSel *sel) {
    const cudaError_t err = launch_reset_kernel_discrete(p, rp, st, sel);
    if (err != cudaSuccess) return err;
    return launch_discrete(p, st, nullptr, false, sel);
}

}  // namespace pct
