// Heuristic baselines (reference: heuristic.py:11-577) as ONE placement-selection kernel over the batched env state.
//
// Every baseline of the reference is the same loop: enumerate placements in a fixed order, ask
// Space.drop_box_virtual for feasibility (+ the rest height / the updated height map), score, keep the best under a strict
// comparison.  Here a block of 64 threads owns one env (staged in shared memory by stage_env_d, pct_block.cuh), every
// thread evaluates one placement of the current 64-chunk with the placement test of the leaf expansion (place_virtual_d), and
// thread 0 folds the chunk's verdicts in enumeration order, so ties resolve exactly as in the sequential reference.
// The result is an ACTION ROW per env ([lx, ly, 0, lx+x, ly+y, 0, 0, 0, 1] — what LeafNode2Action decodes back into the
// chosen orientation), fed to the ordinary pct_step.  "No feasible placement" (the baselines then end the episode without
// stepping) is encoded as a row no item can match, which makes pct_step end the episode with the same counter / ratio.
//
// Included at the end of pct_discrete.cu (same translation unit: it reuses FEAS_THREADS and rest_height).
#pragma once
#include "pct_heur_select.cuh"

namespace pct {

template <bool STAB, bool BIG>
__global__ void __launch_bounds__(FEAS_THREADS, 4) pct_heuristic_kernel(const DParams p, const HParams hp) {
    const int e = blockIdx.x;
    const HeurPick r = heur_select<STAB, BIG>(p, hp, e, nullptr, nullptr);
    if (threadIdx.x == 0) {
        heur_row(hp.rows + (size_t)e * 9, r.found, r.best.lx, r.best.ly, r.best.sx, r.best.sy);
        if (r.found && hp.code == PCT_H_LSAH)
            lsah_note(hp.hstate + (size_t)e * 4, r.maxX, r.maxY, r.minX, r.minY, r.best.lx, r.best.ly, r.best.sx, r.best.sy);
    }
}

bool heur_big(const DParams &p, int code) {
    return (p.W > HEUR_SIDE_MAX || p.L > HEUR_SIDE_MAX) && (code == PCT_H_HM || code == PCT_H_MACS || code == PCT_H_RANDOM);
}

cudaError_t launch_heuristic_discrete(const DParams &p, const HParams &hp, cudaStream_t st) {
    if (heur_big(p, hp.code)) {
        const size_t smem = heur_big_smem(p.W, p.L, p.setting == 2 ? 6 : 2);
        if (p.setting == 2) pct_heuristic_kernel<false, true><<<p.n_envs, FEAS_THREADS, smem, st>>>(p, hp);
        else pct_heuristic_kernel<true, true><<<p.n_envs, FEAS_THREADS, smem, st>>>(p, hp);
    } else if (p.setting == 2) pct_heuristic_kernel<false, false><<<p.n_envs, FEAS_THREADS, 0, st>>>(p, hp);
    else pct_heuristic_kernel<true, false><<<p.n_envs, FEAS_THREADS, 0, st>>>(p, hp);
    return cudaGetLastError();
}

// the dynamic shared memory limit of the large-container instantiations, raised to what the largest container needs (pct_create of a
// discrete handle with W or L > 32; idempotent), so that launch_heuristic_discrete only enqueues
cudaError_t prepare_heuristic_big() {
    const int smem = (int)heur_big_smem(255, 255, 6);
    cudaError_t e = cudaFuncSetAttribute(pct_heuristic_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(pct_heuristic_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    return e;
}

}  // namespace pct
