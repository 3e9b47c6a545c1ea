// Internal: the object behind pct_handle.
#pragma once
#include <string>
#include <vector>
#include "pct_kernels.h"

struct pct_env_batch {
    pct_config cfg;
    int n_envs = 0, device = 0;
    int obs_len = 0;
    bool did_reset = false;
    int64_t launches = 0;
    std::string err;
    // device state
    pct::DEnvHot *d_hot = nullptr;
    pct::DEnvCold *d_cold = nullptr;
    void *c_state = nullptr;  // continuous-domain state (pct_continuous.cu)
    double *d_item_set = nullptr;
    int n_items = 0;
    double *d_stream = nullptr;
    int stream_len = 0;
    int traj_len = 0;
    int32_t *d_ready = nullptr;   // [2 * n_envs] per-env hand-over flags of the overlapped launch mode
    int32_t epoch = 0;
    bool overlap = true;          // PCT_B200_OVERLAP=0: plain back-to-back kernels
    bool overlap_cont = false;    // continuous domain: measured slower overlapped, off unless PCT_B200_OVERLAP_CONT=1
    // delta observation writes (default ON since round 2: faster on the device path, and much faster through pct_step_host with zero-copy;
    // PCT_B200_OBS_DELTA=0 disables): the feasibility kernel writes only the rows that can differ from what the SAME caller buffer already holds
    // (DEnvAux::obs_prev = per env the internal / leaf rows of the tracked buffer that may be non-zero).  Contract (include/pct_b200.h): a caller
    // that hands the same observation pointer to consecutive calls must not have modified the buffer in between.
    bool obs_delta = true;
    // object semantics of the load entries in the real placement = what the reference's Python objects do (DESIGN.md section 3 (b)):
    // pct_apply_kernel<STAB, ALIAS = true> / pctc_apply_kernel<true, true>.  Default ON since round 2 (green on hardware, oracle default flipped with it);
    // PCT_B200_ALIAS=0 selects the snapshot semantics of round 1 (kept for the sensitivity tests).
    bool alias_mode = true;
    bool no_emit_pdl = false;     // PCT_B200_EMIT_PDL=0: launch the emit kernel in plain stream order (A/B measurement of the emit / walk-tail overlap)
    bool k3_block = false;        // PCT_B200_K3=block: round 1's block-per-env feasibility kernel instead of the warp-per-env one (A/B measurements)
    pct::DEnvAux *d_aux = nullptr;  // per-env state of the opt-in variants (allocated when one of them is on)
    const void *tracked_obs = nullptr;
    bool fill_pending = false;
    bool host_zero_copy = true;   // pct_step_host: kernels write the observation straight into the pinned (mapped) host buffer; PCT_B200_HOST_ZEROCOPY=0: staged copies
    bool cont_pre = true;         // continuous feas_emit: resting heights from pre-rounded rectangles (exact; PCT_B200_CONT_PRE=0 disables)
    int32_t *d_hstate = nullptr;  // (n_envs, 4) LSAH footprint state (pct_heuristic_actions; discrete handles)
    double *d_hstate_c = nullptr; // same for the continuous domain (pct_heuristic_actions_f64)
    uint64_t snap_fp = 0;         // fingerprint written into / required of snapshot records (pct_snapshot.cu)
    double *d_query_c = nullptr;  // 2 doubles: result of pct_query_placement_f64
    int32_t *d_query = nullptr;   // 2 + W*L ints: result of pct_query_placement
    int item_mode = 0;
    // staging for the host-buffer entry points
    void *d_obs = nullptr, *d_act = nullptr;
    int32_t *d_idx = nullptr;
    float *d_rew = nullptr;
    uint8_t *d_done = nullptr;
    pct_step_info *d_info = nullptr;
    cudaStream_t own_stream = nullptr;
    void *dbg = nullptr;
    int32_t *d_order = nullptr;   // heaviest-first scheduling order: parity, bucket counts, per-bucket env lists (pct_discrete.cu order_lookup)
    // pooled stability walks (pct_walks.cuh), both domains: create_walk_pools / walk_pools
    void *d_walkq = nullptr;           // [n_envs * CAND_MAX] pool of stability walks of the current step (WalkItem / WalkItemC)
    int32_t *d_walk_ctr = nullptr;     // [n_envs] fill counters (index = first env of the launched range)
    pct::WalkCont *d_contq = nullptr;  // [n_envs * WALK_CONT_PER_ENV] continuations: light-prefix kernel -> continuation kernel
    int32_t *d_cont_ctr = nullptr;     // [8 * (n_envs + 1)] eight counters per (possible) env range
    size_t contq_env_bytes = 0;        // bytes of d_contq per env (WalkCont pool / WalkPiece queue)
    int32_t *d_piece_ready = nullptr, *d_walk_pend = nullptr;  // fork-join walks: per-slot publication flags, per-walk piece counters
    bool walk_fork = false;            // PCT_B200_WALK=fork: fork-join continuation kernel (pct_walkq.cuh) instead of the sequential one — measured equal-to-slower (DESIGN.md section 5), kept as an opt-in
    int walk_blocks = 6;               // its blocks per SM (PCT_B200_WALK_BLOCKS)
    int walk_keep = 264;               // its warps that stay as helpers for forked pieces: two per SM of the H100 (PCT_B200_WALK_KEEP)
    int walk_lanes_tall = 4;           // ... of the tall walks (resting height >= 0.6 H: the longest chains), PCT_B200_WALK_LANES_TALL
    int walk_lanes = 16;               // continuations per warp of pct_walk_kernel (PCT_B200_WALK_LANES; few long serial chains: more warps beat fuller warps)
    bool lpt = false;
    int prof_on = 0;
    std::vector<cudaEvent_t> prof_ev;   // 4 events per recorded step
    int prof_steps = 0;
    int host_groups = 4;          // env ranges pipelined by pct_step_host (kernels of one range overlap the D2H of another)
    int groups = 1;               // env ranges stepped concurrently on internal streams
    cudaStream_t sub[8] = {};
    cudaEvent_t ev_fork = nullptr, ev_join[8] = {};
};

namespace pct {
// allocates the pools of the stability walks with queue entries of `item_bytes` (pct_create, continuous_create; not with PCT_B200_K3=block)
cudaError_t create_walk_pools(pct_env_batch *h, size_t item_bytes);

// the pools of the env range [off, off + cnt): env ranges stepped concurrently (pct_step_host's staged path) own disjoint slices
template <typename Item>
WalkPools<Item> walk_pools(const pct_env_batch *h, int off, int cnt) {
    WalkPools<Item> w{};
    w.walkq = h->d_walkq ? (Item *)h->d_walkq + (size_t)off * CAND_MAX : nullptr;
    w.walk_ctr = h->d_walk_ctr ? h->d_walk_ctr + off : nullptr;
    w.contq = h->d_contq ? (WalkCont *)((char *)h->d_contq + (size_t)off * h->contq_env_bytes) : nullptr;
    w.cont_ctr = h->d_cont_ctr ? h->d_cont_ctr + 8 * (size_t)off : nullptr;
    w.walk_lanes = h->walk_lanes; w.walk_lanes_tall = h->walk_lanes_tall;
    w.walk_fork = h->walk_fork ? 1 : 0; w.walk_blocks = h->walk_blocks; w.walk_keep = h->walk_keep; w.piece_cap = cnt * WALK_PIECES_PER_ENV;
    w.piece_ready = h->d_piece_ready ? h->d_piece_ready + (size_t)off * WALK_PIECES_PER_ENV : nullptr;
    w.walk_pend = h->d_walk_pend ? h->d_walk_pend + (size_t)off * CAND_MAX : nullptr;
    return w;
}
}  // namespace pct
