// The pooled stability walks (round 2): device bodies of the walk stage, shared by the discrete (pct_walk_*_kernel, pct_discrete.cu) and the
// continuous domain (pctc_walk_*_kernel, pct_continuous.cu).  Each domain's kernels are one-line wrappers that instantiate a body with a traits
// type next to them:
//     Params               DParams / CParams (the pools are its member `walk`, a WalkPools<Item>)
//     Item                 the queue entry: WalkItem / WalkItemC (fields env, pack, c, k used here)
//     Geom                 the geometry policy of the stability routine: GeomD / GeomC
//     view(p, item, has)   the walk's view (DWalkView / CWalkView): geometry g, edge pool, root node, and accessors fbits() / flags() /
//                          n_pending() / big() / lock() that give where its env keeps them (the env stays a base pointer into its record)
//     tall(p, item)        the walk rests high up in the bin (resting height >= 0.6 H): pooled apart, fewer lanes per warp
//
// Protocol of the stage (what both domains rely on):
//   - the classification at the end of the candidates kernel fills walkq (counter walk_ctr) and sets each env's n_pending to its number of walks;
//   - every walk delivers its verdict (a feasibility bit in fbits, flags) and then release-decrements n_pending (walk_done); the emit kernel polls
//     n_pending (wait_walks), so it may start while other envs' walks are still running;
//   - sequential continuations: the light-prefix kernel pools them from the front (ordinary walks, cont_ctr[0]) and from the back (tall walks,
//     cont_ctr[1]) of contq, each class owning half of it (the counters may overshoot; the consumer clamps at cap / 2);
//   - fork-join continuations: contq is a piece queue (pct_walkq.cuh); walk_pend[item] counts a walk's pieces, the verdict is the AND over them;
//   - a walk that finds no room in a pool leaves its candidate infeasible and sets PCT_FLAG_CAND_OVERFLOW of its env: never silent;
//   - pool counters are emptied for the next step by the emit kernel (sequential walks: reset_walk_pools) or by the fork-join kernel's last warp out.
#pragma once
#include "pct_common.cuh"
#include "pct_walkq.cuh"

namespace pct {

constexpr int WALK_WARPS = 2, LIGHT_WARPS = 4;  // warps per block of the continuation kernels / of the light-prefix kernels

// a walk of this env has delivered its verdict (fbits / flags written before): release-decrement the env's counter of running walks
__device__ __forceinline__ void walk_done(int32_t *n_pending) {
    __threadfence();
    atomicSub(n_pending, 1);
}

// walk, stage 1: the light prefix of EVERY pooled walk, one lane per walk (stab_light: single-support visits only — small code, no local arrays).
// 81 % of the walks end here; the rest goes to the continuation pool with (node, stack).  Blocks of LIGHT_WARPS warps.
template <class T>
__device__ __forceinline__ void walk_light(const typename T::Params &p) {
    typedef typename T::Geom G;
    const WalkPools<typename T::Item> &w = p.walk;
    const int lane = threadIdx.x & 31;
    const int total = *(volatile const int32_t *)w.walk_ctr;
    const int nwarps = gridDim.x * LIGHT_WARPS;
    const int cap = p.n_envs * WALK_CONT_PER_ENV;
#pragma unroll 1
    for (int base = (blockIdx.x * LIGHT_WARPS + (threadIdx.x >> 5)) * 32; base < total; base += nwarps * 32) {
        const int i = base + lane;
        const bool has = i < total;
        typename T::Item it{};
        if (has) it = w.walkq[i];
        const auto v = T::view(p, it, has);
        int node = NODE_NEW, res = 0;
        Stack4 st{};
        if (has) res = stab_light<G>(v.g, v.root, (int)it.k, it.pack, v.pool, node, st);
        if (res == 1) atomicOr(&v.fbits()[it.c >> 5], 1u << (it.c & 31));
        if (has && res != 2) walk_done(v.n_pending());
        // continuations: walks high up in the bin descend through the deepest support DAGs (host statistics: resting height >= 0.6 H -> up to 8 heavy
        // visits, below -> at most 2), so they are pooled apart (from the END of the pool) and get fewer lanes per warp in the continuation kernel
        if (w.walk_fork) {  // fork-join continuation kernel: one queue of pieces, "enter `node` with the stack st" (pct_walkq.cuh)
            const uint32_t pm = __ballot_sync(FULL, res == 2);
            if (pm) {
                const PieceQueue pq{(WalkPiece *)w.contq, w.piece_ready, w.cont_ctr, w.piece_cap};
                int qb = 0;
                if (lane == 0) qb = pq_reserve_initial(pq, __popc(pm));
                qb = __shfl_sync(FULL, qb, 0);
                if (res == 2) {
                    const int idx = qb + __popc(pm & ((1u << lane) - 1));
                    if (idx < pq.cap) {
                        w.walk_pend[i] = 1;
                        pq.q[idx] = WalkPiece{(uint32_t)i, (uint8_t)node, (uint8_t)EDGE_NIL, 0, 0, st.cx, st.cy, st.m};
                    } else {  // never silent: the candidate stays infeasible and the env is flagged
                        atomicOr(v.flags(), PCT_FLAG_CAND_OVERFLOW);
                        walk_done(v.n_pending());
                        pq_piece_done(pq);
                    }
                }
            }
            continue;
        }
        const bool tall = T::tall(p, it);
        const uint32_t ps = __ballot_sync(FULL, res == 2 && !tall), pt = __ballot_sync(FULL, res == 2 && tall);
        if (ps | pt) {
            int qs = 0, qt = 0;
            if (lane == 0) {
                if (ps) qs = atomicAdd(w.cont_ctr, __popc(ps));
                if (pt) qt = atomicAdd(w.cont_ctr + 1, __popc(pt));
            }
            qs = __shfl_sync(FULL, qs, 0);
            qt = __shfl_sync(FULL, qt, 0);
            if (res == 2) {
                const uint32_t lt = (1u << lane) - 1;
                const int idx = tall ? qt + __popc(pt & lt) : qs + __popc(ps & lt);  // each class owns half of the pool (the counters may overshoot; the consumer clamps)
                if (idx < cap / 2) w.contq[tall ? cap - 1 - idx : idx] = WalkCont{(uint32_t)i, (uint32_t)node, st};
                else { atomicOr(v.flags(), PCT_FLAG_CAND_OVERFLOW); walk_done(v.n_pending()); }  // never silent: the candidate stays infeasible and the env is flagged
            }
        }
    }
}

// walk, stage 2: the continuations — every lane starts with the heavy visit its walk stopped at, then runs the general light / heavy state
// machine to the end of the walk.  Only `walk_lanes` lanes of a warp carry a walk (default 16; 4 for the tall walks): there are few
// continuations (3 per env) and each is a long serial chain; a full warp of them leaves
// fewer warps than the SMs have schedulers, 4-8 per warp multiply the warp instructions (measured sweep).  Blocks of WALK_WARPS warps.
// Expanded inside each continuation kernel (a macro, not an inlined function): the kernel's walk locals (the continuation, the view, the flags word)
// are passed by address to the non-inlined stab_virtual, so they live in local memory, and behind an inlined function boundary the compiler lays
// that frame out in another order — other stack offsets and registers in the stage that bounds a step.
#define PCT_WALK_CONT_BODY(T, p)                                                                                                                \
    typedef typename T::Geom G;                                                                                                                 \
    const int lane = threadIdx.x & 31;                                                                                                         \
    const int cap = p.n_envs * WALK_CONT_PER_ENV;                                                                                               \
    const int n_short = min(*(volatile const int32_t *)p.walk.cont_ctr, cap / 2), n_tall = min(*(volatile const int32_t *)(p.walk.cont_ctr + 1), cap / 2); \
    __syncthreads();                                                                                                                            \
    pdl_launch_dependents();  /* the emit kernel's blocks may become resident now (it also empties the pool counters: read above); each waits for ITS env's last walk */ \
    const int nwarps = gridDim.x * WALK_WARPS, Ls = p.walk.walk_lanes, Lt = p.walk.walk_lanes_tall;                                            \
    const int w_tall = (n_tall + Lt - 1) / Lt, w_all = w_tall + (n_short + Ls - 1) / Ls;                                                        \
    _Pragma("unroll 1")                                                                                                                         \
    for (int wi = blockIdx.x * WALK_WARPS + (threadIdx.x >> 5); wi < w_all; wi += nwarps) {  /* the tall walks (longest chains) are dealt first */ \
        const bool tw = wi < w_tall;                                                                                                            \
        const int L = tw ? Lt : Ls;                                                                                                             \
        const unsigned mask = L >= 32 ? FULL : ((1u << L) - 1u);                                                                                \
        if (lane >= L) continue;                                                                                                                \
        const int i = tw ? wi * Lt + lane : (wi - w_tall) * Ls + lane;                                                                          \
        const bool has = i < (tw ? n_tall : n_short);                                                                                           \
        WalkCont ct{};                                                                                                                          \
        typename T::Item it{};                                                                                                                  \
        if (has) { ct = p.walk.contq[tw ? cap - 1 - i : i]; it = p.walk.walkq[ct.item]; }                                                       \
        const auto v = T::view(p, it, has);                                                                                                     \
        int fl = 0;                                                                                                                             \
        const bool ok = stab_virtual<G>(v.g, v.root, (int)it.k, it.pack, v.pool, v.big(), v.lock(), fl, has, mask,                              \
                                        has ? (int)ct.node : NODE_NEW, &ct.st) != 0;                                                            \
        if (has && ok) atomicOr(&v.fbits()[it.c >> 5], 1u << (it.c & 31));                                                                     \
        if (has && fl) atomicOr(v.flags(), fl);                                                                                                 \
        if (has) walk_done(v.n_pending());                                                                                                      \
    }

// walk, stage 2, fork-join form (opt-in, PCT_B200_WALK=fork): the queue holds PIECES of walks (stab_piece: one chain of visits; a node with k >= 2 supports keeps
// its first subtree and publishes the other k - 1 as new pieces; protocol: pct_walkq.cuh).  A walk's verdict is the AND over its pieces:
// walk_pend[item] counts them, the piece that brings it to zero sets the feasibility bit (unless one failed) and releases the env's n_pending.
// The critical chain of a step's longest walk becomes its longest root-to-floor PATH instead of the sum over its visits (host statistics,
// scratch/stats_paths.py: 51 -> 34 visit units at the 99.99 % quantile) — and the stage did not get faster in
// measurements, whatever the number of helper warps, blocks per SM or pieces per warp: the continuation stage is bound by the issue rate of a few
// hundred divergent, latency-bound warps (warp instructions = thread instructions / 4.8 lanes, ~10 cycles each), not by its longest walk.  Kept as an
// opt-in because it is the measured answer to "would independent subtrees on separate lanes help?" and is parity-tested (tests/test_gpu_walk_fork.py).
struct PieceFork {
    PieceQueue pq;
    int32_t *pend;
    uint32_t item;
    int n_init;
    bool overflow;
    __device__ __forceinline__ void operator()(int child, int skip, double vx, double vy, double vm) {
        if (!pq_fork(pq, n_init, pend, WalkPiece{item, (uint8_t)child, (uint8_t)skip, 1, 0, vx, vy, vm})) overflow = true;
    }
};
// one piece: the chain of visits, then the walk's AND-reduction (walk_pend) and the queue's bookkeeping
template <class T>
__device__ __forceinline__ void run_piece(const typename T::Params &p, const PieceQueue &pq, int n_init, int slot) {
    const WalkPiece pc = pq.q[slot];
    if (slot >= n_init) pq.ready[slot] = 0;
    const typename T::Item it = p.walk.walkq[pc.item];
    const auto v = T::view(p, it, true);
    int32_t *pend = p.walk.walk_pend + pc.item;
    int fl = 0, ok = 0;
    if (!(*(volatile const int32_t *)pend & WALK_FAILED)) {  // a failed sibling has already decided the walk
        PieceFork fork{pq, pend, pc.item, n_init, false};
        ok = stab_piece<typename T::Geom>(v.g, v.root, (int)it.k, it.pack, v.pool, v.big(), v.lock(), fl, (int)pc.node, (int)pc.kind, (int)pc.skip,
                                          pc.a, pc.b, pc.c, fork);
        if (fork.overflow) { fl |= PCT_FLAG_CAND_OVERFLOW; ok = 0; }  // never silent: the candidate stays infeasible and the env is flagged
    }
    if (fl) atomicOr(v.flags(), fl);
    if (!ok) atomicOr(pend, WALK_FAILED);
    __threadfence();
    const int r = atomicSub(pend, 1);
    if ((r & (WALK_FAILED - 1)) == 1) {  // the walk's last piece
        if (!(r & WALK_FAILED)) atomicOr(&v.fbits()[it.c >> 5], 1u << (it.c & 31));
        walk_done(v.n_pending());
    }
    pq_piece_done(pq);
}
template <class T>
__device__ __forceinline__ void walk_fork(const typename T::Params &p) {
    const int lane = threadIdx.x & 31;
    const int wid = blockIdx.x * WALK_WARPS + (threadIdx.x >> 5), n_warps = gridDim.x * WALK_WARPS;
    const PieceQueue pq{(WalkPiece *)p.walk.contq, p.walk.piece_ready, p.walk.cont_ctr, p.walk.piece_cap};
    const int n_init = min(*(volatile const int32_t *)(pq.ctr + PQ_NINIT), pq.cap);  // written by the light-prefix kernel only (completed)
    const int L = p.walk.walk_lanes;
    pdl_launch_dependents();  // the emit kernel's blocks may become resident; each waits for ITS env's last walk
    if (n_init > 0) {
        // the light-prefix kernel's pieces: dealt statically
#pragma unroll 1
        for (int b = wid * L; b < n_init; b += n_warps * L) {
            if (lane < L && b + lane < n_init) run_piece<T>(p, pq, n_init, b + lane);
            __syncwarp();
        }
        // forked pieces: tickets
        const bool keep = wid < p.walk.walk_keep;
#pragma unroll 1
        for (;;) {
            int t0 = -1;
            if (lane == 0 && (keep || *(volatile const int32_t *)(pq.ctr + PQ_ALLOC) - *(volatile const int32_t *)(pq.ctr + PQ_HEAD) > 0))
                t0 = atomicAdd(pq.ctr + PQ_HEAD, L);
            t0 = __shfl_sync(FULL, t0, 0);
            if (t0 < 0) break;  // not a helper and nothing unclaimed in the queue: leave (SM slots for the emit kernel)
            bool fin = false;
            if (lane < L) {
                const int slot = n_init + t0 + lane;
                if (pq_wait(pq, slot)) run_piece<T>(p, pq, n_init, slot);
                else fin = true;
            }
            __syncwarp();
            if (__any_sync(FULL, fin)) break;  // a lane saw the end of all work
        }
    }
    if (lane == 0) pq_warp_exit(pq, n_warps, p.walk.walk_ctr);
}

// emit kernels, one thread per env: wait until the env's last walk has delivered.  The emit kernel is a programmatic dependent of the continuation
// kernel, so its blocks may run while walks are still in flight.  Bounded: a walk that never delivers shows up as PCT_FLAG_SYNC_TIMEOUT of its env.
template <class R>  // DEnvHot / CEnv: the record whose header holds the env's flags
__device__ __forceinline__ void wait_walks(const int32_t *n_pending, R *rec) {
    int spins = 0;
    while (*(volatile const int32_t *)n_pending > 0) {
        __nanosleep(spins < 16 ? 100 : 1000);
        if (++spins > (1 << 22)) { atomicOr(&rec->h.flags, PCT_FLAG_SYNC_TIMEOUT); break; }
    }
    __threadfence();
}

// emit kernels, one thread of the launch: empty the sequential walks' pool counters for the next step (every walk-kernel block has read them before
// it let the emit kernel start).  The fork-join kernel's counters are still live while the emit kernel starts: its last warp out empties them.
template <class Item>
__device__ __forceinline__ void reset_walk_pools(const WalkPools<Item> &w) {
    if (!w.walk_fork) { *w.walk_ctr = 0; w.cont_ctr[0] = 0; w.cont_ctr[1] = 0; }
}

}  // namespace pct
