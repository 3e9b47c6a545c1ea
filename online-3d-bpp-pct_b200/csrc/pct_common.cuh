// Shared device helpers: counter-based RNG, CPython tuple-hash / set-probe emulation, TMA (1-D bulk copy)
// and mbarrier wrappers for sm_90a.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "pct_pyhash.cuh"  // hash_double: _Py_HashDouble, shared with the host build of the tests

namespace pct {

constexpr unsigned FULL = 0xffffffffu;

// ---- counter-based generator shared with the host tests (oracle/pct_oracle.py rnd_u64) ----------------
__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    uint64_t z = x;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__host__ __device__ __forceinline__ uint64_t rnd_u64(uint64_t seed, uint64_t a, uint64_t b) {
    return splitmix64(splitmix64(seed ^ (a * 0x9E3779B97F4A7C15ull)) + b);
}
constexpr uint64_t DENSITY_SALT = 0xABCDEFull;
// uniform in (0,1): np.random.random() re-drawn while == 0 (D:bin3D.py:82-84)
__host__ __device__ __forceinline__ double rnd_density(uint64_t seed, uint64_t a, uint64_t b) {
    uint64_t r = rnd_u64(seed ^ DENSITY_SALT, a, b) >> 11;
    if (r == 0) r = 1;
    return (double)r * (1.0 / 9007199254740992.0);
}

// ---- CPython 3.12 tuple hash of a 6-tuple (Objects/tupleobject.c, xxHash-derived) --------------------
// Call sites in the reference: the `posVec` sets of D:space.py:535,565-569 / C:space.py:532,563-567.
constexpr uint64_t XXP1 = 11400714785074694791ull, XXP2 = 14029467366897019727ull, XXP5 = 2870177450012600261ull;
__device__ __forceinline__ uint64_t tuple_hash6(const uint64_t lane[6]) {
    uint64_t acc = XXP5;
#pragma unroll
    for (int i = 0; i < 6; i++) {
        acc += lane[i] * XXP2;
        acc = (acc << 31) | (acc >> 33);
        acc *= XXP1;
    }
    acc += 6ull ^ (XXP5 ^ 3527539ull);
    if (acc == ~0ull) return 1546275796ull;
    return acc;
}
__device__ __forceinline__ uint64_t tuple_hash_n(const uint64_t *lane, int n) {
    uint64_t acc = XXP5;
    for (int i = 0; i < n; i++) {
        acc += lane[i] * XXP2;
        acc = (acc << 31) | (acc >> 33);
        acc *= XXP1;
    }
    acc += (uint64_t)n ^ (XXP5 ^ 3527539ull);
    if (acc == ~0ull) return 1546275796ull;
    return acc;
}

// ---- CPython 3.12 set insertion, a warp of keys at a time (the candidate lists: pct_cand.cuh, pct_cand_c.cuh) ----------------------
// A lane's place on its key's probe sequence (setobject.c, no deletions): home slot hash & mask; from each window start i the slots
// i .. i + 9 when i + 9 <= mask, else i alone; then perturb >>= 5, i = (i * 5 + 1 + perturb) & mask.
struct SetProbe {
    uint64_t perturb;
    uint32_t i, j;  // window start, offset in the window
    __device__ __forceinline__ void home(uint64_t hash, uint32_t mask) { perturb = hash; i = (uint32_t)hash & mask; j = 0; }
    __device__ __forceinline__ uint32_t slot() const { return i + j; }
    __device__ __forceinline__ void next(uint32_t mask) {
        if (j < 9 && i + 9 <= mask) { j++; return; }
        j = 0;
        perturb >>= 5;
        i = (uint32_t)((uint64_t)i * 5 + 1 + perturb) & mask;
    }
};
// Walks on from the current slot to the first one that is empty (false) or holds the key (`eq`, true); the probe stays there.
template <typename SlotT, typename Eq>
__device__ __forceinline__ bool set_seek(const SlotT *tab, uint32_t mask, SetProbe &pr, Eq eq) {
#pragma unroll 1
    for (;;) {
        const SlotT e = tab[pr.slot()];
        if (e == (SlotT)~(SlotT)0) return false;
        if (eq(e)) return true;
        pr.next(mask);
    }
}
// Ordered parallel insertion.  Every `pending` lane holds a key that is not in the table, and its probe stands on the first slot of its
// sequence that is empty now.  Let c be the lowest pending lane whose slot a lower pending lane holds too.  Inserting the pending lanes
// below c, in lane order, one at a time, puts each of them on the slot it stands on: slots only fill, so the slots before it on its
// sequence are still occupied, and no lower lane of the group takes its slot (their slots all differ).  So they all commit at once;
// `room` caps them at the insertion that makes the set grow.  Lanes from c on wait, even one that holds the lowest claim on its slot: in
// serial order c, or a lane after it, may take that slot first.  A waiting lane whose slot was taken walks on from it (set_seek) to the
// slot a serial insertion would reach at its turn.  The lowest pending lane always commits, so a chunk takes at most as many rounds as
// keys.  Returns the mask of committing lanes (0: none pending).
__device__ __forceinline__ uint32_t set_claim_round(bool pending, uint32_t slot, int lane, uint32_t room) {
    const uint32_t pm = __ballot_sync(FULL, pending);
    const uint32_t same = __match_any_sync(FULL, pending ? slot : 0xFFFFFFFFu) & pm;
    const uint32_t lost = __ballot_sync(FULL, pending && (same & ((1u << lane) - 1)));
    uint32_t cm = pm & ((lost & (0u - lost)) - 1u);  // the pending lanes below the first loser (all of them when none lost)
#pragma unroll 1
    while ((uint32_t)__popc(cm) > room) cm &= ~(0x80000000u >> __clz(cm));
    return cm;
}
// set_table_resize: the keys of `old` re-inserted into the empty table `nt` in old slot order (set_insert_clean: no comparisons), 32 old
// slots at a time in claim rounds.  `hash_of(key)`: the key's hash.  Ends with the warp's stores visible to every lane.
template <typename SlotT, typename HashOf>
__device__ __forceinline__ void set_rehash(const SlotT *old, uint32_t omask, SlotT *nt, uint32_t nmask, int lane, HashOf hash_of) {
    constexpr SlotT EMPTY = (SlotT)~(SlotT)0;
#pragma unroll 1
    for (uint32_t b = 0; b <= omask; b += 32) {
        const uint32_t s = b + lane;
        const SlotT e = s <= omask ? old[s] : EMPTY;
        bool pend = e != EMPTY;
        SetProbe pr{0, 0, 0};
        if (pend) pr.home(hash_of(e), nmask);
#pragma unroll 1
        for (;;) {
            if (pend) set_seek(nt, nmask, pr, [](SlotT) { return false; });
            const uint32_t cm = set_claim_round(pend, pr.slot(), lane, 32);
            if (!cm) break;
            if ((cm >> lane) & 1) { nt[pr.slot()] = e; pend = false; }
            __syncwarp();
        }
    }
}

// ---- TMA 1-D bulk copies + mbarrier (PTX ISA 8.x; SASS: UBLKCP / SYNCS) ---------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_1d(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void tma_store_1d(void *gmem_dst, const void *smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst), "r"(smem_u32(smem_src)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void tma_store_commit_wait() {
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

__device__ __forceinline__ void tma_store_commit_wait_all() {  // completion of the WRITES (not only of the source reads)
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }

// ---- programmatic dependent launch + per-env hand-over flags -------------------------------------------------
// The step is three kernels over the same envs; each lasts as long as its slowest env, so whole SMs idle in every tail.
// With PDL the next kernel's blocks become resident as soon as every block of the previous one has STARTED; the data
// dependency is per env, carried by a flag: the producer publishes `epoch` after its last write of env e, the consumer of
// env e polls for it.  No block ever waits for a block that is not already resident, so the scheme cannot deadlock;
// the poll is bounded anyway (a timeout is reported as a flag, never a hang).
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void env_publish(int32_t *flag, int32_t epoch) {
    __threadfence();
    asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(flag), "r"(epoch) : "memory");
}
__device__ __forceinline__ bool env_wait(const int32_t *flag, int32_t epoch) {
    // poll with relaxed loads (served by L2, no L1 invalidation per iteration: the continuous kernels keep their working set in
    // L1-cached global memory and share the SM with the pollers), then ONE acquire fence once the flag is seen
    for (int it = 0; it < (1 << 22); it++) {
        int32_t v;
        asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(flag) : "memory");
        if (v == epoch) {
            asm volatile("fence.acq_rel.gpu;" ::: "memory");
            return true;
        }
        __nanosleep(it < 64 ? 64 : 512);
    }
    return false;
}

// shuffle=True (D:bin3D.py:114-115 / C:bin3D.py:126-127): one warp permutes the ordered candidate list list[0..n) in place.  Definition
// (include/pct_b200.h, pct_config::shuffle): stable argsort of the keys rnd_u64(seed ^ SALT, global env id, draws << 16 | i).  Rank by
// counting (n^2 / 32 key comparisons per warp; n is 38 on average, <= 1228); keys[n] and tmp[n] are scratch in global memory.
constexpr uint64_t SHUFFLE_SALT = 0x5AFE5EEDull;
template <typename T>
__device__ __noinline__ void shuffle_candidates(T *list, int n, uint64_t *keys, T *tmp, uint64_t seed, uint64_t gid, uint64_t draws, int lane) {
    if (n < 2) return;
    for (int i = lane; i < n; i += 32) keys[i] = rnd_u64(seed ^ SHUFFLE_SALT, gid, (draws << 16) | (uint64_t)i);
    __syncwarp();
    for (int i = lane; i < n; i += 32) {
        const uint64_t ki = keys[i];
        int r = 0;
#pragma unroll 4
        for (int j = 0; j < n; j++) {
            const uint64_t kj = keys[j];
            r += (int)(kj < ki || (kj == ki && j < i));
        }
        tmp[r] = list[i];
    }
    __syncwarp();
    for (int i = lane; i < n; i += 32) list[i] = tmp[i];
    __syncwarp();
}

__device__ __forceinline__ int warp_incl_scan(int v, int lane) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        int t = __shfl_up_sync(FULL, v, d);
        if (lane >= d) v += t;
    }
    return v;
}

}  // namespace pct
