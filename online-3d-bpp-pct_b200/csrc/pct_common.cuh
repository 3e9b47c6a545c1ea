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
