// TEST INFRASTRUCTURE — device unit library of the candidate lists' CPython-set emulation (tests/test_gpu_candidate_units.py).
// The product headers are included unchanged, so every launcher below runs the product's own code, compiled with the product's flags
// (Makefile): the rotation table and canonical keys (pct_rot.cuh), the discrete set emulation build_candidates (pct_cand.cuh) in both
// shared-memory layouts of the step's candidates kernel, the continuous one (PCTC_CANDIDATES_BODY, pct_cand_c.cuh) on a CEnv in global
// memory, and the keyed shuffle (pct_common.cuh).  Launchers take raw device pointers (torch tensors), run on the legacy default stream
// and synchronise: they return the CUDA error code (0 = success).
#include <cstdint>
#include <cuda_runtime.h>
#include "pct_cand.cuh"
#include "pct_cand_c.cuh"
#include "pct_rot.cuh"
#include "pct_common.cuh"
#include "pct_pyhash.cuh"

using namespace pct;

#define GRID(n) dim3((unsigned)(((n) + 127) / 128)), dim3(128)
#define FINISH() do { cudaError_t e_ = cudaGetLastError(); if (e_ != cudaSuccess) return (int)e_; return (int)cudaDeviceSynchronize(); } while (0)

constexpr int OUT_MAX = TAB_A;  // per-case output slots of the ordered lists (the list can hold up to 1229 keys: the overflowing one included)

// item[n][3], R[n] -> out[n][25] = d[6][3], valid, canon[6] of make_rot_tab
__global__ void k_rot_tab(const int *item, const int *R, int n, int *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int nb[3] = {item[3 * i], item[3 * i + 1], item[3 * i + 2]};
    RotTab rt;
    make_rot_tab(nb, R[i], rt);
    int *o = out + 25 * i;
    for (int r = 0; r < 6; r++)
        for (int c = 0; c < 3; c++) o[3 * r + c] = rt.d[r][c];
    o[18] = rt.valid;
    for (int r = 0; r < 6; r++) o[19 + r] = rt.canon[r];
}
extern "C" int cu_rot_tab(const int *item, const int *R, int n, int *out) { if (n > 0) k_rot_tab<<<GRID(n)>>>(item, R, n, out); FINISH(); }

// key[n] of the item item[n][3] (rotation table with R[n]) -> key_hash<BITS>
template <int BITS>
__global__ void k_key_hash(const uint32_t *key, const int *item, const int *R, int n, unsigned long long *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int nb[3] = {item[3 * i], item[3 * i + 1], item[3 * i + 2]};
    RotTab rt;
    make_rot_tab(nb, R[i], rt);
    out[i] = key_hash<BITS>(key[i], &rt);
}
extern "C" int cu_key_hash(int bits, const uint32_t *key, const int *item, const int *R, int n, unsigned long long *out) {
    if (n > 0) {
        if (bits == 4) k_key_hash<4><<<GRID(n)>>>(key, item, R, n, out);
        else k_key_hash<8><<<GRID(n)>>>(key, item, R, n, out);
    }
    FINISH();
}

// lanes[n][6] (element hashes) -> tuple_hash6
__global__ void k_tuple_hash6(const unsigned long long *lanes, int n, unsigned long long *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t l[6];
    for (int c = 0; c < 6; c++) l[c] = lanes[6 * i + c];
    out[i] = tuple_hash6(l);
}
extern "C" int cu_tuple_hash6(const unsigned long long *lanes, int n, unsigned long long *out) { if (n > 0) k_tuple_hash6<<<GRID(n)>>>(lanes, n, out); FINISH(); }

// query q = (case, code): the EMS list of the case starts at ems + 6 * ems_off[case], its item is item[case][3] ->
// tup[q][6] = cand_tuple, hash[q] = cand_hash_c(tup), dims[q][3] + valid[q] = rot_dims_c(item, (code >> 2) & 7)
__global__ void k_cand_c(const double *ems, const int *ems_off, const double *item, const int *q_case, const int *q_code, int n, double *tup,
                         unsigned long long *hash, double *dims, int *valid) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int c = q_case[i];
    const double nb[3] = {item[3 * c], item[3 * c + 1], item[3 * c + 2]};
    double t[6];
    cand_tuple((uint16_t)q_code[i], (const double (*)[6])(ems + 6 * (size_t)ems_off[c]), nb, t);
    for (int k = 0; k < 6; k++) tup[6 * i + k] = t[k];
    hash[i] = cand_hash_c(t);
    double sx, sy, sz;
    valid[i] = rot_dims_c(nb, (q_code[i] >> 2) & 7, sx, sy, sz);
    dims[3 * i] = sx; dims[3 * i + 1] = sy; dims[3 * i + 2] = sz;
}
extern "C" int cu_cand_c(const double *ems, const int *ems_off, const double *item, const int *q_case, const int *q_code, int n, double *tup,
                         unsigned long long *hash, double *dims, int *valid) {
    if (n > 0) k_cand_c<<<GRID(n)>>>(ems, ems_off, item, q_case, q_code, n, tup, hash, dims, valid);
    FINISH();
}

// ---- discrete: build_candidates, one warp (block) per case, shared memory laid out as the step's candidates kernel lays it out:
// A_SLOTS = 2048 (BIGSM: the 2048 stage is table A itself) or 128 (settings 1/3: the 2048 stage is a global buffer, `big`).
// Case c: ems[c][E_MAX][6] with n_ems[c] entries, item[c][3], R[c]; n_raw[c] >= 0 selects the raw-key mode on raw[c][RAW_MAX].
// -> keys[c][OUT_MAX] (the ordered list, as 32-bit values), cnt[c], flags[c].
template <typename SlotT, bool BIGSM>
__global__ void __launch_bounds__(32) k_build_d(const int16_t *ems, const int *n_ems, const int *item, const int *R, const uint32_t *raw,
                                                const int *n_raw, uint32_t *keys, int *cnt, int *flags, SlotT *big) {
    constexpr int A_SLOTS = BIGSM ? TAB_A : 128;
    __shared__ __align__(16) SlotT tabA[A_SLOTS];
    __shared__ __align__(16) SlotT tabB[TAB_B];
    __shared__ RotTab rt;
    __shared__ SetStage stg;
    const int c = blockIdx.x, lane = threadIdx.x;
    const int nb[3] = {item[3 * c], item[3 * c + 1], item[3 * c + 2]};
    if (lane == 0) make_rot_tab(nb, R[c], rt);
    __syncwarp();
    const int16_t (*e)[6] = (const int16_t (*)[6])(ems + (size_t)c * E_MAX * 6);
    SlotT *tbig = BIGSM ? tabA : big + (size_t)c * TAB_A;
    const CandList<SlotT> cl = n_raw[c] >= 0
        ? build_candidates<SlotT>(e, n_ems[c], &rt, R[c], tabA, tabB, tbig, &stg, lane, raw + (size_t)c * RAW_MAX, n_raw[c])
        : build_candidates<SlotT>(e, n_ems[c], &rt, R[c], tabA, tabB, tbig, &stg, lane);
    for (int t = lane; t < cl.n && t < OUT_MAX; t += 32) keys[(size_t)c * OUT_MAX + t] = cl.keys[t];
    if (lane == 0) { cnt[c] = cl.n; flags[c] = cl.flags; }
}
extern "C" int cu_build_d(int bits, int bigsm, const int16_t *ems, const int *n_ems, const int *item, const int *R, const uint32_t *raw,
                          const int *n_raw, int n, uint32_t *keys, int *cnt, int *flags, void *big) {
    if (n > 0) {
        if (bits == 16 && bigsm) k_build_d<uint16_t, true><<<n, 32>>>(ems, n_ems, item, R, raw, n_raw, keys, cnt, flags, (uint16_t *)big);
        else if (bits == 16) k_build_d<uint16_t, false><<<n, 32>>>(ems, n_ems, item, R, raw, n_raw, keys, cnt, flags, (uint16_t *)big);
        else if (bigsm) k_build_d<uint32_t, true><<<n, 32>>>(ems, n_ems, item, R, raw, n_raw, keys, cnt, flags, (uint32_t *)big);
        else k_build_d<uint32_t, false><<<n, 32>>>(ems, n_ems, item, R, raw, n_raw, keys, cnt, flags, (uint32_t *)big);
    }
    FINISH();
}

// ---- continuous: PCTC_CANDIDATES_BODY expanded as pctc_candidates_kernel expands it, one warp (block) per case on env[c] (global memory).
// Case c: ems[ems_off[c] ..), n_ems[c] entries (<= CE_MAX), item[c][3], R[c], draw[c] (the header's draw position, for the shuffle keys);
// the shuffle's env id is env_id_base + c.  -> codes[c][OUT_MAX], cnt[c], flags[c].
__global__ void __launch_bounds__(32) k_build_c(const double *ems, const int *ems_off, const double *item, const int *Rr, const long long *draw,
                                                CEnv *env, int shuffle, unsigned long long seed, long long env_id_base, uint16_t *codes, int *cnt_out,
                                                int *flags) {
    __shared__ uint32_t tabA[CC_TAB], tabB[512];
    __shared__ uint64_t stg_h[32], rs_h[32];
    __shared__ uint32_t rs_c[32];
    __shared__ uint16_t stg_c[32];
    const int lane = threadIdx.x, e = blockIdx.x;
    CEnv *ev = env + e;
    const int n_ems = ems_off[e + 1] - ems_off[e];
    for (int t = lane; t < 6 * n_ems; t += 32) (&ev->ems[0][0])[t] = ems[6 * (size_t)ems_off[e] + t];
    if (lane == 0) {
        ev->h.n_ems = n_ems;
        ev->h.draw_pos = draw[e];
        for (int k = 0; k < 3; k++) ev->h.next_box[k] = item[3 * e + k];
    }
    __syncwarp();
    CParams p = {};
    p.shuffle = shuffle;
    p.seed = seed;
    p.env_id_base = env_id_base;
    int fl = 0;
    const CHdr &h = ev->h;
    const double nb[3] = {h.next_box[0], h.next_box[1], h.next_box[2]};
    const int R = Rr[e];
    PCTC_CANDIDATES_BODY
    for (int t = lane; t < cnt && t < OUT_MAX; t += 32) codes[(size_t)e * OUT_MAX + t] = ev->cand[t];
    if (lane == 0) { cnt_out[e] = cnt; flags[e] = fl; }
}
extern "C" size_t cu_cenv_bytes() { return sizeof(CEnv); }
extern "C" int cu_build_c(const double *ems, const int *ems_off, const double *item, const int *R, const long long *draw, int n, void *env, int shuffle,
                          unsigned long long seed, long long env_id_base, uint16_t *codes, int *cnt, int *flags) {
    if (n > 0) k_build_c<<<n, 32>>>(ems, ems_off, item, R, draw, (CEnv *)env, shuffle, seed, env_id_base, codes, cnt, flags);
    FINISH();
}

// ---- shuffle_candidates<T> on caller lists: case c permutes list[c][0 .. n[c]) (stride OUT_MAX) with (seed, gid[c], draws[c]); keys / tmp are
// per-case global scratch as in the step kernels
template <typename T>
__global__ void __launch_bounds__(32) k_shuffle(T *list, const int *n, const unsigned long long *gid, const unsigned long long *draws, unsigned long long seed,
                                                unsigned long long *keys, T *tmp) {
    const int c = blockIdx.x;
    shuffle_candidates<T>(list + (size_t)c * OUT_MAX, n[c], (uint64_t *)keys + (size_t)c * OUT_MAX, tmp + (size_t)c * OUT_MAX, seed, gid[c], draws[c],
                          threadIdx.x);
}
extern "C" int cu_shuffle(int bits, void *list, const int *n, const unsigned long long *gid, const unsigned long long *draws, unsigned long long seed,
                          int n_case, unsigned long long *keys, void *tmp) {
    if (n_case > 0) {
        if (bits == 16) k_shuffle<uint16_t><<<n_case, 32>>>((uint16_t *)list, n, gid, draws, seed, keys, (uint16_t *)tmp);
        else k_shuffle<uint32_t><<<n_case, 32>>>((uint32_t *)list, n, gid, draws, seed, keys, (uint32_t *)tmp);
    }
    FINISH();
}
extern "C" int cu_out_max() { return OUT_MAX; }
extern "C" int cu_e_max() { return E_MAX; }
extern "C" int cu_raw_max() { return RAW_MAX; }
extern "C" int cu_ce_max() { return CE_MAX; }
