// Item preview and item override of the discrete env (pct_preview_items / pct_set_items, include/pct_b200.h).
//
// Preview: one thread per (row, j).  Column 0 is the env's current item; column j >= 1 is what draw_item delivers on a copy of
// the header whose draw position is advanced by j - 1, so the item formulas stay in draw_item alone.  Nothing is written to the env.
// The buffered preview (pct_buffer_preview_items) is the same kernel body shifted by one column: its entry j is the draw at position + j.
//
// Override: pct_set_items_kernel stands in for the apply kernel of a step.  It writes the listed envs' next_box / next_den and
// initialises every env's info record the way the apply kernel does for a successful step (counter, sticky flags, zeros); the
// rest of the step's pipeline (candidates, walks, emit) then re-expands every env of the batch (launch_discrete with apply = false).  The selected
// form (pct_set_items_only) writes the listed envs' items and records and re-expands those envs alone.
//
// A translation unit of its own (see pct_draw.cuh).
#include "pct_common.cuh"
#include "pct_kernels.h"
#include "pct_draw.cuh"

namespace pct {

constexpr int ITEM_THREADS = 256;

// entry j of row r is preview column j + C0: C0 = 0 for pct_preview_items, C0 = 1 for pct_buffer_preview_items (a buffered env's header
// item is not one of its slots; entry 0 is the next draw)
template <int C0>
__device__ __forceinline__ void preview_entry(const DParams &p, const ItemParams &ip) {
    const int64_t t = (int64_t)blockIdx.x * ITEM_THREADS + threadIdx.x;
    if (t >= (int64_t)ip.n * ip.k) return;
    const int r = (int)(t / ip.k), j = (int)(t - (int64_t)r * ip.k) + C0;
    const int e = ip.env ? ip.env[r] : r;
    double *o = ip.out + (size_t)t * 4;
    if (e < 0 || e >= p.n_envs) {  // not an env of this handle: a zero row
        o[0] = 0; o[1] = 0; o[2] = 0; o[3] = 0;
        return;
    }
    DHdr h = p.hot[e].h;
    if (j > 0) {
        h.draw_pos += j - 1;
        draw_item(p, e, h);
    }
    o[0] = h.next_box[0]; o[1] = h.next_box[1]; o[2] = h.next_box[2]; o[3] = h.next_den;
}

__global__ void __launch_bounds__(ITEM_THREADS) pct_preview_kernel(const DParams p, const ItemParams ip) { preview_entry<0>(p, ip); }
__global__ void __launch_bounds__(ITEM_THREADS) pct_buf_preview_kernel(const DParams p, const ItemParams ip) { preview_entry<1>(p, ip); }

// thread t: item t of the call (if t < n) and the info record of env t (if t < n_envs); the two never touch the same fields.
// SEL (pct_set_items_only): thread t writes item t and the info record of its env, nothing else.
template <bool SEL = false>
__global__ void __launch_bounds__(ITEM_THREADS) pct_set_items_kernel(const DParams p, const ItemParams ip) {
    const int t = blockIdx.x * ITEM_THREADS + threadIdx.x;
    if (t < ip.n) {
        const int e = ip.env ? ip.env[t] : t;
        if (e >= 0 && e < p.n_envs) {
            const int32_t *it = (const int32_t *)ip.items + (size_t)t * 3;
            DHdr &h = p.hot[e].h;
            // a container side is at most 255 (pct_create), the range of the rotation table: a larger side fits nowhere either way
            h.next_box[0] = min(max(it[0], 0), 255); h.next_box[1] = min(max(it[1], 0), 255); h.next_box[2] = min(max(it[2], 0), 255);
            if (ip.density) h.next_den = ip.density[t];
            if (SEL && p.info) {
                pct_step_info info{};
                info.counter = h.n_box;
                info.flags = h.flags;
                p.info[e] = info;
            }
        }
    }
    if (!SEL && t < p.n_envs && p.info) {
        const DHdr &h = p.hot[t].h;
        pct_step_info info{};
        info.counter = h.n_box;
        info.flags = h.flags;
        p.info[t] = info;
    }
}

cudaError_t launch_preview_discrete(const DParams &p, const ItemParams &ip, cudaStream_t st) {
    const int64_t n = (int64_t)ip.n * ip.k;
    pct_preview_kernel<<<(unsigned)((n + ITEM_THREADS - 1) / ITEM_THREADS), ITEM_THREADS, 0, st>>>(p, ip);
    return cudaGetLastError();
}

cudaError_t launch_buffer_preview_discrete(const DParams &p, const ItemParams &ip, cudaStream_t st) {
    const int64_t n = (int64_t)ip.n * ip.k;
    pct_buf_preview_kernel<<<(unsigned)((n + ITEM_THREADS - 1) / ITEM_THREADS), ITEM_THREADS, 0, st>>>(p, ip);
    return cudaGetLastError();
}

cudaError_t launch_set_items_discrete(const DParams &p, const ItemParams &ip, cudaStream_t st, const EnvSel *sel) {
    const int n = sel ? ip.n : max(ip.n, p.n_envs);
    if (sel) pct_set_items_kernel<true><<<(n + ITEM_THREADS - 1) / ITEM_THREADS, ITEM_THREADS, 0, st>>>(p, ip);
    else pct_set_items_kernel<<<(n + ITEM_THREADS - 1) / ITEM_THREADS, ITEM_THREADS, 0, st>>>(p, ip);
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) return err;
    return launch_discrete(p, st, nullptr, false, sel);
}

}  // namespace pct
