// Discrete PCT environment: batched reset / step kernels for sm_90a.
//
// One warp owns one environment for the whole step:
//   TMA bulk load of the env's packed record (header + placed boxes + EMS list) HBM -> shared memory
//   -> decode action -> real placement (warp max-reduce over placed boxes for the resting height,
//      lane 0 runs the load-propagating stability update) -> EMS update (warp ballot / scan compaction)
//   -> candidate leaves in CPython-set order (hash table in shared memory)
//   -> feasibility, ONE LANE PER CANDIDATE (bounds, resting height over all placed boxes, stacking stability)
//   -> ordered compaction of the first `leaf_node_holder` feasible leaves (ballot + popc)
//   -> coalesced observation write, TMA bulk store of the record back to HBM.
//
// Reference behaviour restated here (D: = pct_envs/PctDiscrete0/ in the reference repo):
//   PackingDiscrete.step / reset / cur_observation / get_possible_position / LeafNode2Action  D:bin3D.py:61-188
//   Space.drop_box / drop_box_virtual / check_box / update_height_graph                       D:space.py:316-454
//   Space.GENEMS / Difference / EliminateInscribedEMS / EMSPoint                               D:space.py:457-570
//   ShmemVecEnv worker auto-reset                                                              wrapper/shmem_vec_env.py:139-143
// The height map of the reference is not materialised: max(plain[lx:lx+x, ly:ly+y]) equals the maximum top
// over placed boxes whose footprint overlaps the query footprint (update_height_graph sets covered cells to
// the new top, which is >= every older value there).
//
// Code-size discipline: the first version of this kernel was instruction-fetch bound (ncu r1a:
// stalled_no_instruction 11.3 of 19 stalled warps per issue, 202 KB of SASS).  Phases are __noinline__
// functions, loops over chunks are dynamic, candidate keys are canonical integers compared with one
// instruction instead of being re-derived from the EMS list on every probe.
#include "pct_common.cuh"
#include "pct_stability.cuh"
#include "pct_kernels.h"
#include "pct_geom.cuh"
#include "pct_walks.cuh"
#include "pct_obs.cuh"
#include "pct_block.cuh"

namespace pct {

// ------------------------------------------------------------------------------------------------------
// NodeD / GeomD (geometry policy of the stability routine) and rest_height: pct_geom.cuh

// ---- shared-memory layout of one warp ------------------------------------------------------------------
// Candidate keys are canonical integers: xs | ys << B | zs << 2B | rot << 3B  (rot = first rotation index with
// the same oriented dims).  B = 4 bits when every container side is <= 16 (16-bit table slots), else 8 bits
// (32-bit slots).
// The CPython-set emulation walks table sizes 8 -> 32 -> 128 -> 512 -> 2048, alternating between two buffers:
// A holds the 8 / 128 / 2048 stages, B the 32 / 512 stages.  BIGSM = true keeps the 2048 stage in shared memory
// (setting 2: 6 orientations, hundreds of candidates per step); BIGSM = false (settings 1/3: <= 306 candidates in
// practice) keeps A at 128 slots and spills the rare 2048 stage to the env's cold record in HBM, which keeps a warp's
// share of shared memory at 5056 / 6336 B (16- / 32-bit slots).  4096 envs on 132 SMs run in one resident wave when 32 warps fit in one SM
// (ceil(4096 / 132) = 32): 16 two-warp blocks take 162 / 203 KB of the 227 KB, and the registers must stay at 64 per thread
// (K2_MINB = 16; without the bound sm_90a gives the kernel 72-74 and 28 warps fit).  Measured on the H100, the bound loses: the tail of
// 1.14 waves costs less than the extra instructions at 64 registers, so the default leaves the registers free.
template <typename SlotT, bool BIGSM>
struct Lay {
    static constexpr int A_SLOTS = BIGSM ? TAB_A : 128;
    static constexpr int HOT = 0;
    static constexpr int TAB_A_OFF = HOT_PREFIX;
    static constexpr int TAB_B_OFF = TAB_A_OFF + A_SLOTS * sizeof(SlotT);
    static constexpr int LEAF = TAB_B_OFF + TAB_B * sizeof(SlotT);  // NL_MAX x 6 x i16
    static constexpr int MISC = LEAF + NL_MAX * 12;                 // mbarrier (8) + lock (4) + pad (4) + RotTab (32) + SetStage (384)
    static constexpr int PER_WARP = MISC + 48 + 384;
    static constexpr int BITS = sizeof(SlotT) == 2 ? 4 : 8;
    static_assert(TAB_A_OFF % 16 == 0 && PER_WARP % 16 == 0, "alignment");
    static_assert(E_MAX * 12 <= MISC - TAB_A_OFF, "EMS temp aliases tables + leaf buffer");
};

}  // namespace pct
#include "pct_rot.cuh"  // RotTab, make_rot_tab, key_pack / key_unpack / key_hash
namespace pct {

// ---- EMS update (GENEMS + Difference + EliminateInscribedEMS, D:space.py:457-531) -------------------------
__device__ __noinline__ int genems_warp(int16_t (*ems)[6], const int n0, int16_t (*tmp)[6], uint2 *pk, const int16_t *it, double low_bound, int lane,
                                        int &flags) {
    const double lb = low_bound == 0 ? 0.1 : low_bound;
    const int nch = (n0 + 31) >> 5;
    // pass 1: survivors (EMS not intersecting the new box) keep their order
    int off = 0;
#pragma unroll 1
    for (int c = 0; c < nch; c++) {
        const int i = c * 32 + lane;
        bool keep = false;
        if (i < n0) {
            const int16_t *m = ems[i];
            keep = !(max((int)m[0], (int)it[0]) < min((int)m[3], (int)it[3]) && max((int)m[1], (int)it[1]) < min((int)m[4], (int)it[4]) &&
                     max((int)m[2], (int)it[2]) < min((int)m[5], (int)it[5]));
        }
        const uint32_t bm = __ballot_sync(FULL, keep);
        if (keep) {
            const int p = off + __popc(bm & ((1u << lane) - 1));
#pragma unroll
            for (int t = 0; t < 6; t++) tmp[p][t] = ems[i][t];
        }
        off += __popc(bm);
    }
    // pass 2: children of the intersected EMS, parent order then fixed child order (left, right, front, back, top)
    bool overflow = false;
#pragma unroll 1
    for (int c = 0; c < nch; c++) {
        const int i = c * 32 + lane;
        uint32_t cm = 0;
        int a1 = 0, b1 = 0, c1 = 0, a2 = 0, b2 = 0, c2 = 0, x1 = 0, y1 = 0, x2 = 0, y2 = 0, z2 = 0;
        if (i < n0) {
            const int16_t *m = ems[i];
            a1 = m[0]; b1 = m[1]; c1 = m[2]; a2 = m[3]; b2 = m[4]; c2 = m[5];
            x1 = max(a1, (int)it[0]); y1 = max(b1, (int)it[1]);
            const int z1 = max(c1, (int)it[2]);
            x2 = min(a2, (int)it[3]); y2 = min(b2, (int)it[4]); z2 = min(c2, (int)it[5]);
            if (x1 < x2 && y1 < y2 && z1 < z2) {  // clamp + degenerate test of D:space.py:464-475
                const bool ux = (double)(a2 - a1) >= lb, uy = (double)(b2 - b1) >= lb, uz = (double)(c2 - c1) >= lb;
                if ((double)(x1 - a1) >= lb && uy && uz) cm |= 1;
                if ((double)(a2 - x2) >= lb && uy && uz) cm |= 2;
                if (ux && (double)(y1 - b1) >= lb && uz) cm |= 4;
                if (ux && (double)(b2 - y2) >= lb && uz) cm |= 8;
                if (ux && uy && (double)(c2 - z2) >= lb) cm |= 16;
            }
        }
        const int cnt = __popc(cm);
        const int incl = warp_incl_scan(cnt, lane);
        int p = off + incl - cnt;
#pragma unroll 1
        for (int ch = 0; ch < 5 && cm; ch++) {
            if (!(cm & (1u << ch))) continue;
            int q0 = a1, q1 = b1, q2 = c1, q3 = a2, q4 = b2, q5 = c2;
            if (ch == 0) q3 = x1;
            else if (ch == 1) q0 = x2;
            else if (ch == 2) q4 = y1;
            else if (ch == 3) q1 = y2;
            else q2 = z2;
            if (p < EMS_TMP_MAX) {
                tmp[p][0] = (int16_t)q0; tmp[p][1] = (int16_t)q1; tmp[p][2] = (int16_t)q2;
                tmp[p][3] = (int16_t)q3; tmp[p][4] = (int16_t)q4; tmp[p][5] = (int16_t)q5;
            } else overflow = true;
            p++;
        }
        off += __shfl_sync(FULL, incl, 31);
    }
    if (__any_sync(FULL, overflow)) flags |= PCT_FLAG_EMS_OVERFLOW;
    const int n = off < EMS_TMP_MAX ? off : EMS_TMP_MAX;  // intermediate list (survivors + children), before the inscribed-EMS purge
    __syncwarp();
    // EliminateInscribedEMS: drop i if some j != i contains it (non-strict; identical twins delete each other).
    // The O(n^2) containment test was a large share of the apply kernel's warp instructions: six 16-bit loads and
    // six compares per pair.  Coordinates are <= 255 (pct_create), so an EMS packs into two words of three 9-bit fields — lows as they are, highs
    // as 255 - v, which turns all six tests into "field of a >= field of b" — and with a guard bit per field one subtraction tests three fields:
    // ((a | G) - b) keeps the guard of a field iff a_f >= b_f (fields are >= 1 after the OR, so no borrow crosses a field).
    constexpr uint32_t G = (1u << 8) | (1u << 17) | (1u << 26);
    for (int i = lane; i < n; i += 32) {
        const int16_t *m = tmp[i];
        pk[i] = make_uint2((uint32_t)m[0] | ((uint32_t)m[1] << 9) | ((uint32_t)m[2] << 18),
                           (uint32_t)(255 - m[3]) | ((uint32_t)(255 - m[4]) << 9) | ((uint32_t)(255 - m[5]) << 18));
    }
    __syncwarp();
    int w = 0;
    const int nch2 = (n + 31) >> 5;
#pragma unroll 1
    for (int c = 0; c < nch2; c++) {
        const int i = c * 32 + lane;
        bool keep = false;
        if (i < n) {
            const uint2 a = pk[i];
            const uint32_t aL = a.x | G, aH = a.y | G;
            int hit = 0;
#pragma unroll 4
            for (int j = 0; j < n; j++) {
                const uint2 b = pk[j];
                hit |= (int)(((aL - b.x) & (aH - b.y) & G) == G && j != i);
            }
            keep = !hit;
        }
        const uint32_t bm = __ballot_sync(FULL, keep);
        if (keep) {
            const int p = w + __popc(bm & ((1u << lane) - 1));
            if (p < E_MAX) {
#pragma unroll
                for (int t = 0; t < 6; t++) ems[p][t] = tmp[i][t];
            }
        }
        w += __popc(bm);
    }
    if (w > E_MAX) { flags |= PCT_FLAG_EMS_OVERFLOW; w = E_MAX; }
    __syncwarp();
    return w;
}

}  // namespace pct
#include "pct_cand.cuh"  // the CPython-set emulation build_candidates and the EV / EP / CP / FC generators
#include "pct_draw.cuh"  // the item source and the env reset, draw_item / reset_space (included here, between the phases they sit among in the code layout)
namespace pct {

// Delta variant (default, PCT_B200_OBS_DELTA=0 disables): the caller hands back the SAME observation buffer every step, and prev[0] / prev[1]
// hold how many internal / leaf rows of it may be non-zero.  75 % of the (NB + NL + 1) x 9 observation is zero padding, so only the
// rows below max(now, prev) and the next-item row are written (and prev is updated); every other row is zero already.  The written
// values are the ones write_obs computes.  The host resets prev to {NB, NL} whenever the buffer changes.
template <typename OT, bool WARP_SCOPE = false, int PART = 0>
__device__ __noinline__ void write_obs_delta(const DParams &p, int e, const DEnvHot *hot, const DEnvCold *cold, const int16_t (*leaf)[6], int n_leaf,
                                             int tid, int nthreads) {
    OT *obs = (OT *)p.obs + (size_t)e * (size_t)((p.nb + p.nl + 1) * 9);
    int32_t *prev = p.aux[e].obs_prev;
    const int n_box = hot->h.n_box;
    const int pb = min(prev[0], p.nb), pl = min(prev[1], p.nl);
    if constexpr (WARP_SCOPE) __syncwarp(); else __syncthreads();  // every thread of the env has read prev before thread 0 replaces it below
    const int wb = PART == 2 ? 0 : max(max(n_box, pb), 1);  // row 0 always carries its valid flag (D:space.py:294-295)
    const int wl = PART == 1 ? 0 : max(n_leaf, pl);
    int s0 = hot->h.next_box[0], s1 = hot->h.next_box[1], s2 = hot->h.next_box[2];
    if (s1 < s0) { int t = s0; s0 = s1; s1 = t; }
    if (s2 < s1) { int t = s1; s1 = s2; s2 = t; }
    if (s1 < s0) { int t = s0; s0 = s1; s1 = t; }
    const OT den = (OT)hot->h.next_den;
    const bool s3 = p.setting == 3;
    const int total = (wb + wl + (PART == 2 ? 0 : 1)) * 9;
#pragma unroll 1
    for (int f = tid; f < total; f += nthreads) {
        const int r = f / 9, col = f - r * 9;
        OT v = 0;
        int row;
        if (r < wb) {
            row = r;
            if (row < n_box) {
                if (col < 6) v = (OT)hot->box[row][col];
                else if (col == 6) v = s3 ? (OT)cold->density[row] : (OT)1;
                else if (col == 8) v = 1;
            } else if (row == 0 && col == 8) v = 1;
        } else if (r < wb + wl) {
            const int k = r - wb;
            row = p.nb + k;
            if (k < n_leaf) {
                if (col < 5) v = (OT)leaf[k][col];
                else if (col == 5) v = (OT)p.H;
                else if (col == 8) v = 1;
            }
        } else {
            row = p.nb + p.nl;
            if (col == 0) v = den;
            else if (col == 3) v = (OT)s0;
            else if (col == 4) v = (OT)s1;
            else if (col == 5) v = (OT)s2;
            else if (col == 8) v = 1;
        }
        obs[row * 9 + col] = v;
    }
    if (tid == 0) {
        if (PART != 2) prev[0] = max(n_box, 1);
        if (PART != 1) prev[1] = n_leaf;
    }
}

// ======================================================================================================
// The step is a pipeline of three kernels (plus the optional synthetic-policy kernel).  A monolithic
// one-warp-per-env kernel was measured first: it was instruction-fetch bound
// (each warp streamed ~80 KB of SASS once per step, warps of an SM sat in different phases) and its duration
// was the latency of the slowest env.  Splitting by phase keeps every kernel's code small and hot in the
// instruction cache and lets the heavy phase run one THREAD per candidate leaf.
//   K1 apply      warp / env    action decode, real placement (+ load-propagating stability), EMS update,
//                               reward / done / info, auto-reset, next item
//   K2 candidates warp / env    EMSPoint in CPython-set order -> ordered candidate list in HBM
//   K3 feas_emit  block / env   thread per candidate: bounds, resting height, virtual stability;
//                               ordered compaction into the leaf slots; observation write
// ======================================================================================================
#ifdef PCT_PHASE_TIMERS
__device__ __forceinline__ long long gtime() { long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; }
#define KT_BEGIN() const long long kt0_ = gtime(); const long long kc0_ = clock64()
#define KT_END(e, k) do { if (p.mode == 1 && p.dbg) { p.dbg[(size_t)(e) * 16 + (k) * 4 + 0] = kt0_; p.dbg[(size_t)(e) * 16 + (k) * 4 + 1] = gtime(); \
        p.dbg[(size_t)(e) * 16 + (k) * 4 + 2] = clock64() - kc0_; } } while (0)
#else
#define KT_BEGIN()
#define KT_END(e, k)
#endif
#ifndef K1_MINB
#define K1_MINB 6   // sweeps: B200 (r1) 168 regs / 6 blocks per SM beat 72 regs / 14 blocks; H100 5 ties, 7 and 8 (128 regs, spills) lose 1.4 %
#endif
#ifndef K2_MINB
#define K2_MINB 1   // sweep (H100): 16 (64 regs, one resident wave, see Lay) is 0.8 % slower than no bound (74 regs, 1.14 waves)
#endif
#ifndef K3_MINB
#define K3_MINB 8   // sweep (B200, r1): 128 regs / 8 blocks per SM; the block-mode kernel is not re-measured on the H100
#endif
// ---- block scheduling order (longest-processing-time-first) --------------------------------------------------------------------------
// A launch lasts as long as its slowest block and blocks are dispatched in index order, so the envs with the most expected work (boxes placed
// drive the real stability descent and the EMS update) get the lowest slots.  No sorting pass: pct_apply_kernel files every env under its
// work key for the NEXT step (one atomicAdd into a 64-bucket histogram + one store into that bucket's list), and the apply / candidates
// kernels of the next step turn their slot into an env with a 64-entry warp scan.  Two parities: a step reads what the previous step
// wrote; the emit kernel (last of the sequence) empties the buckets just consumed and flips the parity ON THE DEVICE, so captured graphs replay
// correctly.  Layout of DParams::order (int32): [0] parity, [2 + 64 * par + j] count of bucket j = 63 - key, [ORD_LIST + (64 * par + j) * n_envs + i] envs.
constexpr int ORD_BUCKETS = 64, ORD_CNT = 2, ORD_LIST = ORD_CNT + 2 * ORD_BUCKETS;
__device__ __forceinline__ int order_lookup(const int32_t *ord, int n_envs, int slot, int lane) {
    const int par = *(volatile const int32_t *)ord & 1;
    const int32_t *cnt = ord + ORD_CNT + ORD_BUCKETS * par;
    const int a = cnt[2 * lane], b = cnt[2 * lane + 1];
    int incl = a + b;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int t = __shfl_up_sync(FULL, incl, d);
        if (lane >= d) incl += t;
    }
    const uint32_t m = __ballot_sync(FULL, slot < incl);
    if (m == 0) return slot;  // not a whole-batch history (cannot happen after pct_create's initialisation): identity
    const int f = __ffs(m) - 1;
    const int incl_f = __shfl_sync(FULL, incl, f), a_f = __shfl_sync(FULL, a, f), b_f = __shfl_sync(FULL, b, f);
    int off = slot - (incl_f - a_f - b_f), j = 2 * f;
    if (off >= a_f) { off -= a_f; j++; }
    return ord[ORD_LIST + (size_t)(ORD_BUCKETS * par + j) * n_envs + off];
}
__device__ __forceinline__ void order_file(int32_t *ord, int n_envs, int e, int n_box, int n_ems) {
    const int par = *(volatile const int32_t *)ord & 1;
    const int j = 63 - min(63, n_box + (n_ems >> 1));
    const int pos = atomicAdd(ord + ORD_CNT + ORD_BUCKETS * (par ^ 1) + j, 1);
    if (pos < n_envs) ord[ORD_LIST + (size_t)(ORD_BUCKETS * (par ^ 1) + j) * n_envs + pos] = e;
}

constexpr int K1_SM_PER_WARP = sizeof(DEnvHot) + EMS_TMP_MAX * 12 + 16 + EDGE_STAGE * 32 + POLY_STAGE * 16 + EMS_TMP_MAX * 8;  // record + EMS temp + mbarrier/lock + staged loads + packed EMS temp
static_assert(K1_SM_PER_WARP % 16 == 0, "alignment");

// SEL: the selected launch (EnvSel): slot -> the selection's env, no scheduling order
template <bool STAB, bool ALIAS = false, bool SEL = false>
__global__ void __launch_bounds__(32 * WARPS_PER_BLOCK, K1_MINB) pct_apply_kernel(const __grid_constant__ ParamsT<DParams, SEL> p) {  // ALIAS: see EdgePoolA (the default; PCT_B200_ALIAS=0 selects the snapshot kernel)
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int slot = blockIdx.x * WARPS_PER_BLOCK + warp;
    int e;
    if constexpr (SEL) {
        e = sel_env(p.sel, p.n_envs, slot);
        if (e < 0) return;
    } else {
        if (slot >= p.n_envs) return;
        e = (p.order && p.mode == 1) ? order_lookup(p.order, p.n_envs, slot, lane) : slot;  // heaviest envs first (longest-processing-time-first)
    }
    unsigned char *sm = smem_raw + (size_t)warp * K1_SM_PER_WARP;
    DEnvHot *hot = (DEnvHot *)sm;
    // per-warp layout: record | EMS temp (3 KB) | packed EMS temp (2 KB) | mbarrier + lock | staged loads | staged polygons.  The two EMS areas are
    // only used by GENEMS, after the descent: the descent's working arrays (StabScratch, 4 KB) are aliased onto them
    int16_t (*ems_tmp)[6] = (int16_t (*)[6])(sm + sizeof(DEnvHot));
    uint2 *ems_pk = (uint2 *)(sm + sizeof(DEnvHot) + EMS_TMP_MAX * 12);
    static_assert(sizeof(StabScratch) <= EMS_TMP_MAX * 12 + EMS_TMP_MAX * 8 && sizeof(DEnvHot) % 8 == 0, "the descent's scratch fits the EMS temp areas");
    StabScratch *scr = (StabScratch *)ems_tmp;
    uint64_t *mbar = (uint64_t *)(sm + sizeof(DEnvHot) + EMS_TMP_MAX * 12 + EMS_TMP_MAX * 8);
    int *lock = (int *)(mbar + 1);
    Stack4 *st_sm = (Stack4 *)(sm + sizeof(DEnvHot) + EMS_TMP_MAX * 12 + EMS_TMP_MAX * 8 + 16);
    double *poly_sm = (double *)(st_sm + EDGE_STAGE);
    DEnvHot *ghot = p.hot + e;
    DEnvCold *cold = p.cold + e;
    DHdr &h = hot->h;
    KT_BEGIN();
    if (p.ready) pdl_launch_dependents();
    if (lane == 0) *lock = 0;
    float reward = 0.f;
    int done = 0;
    pct_step_info info{};

    if (p.mode == 0) {
        // ---------------- reset (D:bin3D.py:61-67, D:space.py:290-314) ----------------
        const int64_t dp = p.keep_draw ? ghot->h.draw_pos : 0;  // box_creator.reset() does not rewind the item source
        for (int t = lane; t < (int)(sizeof(DEnvHot) / 4); t += 32) ((uint32_t *)hot)[t] = 0;
        __syncwarp();
        if (lane == 0) hot->h.draw_pos = dp;
        __syncwarp();
        reset_space(hot, p, e, lane);
    } else {
        // ---------------- stage the env record: HBM -> smem via TMA ----------------
        if (lane == 0) {
            mbar_init(mbar, 1);
            fence_proxy_async();
        }
        __syncwarp();
        if (lane == 0) {
            mbar_expect_tx(mbar, (uint32_t)sizeof(DEnvHot));
            tma_load_1d(hot, ghot, (uint32_t)sizeof(DEnvHot), mbar);
        }
        mbar_wait(mbar, 0);
        __syncwarp();
        if (STAB && h.n_edge > 0) {  // stage the load edges and support polygons too (second phase of the same mbarrier)
            const uint32_t bytes = (uint32_t)min(h.n_edge, EDGE_STAGE) * (uint32_t)sizeof(Stack4);
            const uint32_t pbytes = (uint32_t)min(h.n_poly, POLY_STAGE) * 16u;
            if (lane == 0) {
                mbar_expect_tx(mbar, bytes + pbytes);
                tma_load_1d(st_sm, cold->e_st, bytes, mbar);
                if (pbytes) tma_load_1d(poly_sm, cold->poly, pbytes, mbar);
            }
            mbar_wait(mbar, 1);
            __syncwarp();
        }

        const int nb0 = h.next_box[0], nb1 = h.next_box[1], nb2 = h.next_box[2];
        const int n_box0 = h.n_box, n_leaf0 = h.n_leaf, flags0 = h.flags;
        const double next_den0 = h.next_den;
        __syncwarp();
        // ---- LeafNode2Action (D:bin3D.py:139-149) ----
        int lx = 0, ly = 0, x = nb0, y = nb1, z = nb2;
        bool bad = false;
        {
            double a0 = 0, a1 = 0, a3 = 0, a4 = 0;
            bool zero = true;
            if (p.leaf_idx) {
                const int k = p.leaf_idx[e];
                if (k >= 0 && k < n_leaf0) {
                    zero = false;
                    const int16_t *l = cold->leaf[k];
                    a0 = l[0]; a1 = l[1]; a3 = l[3]; a4 = l[4];
                }
            } else {
                double a[6], s = 0;
#pragma unroll
                for (int t = 0; t < 6; t++) {
                    a[t] = p.action_f64 ? ((const double *)p.actions)[(size_t)e * 9 + t] : (double)((const float *)p.actions)[(size_t)e * 9 + t];
                    s += a[t];
                }
                zero = (s == 0);
                a0 = a[0]; a1 = a[1]; a3 = a[3]; a4 = a[4];
            }
            if (!zero) {
                x = (int)(a3 - a0);
                y = (int)(a4 - a1);
                // z = what is left of next_box after list.remove(x), list.remove(y)
                int r0 = nb0, r1 = nb1, r2 = nb2, n = 3;
                if (r0 == x) { r0 = r1; r1 = r2; n = 2; }
                else if (r1 == x) { r1 = r2; n = 2; }
                else if (r2 == x) n = 2;
                else bad = true;
                if (n == 2) {
                    if (r0 == y) r0 = r1;
                    else if (r1 != y) bad = true;
                }
                z = r0;
                lx = (int)a0;
                ly = (int)a1;
            }
        }
        // ---- Space.drop_box (D:space.py:347-389) ----
        const int maxax = max(p.W, p.L);
        bool ok = !bad && lx >= 0 && ly >= 0 && lx < maxax && ly < maxax && x > 0 && y > 0;
        int max_h = 0;
        if (STAB && lane == 0) {  // CSR slot / incoming-list head of the box about to be placed
            hot->e_off[n_box0] = (uint16_t)h.n_edge;
            hot->poly_off[n_box0] = (uint16_t)h.n_poly;
            if (n_box0 < NB_MAX) hot->first_in[n_box0] = EDGE_NIL;  // box NB_MAX + 1 is never committed and nothing rests on a box during its own descent
        }
        __syncwarp();
        if (ok) {
            // resting height: warp max-reduce over the placed boxes whose footprint overlaps
            max_h = __reduce_max_sync(FULL, rest_height(hot->box, lane, n_box0, 32, lx, ly, lx + x, ly + y));
            if (lx + x > p.W || ly + y > p.L) ok = false;
            else if (max_h + z > p.H) ok = false;
            else if (STAB && max_h != 0) {
                int res = 0;
                if (lane == 0) {
                    int fl = 0;
                    GeomD g{hot->box, n_box0, p.setting == 3 ? cold->density : nullptr};
                    NodeD root{lx, ly, max_h, x, y, z, (double)(x * y * z) * next_den0};
                    if constexpr (ALIAS) {  // the reference's object semantics of the load entries (DESIGN.md section 3 (b))
                        EdgePoolA pool;
                        static_cast<EdgePool &>(pool) = EdgePool{hot->e_lower, hot->e_next, hot->e_off, hot->first_in, hot->last_in, cold->e_st, st_sm, h.n_edge,
                                                                 hot->poly_off, &cold->poly[0][0], poly_sm, h.n_poly};
                        DEnvAux *ax = p.aux + e;
                        pool.box_st = ax->box_st; pool.e_upper = ax->e_upper; pool.e_alias = ax->e_alias;
                        res = stability_check<true, GeomD, true>(g, root, pool, &cold->big, lock, n_box0, fl, nullptr, scr);
                        if (!res) alias_sync_loads(pool);
                        h.n_edge = pool.n;
                        h.n_poly = pool.n_poly;
                    } else {
                    EdgePool pool{hot->e_lower, hot->e_next, hot->e_off, hot->first_in, hot->last_in, cold->e_st, st_sm, h.n_edge,
                                  hot->poly_off, &cold->poly[0][0], poly_sm, h.n_poly};
                    res = stability_check<true, GeomD>(g, root, pool, &cold->big, lock, n_box0, fl, nullptr, scr);
                    h.n_edge = pool.n;
                    h.n_poly = pool.n_poly;
                    }
                    h.flags |= fl;
                }
                __syncwarp();
                ok = __shfl_sync(FULL, res, 0) != 0;
            }
            if (ok && n_box0 >= p.nb) {
                ok = false;
                if (lane == 0) h.flags |= PCT_FLAG_BOX_OVERFLOW;
            }
        }
        if (lane == 0 && !bad && (lx < 0 || ly < 0 || lx >= maxax || ly >= maxax)) {
            // np.max(plain[lx:lx + x, ly:ly + y]) raises on an empty slice of the max(W, L)-square plain (D:space.py:354-355).  Unlike the
            // oracle's guard, no x <= 0 / y <= 0 term: when !bad, x and y are sides of the item (>= 1), so only the start can empty the slice
            auto py = [maxax](int i) { return i < 0 ? max(i + maxax, 0) : min(i, maxax); };  // Python's clamp of a slice bound
            bad = py(lx) >= py(lx + x) || py(ly) >= py(ly + y);
        }
        if (bad && lane == 0) h.flags |= PCT_FLAG_BAD_ACTION;
        __syncwarp();
        const double binvol = (double)(p.W * p.L * p.H);
        if (ok) {
            int16_t *b = hot->box[n_box0];
            if (lane == 0) {
                b[0] = (int16_t)lx; b[1] = (int16_t)ly; b[2] = (int16_t)max_h;
                b[3] = (int16_t)(lx + x); b[4] = (int16_t)(ly + y); b[5] = (int16_t)(max_h + z);
                if (p.setting == 3) cold->density[n_box0] = next_den0;
                h.n_box = n_box0 + 1;
                h.vol_sum += x * y * z;
                if (STAB) { hot->e_off[n_box0 + 1] = (uint16_t)h.n_edge; hot->poly_off[n_box0 + 1] = (uint16_t)h.n_poly; }
            }
            const int n_ems0 = h.n_ems;
            __syncwarp();
            int fl = 0;
            // GENEMS only runs for LNES == 'EMS' (D:bin3D.py:172-175); 'EVM' is EventPoint over the list it maintains
            const int n_ems = (p.lnes == 0 || p.lnes == 5) ? genems_warp(hot->ems, n_ems0, ems_tmp, ems_pk, b, p.low_bound, lane, fl) : n_ems0;
            const double rw = (double)(nb0 * nb1 * nb2) / binvol * 10;  // D:bin3D.py:180-183
            reward = (float)rw;
            info.counter = n_box0 + 1;
            info.flags = flags0 | fl;
            if (lane == 0) {
                h.n_ems = n_ems;
                h.flags |= fl;
                h.ep_len++;
                h.ep_reward += rw;
                draw_item(p, e, h);
            }
            __syncwarp();
        } else {
            // terminal step (D:bin3D.py:160-165) followed by the worker's auto-reset (shmem_vec_env.py:141-142)
            done = 1;
            info.counter = n_box0;
            info.flags = h.flags;
            info.ratio = (float)((double)h.vol_sum / binvol);
            info.ep_reward = (float)h.ep_reward;
            info.ep_len = h.ep_len + 1;
            __syncwarp();
            if (!p.no_auto_reset) reset_space(hot, p, e, lane);
        }
    }
    fence_proxy_async();
    __syncwarp();
    if (lane == 0) {
        if (p.reward) p.reward[e] = reward;
        if (p.done) p.done[e] = (uint8_t)done;
        if (p.info) p.info[e] = info;
        if (p.order) order_file(p.order, p.n_envs, e, h.n_box, h.n_ems);  // this env's slot in the next step's launches
        // record back to HBM: smem -> global via TMA bulk store
        tma_store_1d(ghot, hot, (uint32_t)sizeof(DEnvHot));
        if (STAB && p.mode == 1 && h.n_edge > 0) tma_store_1d(cold->e_st, st_sm, (uint32_t)min(h.n_edge, EDGE_STAGE) * (uint32_t)sizeof(Stack4));
        if (STAB && p.mode == 1 && h.n_poly > 0) tma_store_1d(cold->poly, poly_sm, (uint32_t)min(h.n_poly, POLY_STAGE) * 16u);
        if (p.ready) {  // overlapped mode: the record must be globally visible before the hand-over flag
            tma_store_commit_wait_all();
            fence_proxy_async_all();
            env_publish(p.ready + e, p.epoch);
        } else
            tma_store_commit_wait();
        KT_END(p.env_id_base + e - p.env_id_base0, 0);
    }
}

// ---- K2: candidate leaves -----------------------------------------------------------------------------------
// __grid_constant__ (K1, K2, emit): the __noinline__ phases take `const DParams &`; without it every thread first copies the 320 B parameter
// block into its local-memory frame, so that the reference has an address, and reads the fields back from there.
// EVM: the LNES='EVM' instantiation (gen_event_point_m), kept apart so that the other schemes' instantiations keep their code and registers
template <typename SlotT, bool BIGSM, bool SEL = false, bool EVM = false>
__global__ void __launch_bounds__(32 * WARPS_PER_BLOCK, K2_MINB) pct_candidates_kernel(const __grid_constant__ ParamsT<DParams, SEL> p) {
    typedef Lay<SlotT, BIGSM> LY;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int slot = blockIdx.x * WARPS_PER_BLOCK + warp;
    int e;
    if constexpr (SEL) {
        e = sel_env(p.sel, p.n_envs, slot);
        if (e < 0) return;
    } else {
        if (slot >= p.n_envs) return;
        e = (p.order && p.mode == 1) ? order_lookup(p.order, p.n_envs, slot, lane) : slot;
    }
    unsigned char *sm = smem_raw + (size_t)warp * LY::PER_WARP;
    DEnvHot *hot = (DEnvHot *)(sm + LY::HOT);
    SlotT *tabA = (SlotT *)(sm + LY::TAB_A_OFF), *tabB = (SlotT *)(sm + LY::TAB_B_OFF);
    uint64_t *mbar = (uint64_t *)(sm + LY::MISC);
    RotTab *rt = (RotTab *)(sm + LY::MISC + 16);
    SetStage *stg = (SetStage *)(sm + LY::MISC + 48);
    static_assert(sizeof(RotTab) <= 32 && sizeof(SetStage) == 384, "RotTab / SetStage slots");
    DEnvHot *ghot = p.hot + e;
    DEnvCold *cold = p.cold + e;
    KT_BEGIN();
    int sync_fl = 0;
    if (p.ready) {  // overlapped mode: wait for the apply kernel's hand-over of THIS env
        pdl_launch_dependents();
        if (lane == 0 && !env_wait(p.ready + e, p.epoch)) sync_fl = PCT_FLAG_SYNC_TIMEOUT;
        __syncwarp();
    }
    if (lane == 0) {
        mbar_init(mbar, 1);
        fence_proxy_async_all();
    }
    __syncwarp();
    if (lane == 0) {  // header + boxes + EMS list only
        mbar_expect_tx(mbar, (uint32_t)HOT_PREFIX);
        tma_load_1d(hot, ghot, (uint32_t)HOT_PREFIX, mbar);
    }
    mbar_wait(mbar, 0);
    __syncwarp();
    const DHdr &h = hot->h;
    const int nb3[3] = {h.next_box[0], h.next_box[1], h.next_box[2]};
    const int R = p.setting == 2 ? 6 : 2;
    if (lane == 0) make_rot_tab(nb3, R, *rt);
    __syncwarp();
    SlotT *cand = nullptr;
    int fl = 0, n_cand = 0;
    SlotT *out = (SlotT *)cold->cand;
    constexpr int KB = sizeof(SlotT) == 2 ? 4 : 8;
    if constexpr (EVM) {
        const CandList<SlotT> cl = gen_event_point_m<SlotT>(hot, rt, R, p.W, p.L, p.H, tabA, tabB,
                                                            BIGSM ? tabA : (SlotT *)cold->tab_big, cold->raw, out, lane);
        cand = cl.keys; n_cand = cl.n; fl = cl.flags;
    } else if (p.lnes == 0) {
        const CandList<SlotT> cl = build_candidates<SlotT>(hot->ems, h.n_ems, rt, R, tabA, tabB, BIGSM ? tabA : (SlotT *)cold->tab_big, stg, lane);
        cand = cl.keys; n_cand = cl.n; fl = cl.flags;
    } else {
        uint32_t *raw = cold->raw;
        RawList rl;
        if (p.lnes == 4) rl = gen_full_coord<KB>(hot->box, h.n_box, rt, R, p.W, p.L, p.H, raw, lane);
        else if (p.lnes == 1) rl = RawList{gen_event_point<KB>(rt, R, p.W, p.L, raw, lane), 0};
        else rl = gen_level_points<KB>(hot->box, h.n_box, rt, R, p.W, p.L, p.H, p.lnes == 2, raw, lane);
        fl = rl.flags;
        if (rl.n == -2) {  // empty bin under EP / CP: the reference returns a 2-element LIST (D:space.py:700-701)
            if (lane < 2) out[lane] = (SlotT)key_pack<KB>(0, 0, 0, rt->canon[lane]);
            n_cand = 2;
            cand = out;
        } else {
            const CandList<SlotT> cl = build_candidates<SlotT>(hot->ems, h.n_ems, rt, R, tabA, tabB, BIGSM ? tabA : (SlotT *)cold->tab_big, stg, lane, raw, rl.n);
            cand = cl.keys; n_cand = cl.n; fl |= cl.flags;
        }
    }
    if (cand != out)
        for (int t = lane; t < n_cand; t += 32) out[t] = cand[t];
    fl |= sync_fl;
    __syncwarp();
    if (p.shuffle) {  // scratch: cold->raw + cold->tab_big (contiguous, 16 KB, free once the list is in `out`): keys at 0, permuted list at 10 KB
        static_assert(offsetof(DEnvCold, tab_big) == offsetof(DEnvCold, raw) + sizeof(uint32_t) * RAW_MAX, "raw and tab_big are contiguous");
        static_assert(CAND_MAX * 8 <= 10240 && 10240 + CAND_MAX * 4 <= (RAW_MAX + TAB_A) * 4, "shuffle scratch fits");
        shuffle_candidates<SlotT>(out, n_cand, (uint64_t *)cold->raw, (SlotT *)((char *)cold->raw + 10240), p.seed, (uint64_t)(p.env_id_base + e),
                                  (uint64_t)h.draw_pos, lane);
        cand = out;
    }
    if (p.walk.walkq) {
        // ---- classify (round 2; see "K3 (round 2)" below): drop_box_virtual (D:space.py:393-433) + check_box (:436-454), integer part ----
        constexpr bool STAB = !BIGSM;
        const int n_box = h.n_box, nl = p.nl;
        const uint32_t lt = (1u << lane) - 1;
        int pos = 0, nf = 0, n_walk = 0;
#pragma unroll 1
        while (pos < n_cand && nf < nl) {
            const int c = pos + lane;
            bool feas = false, pend = false;
            int mh = 0, k = 0, xs = 0, ys = 0, zs = 0, rot = 0, sx = 0, sy = 0, sz = 0;
            uint32_t pack = 0;
            if (c < n_cand) {
                key_unpack<KB>((uint32_t)cand[c], xs, ys, zs, rot);
                sx = rt->d[rot][0]; sy = rt->d[rot][1]; sz = rt->d[rot][2];
                bool far_out = false;
                if (STAB) mh = rest_height_supports(hot->box, n_box, xs, ys, xs + sx, ys + sy, k, pack, far_out);
                else mh = rest_height(hot->box, 0, n_box, 1, xs, ys, xs + sx, ys + sy);
                if (xs + sx > p.W || ys + sy > p.L) feas = false;
                else if (mh + sz > p.H) feas = false;
                else if (!STAB || mh == 0) feas = true;
                else pend = !far_out;  // far_out: the centre is outside the supports' bounding box -> the root test fails (rest_height_supports)
            }
            const uint32_t fm = __ballot_sync(FULL, feas), pm = __ballot_sync(FULL, pend);
            if (lane == 0) cold->fbits[pos >> 5] = fm;
            nf += __popc(fm);
            n_walk += __popc(pm);
            if (pm) {
                int qb = 0;
                if (lane == 0) qb = atomicAdd(p.walk.walk_ctr, __popc(pm));
                qb = __shfl_sync(FULL, qb, 0);
                if (pend) {
                    WalkItem it;
                    it.env = (uint32_t)e; it.pack = pack; it.c = (uint16_t)c;
                    it.xs = (uint8_t)xs; it.ys = (uint8_t)ys; it.mh = (uint8_t)mh; it.sx = (uint8_t)sx; it.sy = (uint8_t)sy; it.sz = (uint8_t)sz;
                    it.k = (uint8_t)min(k, 255); it.pad_ = 0;
                    p.walk.walkq[qb + __popc(pm & lt)] = it;
                }
            }
            pos += 32;
        }
        if (lane == 0) { cold->n_fw = pos >> 5; cold->n_pending = n_walk; }
        // cur_observation, part 1 (D:bin3D.py:70-93): internal-node rows + item row are final since the apply kernel
        if (p.obs) {
            const bool delta = (p.opt & PCT_OPT_DELTA) != 0;
            if (p.obs_f64) { if (delta) write_obs_delta<double, true, 1>(p, e, hot, cold, nullptr, 0, lane, 32); else write_obs<double, 1>(p, e, hot, cold, nullptr, 0, lane, 32); }
            else { if (delta) write_obs_delta<float, true, 1>(p, e, hot, cold, nullptr, 0, lane, 32); else write_obs<float, 1>(p, e, hot, cold, nullptr, 0, lane, 32); }
        }
    }
    if (lane == 0) {
        ghot->h.n_cand = n_cand;
        if (fl) ghot->h.flags = h.flags | fl;
        if (p.ready) env_publish(p.ready + p.n_envs + e, p.epoch);
        KT_END(p.env_id_base + e - p.env_id_base0, 1);
    }
}

// ---- K3: feasibility (thread per candidate) + leaf compaction + observation ------------------------------------
#ifndef FEAS_WARPS_N
#define FEAS_WARPS_N 2
#endif
constexpr int FEAS_WARPS = FEAS_WARPS_N;
constexpr int FEAS_THREADS = 32 * FEAS_WARPS;
// the block's shared memory: the staged env, the leaves in order, the rotation table of the item, the per-warp ballots of the compaction
struct FeasSmD {
    StageD s;
    int16_t leaf[NL_MAX][6];
    RotTab rt;
    uint32_t wb[FEAS_WARPS];
};

template <typename OT, bool STAB, typename SlotT, bool DELTA = false, bool SEL = false>
__global__ void __launch_bounds__(FEAS_THREADS, K3_MINB) pct_feas_emit_kernel(const ParamsT<DParams, SEL> p) {
    constexpr int BITS = sizeof(SlotT) == 2 ? 4 : 8;
    __shared__ __align__(16) FeasSmD sm;
    const int tid = threadIdx.x, lane = tid & 31;
    int e = blockIdx.x;  // (round 1's heaviest-first permutation of this kernel went with the sorting pass; the legacy mode runs in env order)
    if constexpr (SEL) {
        e = sel_env(p.sel, p.n_envs, e);
        if (e < 0) return;  // the whole block
    }
    DEnvHot *hot = &sm.s.hot;
    DEnvHot *ghot = p.hot + e;
    DEnvCold *cold = p.cold + e;
    KT_BEGIN();
    StagedD sd = stage_env_d<STAB>(sm.s, p, e, true);
    const DHdr &h = hot->h;
    const int nb3[3] = {h.next_box[0], h.next_box[1], h.next_box[2]};
    if (tid == 0) make_rot_tab(nb3, p.setting == 2 ? 6 : 2, sm.rt);
    __syncthreads();
    const int n_cand = h.n_cand;
    const double den = h.next_den;
    const SlotT *cand = (const SlotT *)cold->cand;
    const RotTab *rt = &sm.rt;
    int fl = 0;
    // ---------------- get_possible_position (D:bin3D.py:100-136): first `nl` feasible candidates in order ----------------
    const int n_leaf = first_feasible<FEAS_WARPS>(n_cand, p.nl, sm.leaf, sm.wb, [&](int c, int16_t *row) {
        int xs, ys, zs, rot, mh;
        key_unpack<BITS>(cand[c], xs, ys, zs, rot);
        const int sx = rt->d[rot][0], sy = rt->d[rot][1], sz = rt->d[rot][2];
#ifdef PCT_PHASE_TIMERS
        const long long c0 = clock64();
        int fl2 = 0;
        long long prof[6];
        const bool feas = place_virtual_d<STAB>(p, sd.g, sd.pool, &cold->big, &sm.s.lock, sx, sy, sz, xs, ys, den, mh, fl2, prof) != 0;
        const long long dc = clock64() - c0;
        fl |= fl2 & 0xFFFF;
        // recorded only for placements that ran the stability check (it counts its visits from bit 16 of fl2); dc also covers the
        // resting height and the bounds tests in front of it
        if (p.mode == 1 && p.dbg && (fl2 >> 16) != 0) {
            unsigned long long packed = ((unsigned long long)dc << 24) | ((unsigned long long)((fl2 >> 16) & 0xFF) << 8) | (unsigned long long)((fl2 >> 24) & 0xFF);
            long long *slot = &p.dbg[(size_t)(p.env_id_base + e - p.env_id_base0) * 16];
            if (atomicMax((unsigned long long *)&slot[12], packed) < packed)
                { slot[3] = prof[0]; slot[7] = prof[1]; slot[11] = prof[2]; slot[13] = prof[3]; slot[14] = prof[4]; }
        }
#else
        const bool feas = place_virtual_d<STAB>(p, sd.g, sd.pool, &cold->big, &sm.s.lock, sx, sy, sz, xs, ys, den, mh, fl) != 0;
#endif
        row[0] = (int16_t)xs; row[1] = (int16_t)ys; row[2] = (int16_t)zs;
        row[3] = (int16_t)(xs + sx); row[4] = (int16_t)(ys + sy); row[5] = (int16_t)(zs + sz);
        return feas;
    });
    fl = __reduce_or_sync(FULL, fl);
    if (fl && lane == 0) atomicOr(&ghot->h.flags, fl);
    __syncthreads();
    // persist the emitted leaves for the leaf-index action path; header / info
    for (int t = tid; t < n_leaf * 6; t += FEAS_THREADS) ((int16_t *)cold->leaf)[t] = ((int16_t *)sm.leaf)[t];
    if (tid == 0) {
        ghot->h.n_leaf = n_leaf;
        if (p.info) {
            p.info[e].n_leaf = n_leaf;
            p.info[e].n_cand = n_cand;
            p.info[e].n_ems = h.n_ems;
            p.info[e].flags |= h.flags;
        }
    }
    // ---------------- cur_observation (D:bin3D.py:70-93) ----------------
    if constexpr (DELTA) write_obs_delta<OT>(p, e, hot, cold, sm.leaf, n_leaf, tid, FEAS_THREADS);
    else write_obs<OT>(p, e, hot, cold, sm.leaf, n_leaf, tid, FEAS_THREADS);
    if (tid == 0) KT_END(p.env_id_base + e - p.env_id_base0, 2);
}

// ---- K3 (round 2): pooled stability walks + emit ---------------------------------------------------------------------
// Profiles of the kernel above (round 1) and of a warp-per-env variant:
// the launch lasts 2x the SMs' mean active time — it ends when the env with the most and deepest stability walks ends (a serial chain
// inside one block) —, most of the warp instructions sit in the walk at 2-5 active lanes, every candidate scans the boxes twice, and capping
// registers for occupancy only trades stalls for spills.  Round 2 cuts the work by KIND instead of by env:
//   classify  (end of K2, warp per env, integer only) bounds + ONE pass over the boxes for resting height, supports and the exact
//             quick reject (rest_height_supports) -> infeasible / feasible / needs a stability walk; feasibility bits per 32-candidate
//             chunk; the walks of ALL envs go into one global pool;
//   walk      two kernels over the pool, 32 walks per warp from whichever envs (a heavy env's walks spread over many warps and SMs):
//             pct_walk_light_kernel runs every walk's LIGHT PREFIX (stab_light: visits of nodes with <= 1 support; 81 % of the walks are
//             nothing else) and hands the rest — walks standing in front of a node with >= 2 supports, with (node, stack) — to
//             pct_walk_kernel, whose lanes therefore all START with a heavy visit (dense) and finish through stab_virtual;
//   emit      pct_emit_kernel (warp per env): the first `nl` set feasibility bits in candidate order -> leaf slots, observation.
// get_possible_position stops at `nl` feasible candidates (D:bin3D.py:117-136); here classification stops once `nl` candidates are KNOWN
// feasible and the emit kernel takes the first `nl` set bits: the same ordered prefix (walks past the cut are wasted work, not wrong).
#ifndef WALK_MINB
#define WALK_MINB 6   // sweep (H100): 6 (165 regs, no spill) beats 8 (128 regs, the B200 choice) by 1.7 % and 10 (96 regs) by 5 %
#endif
#ifndef LIGHT_MINB
#define LIGHT_MINB 6  // sweep (H100): 4 and 8 both slower
#endif
// the discrete domain's side of the walk stage (pct_walks.cuh): hot record for the geometry, cold record for the walk's verdict and scratch
struct DWalkView {
    GeomD g;
    EdgePool pool;
    NodeD root;
    DEnvCold *cold;
    const DEnvHot *hot;
    __device__ __forceinline__ uint32_t *fbits() const { return cold->fbits; }
    __device__ __forceinline__ int32_t *flags() const { return const_cast<int32_t *>(&hot->h.flags); }
    __device__ __forceinline__ int32_t *n_pending() const { return &cold->n_pending; }
    __device__ __forceinline__ BigScratch *big() const { return &cold->big; }
    __device__ __forceinline__ int32_t *lock() const { return &cold->lock; }
};
struct DWalk {
    typedef DParams Params;
    typedef WalkItem Item;
    typedef GeomD Geom;
    static __device__ __forceinline__ DWalkView view(const DParams &p, const WalkItem &it, bool has) {
        const DEnvHot *hot = p.hot + it.env;
        DEnvCold *cold = p.cold + it.env;
        const DHdr &h = hot->h;
        const int sx = it.sx, sy = it.sy, sz = it.sz;
        return DWalkView{GeomD{hot->box, has ? h.n_box : 0, p.setting == 3 ? cold->density : nullptr},
                               EdgePool{const_cast<uint8_t *>(hot->e_lower), const_cast<uint8_t *>(hot->e_next), const_cast<uint16_t *>(hot->e_off),
                                        const_cast<uint8_t *>(hot->first_in), const_cast<uint8_t *>(hot->last_in), cold->e_st, cold->e_st, has ? h.n_edge : 0,
                                        const_cast<uint16_t *>(hot->poly_off), &cold->poly[0][0], &cold->poly[0][0], has ? h.n_poly : 0},
                               NodeD{(int)it.xs, (int)it.ys, (int)it.mh, sx, sy, sz, (double)(sx * sy * sz) * (has ? h.next_den : 1.0)},
                         cold, hot};
    }
    static __device__ __forceinline__ bool tall(const DParams &p, const WalkItem &it) { return (int)it.mh * 5 >= p.H * 3; }
};

__global__ void __launch_bounds__(32 * LIGHT_WARPS, LIGHT_MINB) pct_walk_light_kernel(const DParams p) { walk_light<DWalk>(p); }
__global__ void __launch_bounds__(32 * WALK_WARPS, WALK_MINB) pct_walk_kernel(const DParams p) { PCT_WALK_CONT_BODY(DWalk, p) }
__global__ void __launch_bounds__(32 * WALK_WARPS, WALK_MINB) pct_walk_fork_kernel(const DParams p) { walk_fork<DWalk>(p); }

#ifndef EMIT_WARPS_N
#define EMIT_WARPS_N 4
#endif
constexpr int EMIT_WARPS = EMIT_WARPS_N;
constexpr int EMIT_STAGE = sizeof(DHdr) + NB_MAX * 12;  // header + placed boxes: all the observation needs from the hot record
constexpr int EMIT_SM_PER_WARP = EMIT_STAGE + NL_MAX * 12 + 48;
static_assert(EMIT_STAGE % 16 == 0 && EMIT_SM_PER_WARP % 16 == 0, "TMA bulk copies move multiples of 16 bytes");

template <typename OT, typename SlotT, bool DELTA, bool SEL = false>
__global__ void __launch_bounds__(32 * EMIT_WARPS) pct_emit_kernel(const __grid_constant__ ParamsT<DParams, SEL> p) {
    constexpr int BITS = sizeof(SlotT) == 2 ? 4 : 8;
    __shared__ __align__(16) unsigned char smem[EMIT_WARPS * EMIT_SM_PER_WARP];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int e = blockIdx.x * EMIT_WARPS + warp;
    // last kernel of the launch sequence that touches the walk pools (both walk kernels have completed: plain stream order): empty them for the next step
    if (blockIdx.x == 0 && threadIdx.x == 0 && p.walk.walk_ctr) reset_walk_pools(p.walk);
    if (blockIdx.x == 0 && p.order) {
        // ... and the last one of the step: the apply and candidates kernels have consumed this parity's buckets (both completed before the walk kernels
        // started) and the apply kernel has filled the other parity's; empty the consumed ones and flip
        const int par = *(volatile const int32_t *)p.order & 1;
        if (threadIdx.x < ORD_BUCKETS) p.order[ORD_CNT + ORD_BUCKETS * par + threadIdx.x] = 0;
        __syncthreads();
        if (threadIdx.x == 0) { __threadfence(); *(volatile int32_t *)p.order = par ^ 1; }
    }
    if constexpr (SEL) {  // after the pool reset above: block 0 exists whenever the launch does
        e = sel_env(p.sel, p.n_envs, e);
        if (e < 0) return;
    }
    if (e >= p.n_envs) return;
    unsigned char *sm = smem + warp * EMIT_SM_PER_WARP;
    DEnvHot *hot = (DEnvHot *)sm;  // only the header and the boxes are staged
    int16_t (*leaf)[6] = (int16_t (*)[6])(sm + EMIT_STAGE);
    uint64_t *mbar = (uint64_t *)(sm + EMIT_STAGE + NL_MAX * 12);
    RotTab *rt = (RotTab *)(sm + EMIT_STAGE + NL_MAX * 12 + 16);
    DEnvHot *ghot = p.hot + e;
    DEnvCold *cold = p.cold + e;
    const uint32_t lt = (1u << lane) - 1;
    if (lane == 0) {
        mbar_init(mbar, 1);
        fence_proxy_async();
        wait_walks(&cold->n_pending, ghot);
        fence_proxy_async_all();
    }
    __syncwarp();
    if (lane == 0) {
        mbar_expect_tx(mbar, (uint32_t)EMIT_STAGE);
        tma_load_1d(hot, ghot, (uint32_t)EMIT_STAGE, mbar);
    }
    mbar_wait(mbar, 0);
    __syncwarp();
    const DHdr &h = hot->h;
    const int nb3[3] = {h.next_box[0], h.next_box[1], h.next_box[2]};
    if (lane == 0) make_rot_tab(nb3, p.setting == 2 ? 6 : 2, *rt);
    __syncwarp();
    const int nl = p.nl, nw = cold->n_fw;
    const SlotT *cand = (const SlotT *)cold->cand;
    // ---------------- leaves = the first `nl` feasible candidates in order ----------------
    int base = 0;
#pragma unroll 1
    for (int w = 0; w < nw && base < nl; w++) {
        const uint32_t bits = cold->fbits[w];
        if ((bits >> lane) & 1u) {
            const int kk = base + __popc(bits & lt);
            if (kk < nl) {
                int xs, ys, zs, rot;
                key_unpack<BITS>(cand[w * 32 + lane], xs, ys, zs, rot);
                leaf[kk][0] = (int16_t)xs; leaf[kk][1] = (int16_t)ys; leaf[kk][2] = (int16_t)zs;
                leaf[kk][3] = (int16_t)(xs + rt->d[rot][0]); leaf[kk][4] = (int16_t)(ys + rt->d[rot][1]); leaf[kk][5] = (int16_t)(zs + rt->d[rot][2]);
            }
        }
        base += __popc(bits);
    }
    const int n_leaf = min(base, nl);
    __syncwarp();
    // persist the emitted leaves for the leaf-index action path; header / info
    for (int t = lane; t < n_leaf * 6; t += 32) ((int16_t *)cold->leaf)[t] = ((int16_t *)leaf)[t];
    if (lane == 0) {
        ghot->h.n_leaf = n_leaf;
        if (p.info) {
            p.info[e].n_leaf = n_leaf;
            p.info[e].n_cand = h.n_cand;
            p.info[e].n_ems = h.n_ems;
            p.info[e].flags |= h.flags;
        }
    }
    // ---------------- cur_observation (D:bin3D.py:70-93) ----------------
    if constexpr (DELTA) write_obs_delta<OT, true, 2>(p, e, hot, cold, leaf, n_leaf, lane, 32);  // leaf rows: the rest was written by the candidates kernel
    else write_obs<OT, 2>(p, e, hot, cold, leaf, n_leaf, lane, 32);
}

// uniform-random valid-leaf policy (SURVEY.md §8(d)): reads only the record headers
__global__ void pct_policy_random_kernel(const DEnvHot *hot, int n_envs, int64_t env_id_base, uint64_t seed, int64_t t, const int64_t *t_dev,
                                         int32_t *leaf_idx) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_envs) return;
    if (t_dev) t = *t_dev;
    const int n = hot[e].h.n_leaf;
    leaf_idx[e] = n > 0 ? (int32_t)(rnd_u64(seed, (uint64_t)(env_id_base + e), (uint64_t)t) % (uint64_t)n) : 0;
}

__global__ void pct_fill_prev_kernel(DEnvAux *aux, int n, int nb, int nl) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { aux[i].obs_prev[0] = nb; aux[i].obs_prev[1] = nl; }
}
void launch_fill_prev(DEnvAux *aux, int n_envs, int nb, int nl, cudaStream_t st) {
    pct_fill_prev_kernel<<<(n_envs + 255) / 256, 256, 0, st>>>(aux, n_envs, nb, nl);
}

// ---- launchers ---------------------------------------------------------------------------------------------
template <typename K>
static cudaError_t set_smem(K kernel, size_t smem) {
    return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
}

// apply = false: the pipeline without K1 (pct_set_items / pct_reset_envs: their kernel in pct_items.cu has already run); the caller passes ready = order = nullptr.
// SEL: the selected launch of p.sel (ready = order = nullptr too): the SEL instantiations over p.sel.slots(n_envs) slots, the walk kernels as they are
template <typename OT, bool STAB, typename SlotT, bool SEL>
static cudaError_t launch_t(const ParamsT<DParams, SEL> &p_in, cudaStream_t st, cudaEvent_t *prof, bool apply = true) {
    constexpr bool BIGSM = !STAB;
    static bool attr_set = false;
    const size_t smem1 = (size_t)K1_SM_PER_WARP * WARPS_PER_BLOCK;
    const size_t smem2 = (size_t)Lay<SlotT, BIGSM>::PER_WARP * WARPS_PER_BLOCK;
    ParamsT<DParams, SEL> p = p_in;
    const bool k3_old = (p.opt & PCT_OPT_K3_BLOCK) != 0 || !p.walk.walkq;  // PCT_B200_K3=block: round 1's block-per-env / thread-per-candidate kernel (A/B measurements)
    if (k3_old) p.walk.walkq = nullptr;  // K2 then skips the classification
    if (!attr_set) {
        cudaError_t err = set_smem(pct_apply_kernel<STAB, false, SEL>, smem1);
        if (err == cudaSuccess && STAB) err = set_smem(pct_apply_kernel<STAB, STAB, SEL>, smem1);  // the ALIAS variant (stability settings only)
        if (err == cudaSuccess) err = set_smem(pct_candidates_kernel<SlotT, BIGSM, SEL>, smem2);
        if (err == cudaSuccess) err = set_smem(pct_candidates_kernel<SlotT, BIGSM, SEL, true>, smem2);
        if (err != cudaSuccess) return err;
        attr_set = true;
    }
    int slots = p.n_envs;
    if constexpr (SEL) slots = p.sel.slots(p.n_envs);
    const int blocks = (slots + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK;
    auto *const k2 = p.lnes == 5 ? pct_candidates_kernel<SlotT, BIGSM, SEL, true> : pct_candidates_kernel<SlotT, BIGSM, SEL>;
    if (prof) cudaEventRecord(prof[0], st);
    if (apply) {
        if (STAB && (p.opt & PCT_OPT_ALIAS)) pct_apply_kernel<STAB, STAB, SEL><<<blocks, 32 * WARPS_PER_BLOCK, smem1, st>>>(p);
        else pct_apply_kernel<STAB, false, SEL><<<blocks, 32 * WARPS_PER_BLOCK, smem1, st>>>(p);
    }
    if (prof) cudaEventRecord(prof[1], st);
    cudaError_t err = cudaSuccess;
    if (!SEL && p.ready) {
        // overlapped mode (programmatic dependent launch): the candidates blocks become resident while the apply kernel's tail is
        // still running and pick their env up through the per-env hand-over flags
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[0].val.programmaticStreamSerializationAllowed = 1;
        cudaLaunchConfig_t cfg{};
        cfg.stream = st; cfg.attrs = at; cfg.numAttrs = 1;
        cfg.gridDim = dim3(blocks); cfg.blockDim = dim3(32 * WARPS_PER_BLOCK); cfg.dynamicSmemBytes = smem2;
        err = cudaLaunchKernelEx(&cfg, k2, p);
        if (err != cudaSuccess) return err;
        if (k3_old) {
            cfg.gridDim = dim3(p.n_envs); cfg.blockDim = dim3(FEAS_THREADS); cfg.dynamicSmemBytes = 0;
            err = (p.opt & PCT_OPT_DELTA) ? cudaLaunchKernelEx(&cfg, pct_feas_emit_kernel<OT, STAB, SlotT, true, SEL>, p)
                             : cudaLaunchKernelEx(&cfg, pct_feas_emit_kernel<OT, STAB, SlotT, false, SEL>, p);
            if (err != cudaSuccess) return err;
        }
    } else {
        k2<<<blocks, 32 * WARPS_PER_BLOCK, smem2, st>>>(p);
        if (prof) cudaEventRecord(prof[2], st);
        if (k3_old) {
            if (p.opt & PCT_OPT_DELTA) pct_feas_emit_kernel<OT, STAB, SlotT, true, SEL><<<slots, FEAS_THREADS, 0, st>>>(p);
            else pct_feas_emit_kernel<OT, STAB, SlotT, false, SEL><<<slots, FEAS_THREADS, 0, st>>>(p);
        }
    }
    if (!k3_old) {
        // the pooled walks need EVERY env's classification (plain stream order = full dependency), the emit kernel every walk
        if (p.ready && prof) cudaEventRecord(prof[2], st);
        if (STAB) {
            int n_sm = 0;
            err = sm_count(&n_sm);
            if (err != cudaSuccess) return err;
            const DParams &pw = p;  // the walks carry their env (WalkItem::env) and size the continuation pool from p.n_envs: the same kernels serve a selection
            pct_walk_light_kernel<<<n_sm * LIGHT_MINB, 32 * LIGHT_WARPS, 0, st>>>(pw);
            if (p.walk.walk_fork) pct_walk_fork_kernel<<<n_sm * max(1, min(p.walk.walk_blocks, WALK_MINB)), 32 * WALK_WARPS, 0, st>>>(pw);  // one resident wave
            else pct_walk_kernel<<<n_sm * WALK_MINB, 32 * WALK_WARPS, 0, st>>>(pw);  // one resident wave (every block starts at once: the emit kernel may follow)
        }
        const int eb = (slots + EMIT_WARPS - 1) / EMIT_WARPS;
        {   // programmatic dependent of the continuation kernel (setting 2: of the candidates kernel, whose blocks never trigger early -> plain order)
            cudaLaunchAttribute at[1];
            at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
            at[0].val.programmaticStreamSerializationAllowed = 1;
            cudaLaunchConfig_t cfg{};
            cfg.stream = st; cfg.attrs = at; cfg.numAttrs = (STAB && p.ready && !(p.opt & PCT_OPT_NO_EMIT_PDL)) ? 1 : 0;
            cfg.gridDim = dim3(eb); cfg.blockDim = dim3(32 * EMIT_WARPS); cfg.dynamicSmemBytes = 0;
            err = (p.opt & PCT_OPT_DELTA) ? cudaLaunchKernelEx(&cfg, pct_emit_kernel<OT, SlotT, true, SEL>, p) : cudaLaunchKernelEx(&cfg, pct_emit_kernel<OT, SlotT, false, SEL>, p);
            if (err != cudaSuccess) return err;
        }
    }
    if (prof) cudaEventRecord(prof[3], st);
    return cudaGetLastError();
}
template <typename OT, bool STAB>
static cudaError_t launch_s(const DParams &p, cudaStream_t st, cudaEvent_t *prof, bool apply, const EnvSel *sel) {
    const bool narrow = p.W <= 16 && p.L <= 16 && p.H <= 16;
    if (sel) {
        SelParams<DParams> ps;
        static_cast<DParams &>(ps) = p;
        ps.sel = *sel;
        return narrow ? launch_t<OT, STAB, uint16_t, true>(ps, st, nullptr, apply) : launch_t<OT, STAB, uint32_t, true>(ps, st, nullptr, apply);
    }
    if (narrow) return launch_t<OT, STAB, uint16_t, false>(p, st, prof, apply);
    return launch_t<OT, STAB, uint32_t, false>(p, st, prof, apply);
}

// number of kernels one reset / step enqueues (for pct_kernel_launches): apply, candidates (+ classify), [walk], emit, order / pool reset
int discrete_kernels_per_step(const DParams &p) {
    if ((p.opt & PCT_OPT_K3_BLOCK) || !p.walk.walkq) return 3;
    return 3 + (p.setting != 2 ? 2 : 0);
}

cudaError_t launch_discrete(const DParams &p, cudaStream_t st, cudaEvent_t *prof, bool apply, const EnvSel *sel) {
    const bool stab = p.setting != 2;
    if (p.obs_f64) return stab ? launch_s<double, true>(p, st, prof, apply, sel) : launch_s<double, false>(p, st, prof, apply, sel);
    return stab ? launch_s<float, true>(p, st, prof, apply, sel) : launch_s<float, false>(p, st, prof, apply, sel);
}

// the apply kernel alone, in plain stream order (pct_buffer_step / pct_buffer_reset: the buffered pipeline's own kernels run around it);
// SEL: over the selection's slots (pct_buffer_step_envs)
template <bool STAB, bool SEL>
static cudaError_t launch_apply_s(const ParamsT<DParams, SEL> &p, int slots, cudaStream_t st) {
    static bool attr_set = false;
    const size_t smem1 = (size_t)K1_SM_PER_WARP * WARPS_PER_BLOCK;
    if (!attr_set) {
        cudaError_t err = set_smem(pct_apply_kernel<STAB, false, SEL>, smem1);
        if (err == cudaSuccess && STAB) err = set_smem(pct_apply_kernel<STAB, STAB, SEL>, smem1);
        if (err != cudaSuccess) return err;
        attr_set = true;
    }
    const int blocks = (slots + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK;
    if (STAB && (p.opt & PCT_OPT_ALIAS)) pct_apply_kernel<STAB, STAB, SEL><<<blocks, 32 * WARPS_PER_BLOCK, smem1, st>>>(p);
    else pct_apply_kernel<STAB, false, SEL><<<blocks, 32 * WARPS_PER_BLOCK, smem1, st>>>(p);
    return cudaGetLastError();
}
cudaError_t launch_apply_discrete(const DParams &p, cudaStream_t st, const EnvSel *sel) {
    if (sel) {
        SelParams<DParams> ps;
        static_cast<DParams &>(ps) = p;
        ps.sel = *sel;
        const int slots = sel->slots(p.n_envs);
        return p.setting != 2 ? launch_apply_s<true, true>(ps, slots, st) : launch_apply_s<false, true>(ps, slots, st);
    }
    return p.setting != 2 ? launch_apply_s<true, false>(p, p.n_envs, st) : launch_apply_s<false, false>(p, p.n_envs, st);
}

cudaError_t launch_policy_random_discrete(const DEnvHot *hot, int n_envs, int64_t env_id_base, uint64_t seed, int64_t t, int32_t *leaf_idx,
                                          cudaStream_t st, const int64_t *t_dev) {
    pct_policy_random_kernel<<<(n_envs + 127) / 128, 128, 0, st>>>(hot, n_envs, env_id_base, seed, t, t_dev, leaf_idx);
    return cudaGetLastError();
}

}  // namespace pct

#include "pct_heuristics.cuh"
#include "pct_query.cuh"
