// Snapshot / restore of env states (include/pct_b200.h: pct_snapshot_bytes, pct_snapshot, pct_restore), both domains.
//
// A record is what carries over from one step to the next (DESIGN.md section 10): the per-env fields a step reads before it writes them.
// Its layout is fixed per domain (fixed stride, so records can be indexed) and mirrors the env structs at the same offsets modulo 16, so
// every field moves with 16-byte vector copies between a byte head and tail.  Only the live prefixes the header counts describe are
// moved; the rest of a record is never written or read.  Records hold no pointers and nothing slot-dependent: a record restores into any
// slot of any handle whose fingerprint (domain, setting, container, holders, lnes, alias mode) matches.
//
//   [0, 16)        SnapHdr: magic, layout version, fingerprint
//   discrete       DEnvHot (whole struct layout)          | DEnvCold [0, cand): leaf, density, e_st, poly | DEnvAux alias arrays | LSAH int32[4]
//   continuous     CEnv [0, ems_tmp): hdr, box, den, ems  | CEnv [e_off, cand): CSR, edges, loads, polygons, leaf | DEnvAux alias arrays | LSAH double[4]
#include <cstddef>
#include "pct_kernels.h"
#include "pct_handle.h"
#include "pct_obs.cuh"
#include "pct_continuous.cuh"

namespace pct {

struct SnapHdr {
    uint32_t magic, version;
    uint64_t fingerprint;
};
static_assert(sizeof(SnapHdr) == 16, "record header");
constexpr uint32_t SNAP_MAGIC = 0x53544350u;  // "PCTS"
constexpr uint32_t SNAP_VERSION = 1;
constexpr int SNAP_THREADS = 128;              // one block per env

constexpr size_t up16(size_t x) { return (x + 15) & ~(size_t)15; }
constexpr size_t AUX_BYTES = offsetof(DEnvAux, obs_prev);  // box_st, e_upper, e_alias (obs_prev belongs to the caller's buffer, not to the env)
// discrete record
constexpr size_t D_HOT = sizeof(SnapHdr);
constexpr size_t D_COLD = D_HOT + sizeof(DEnvHot);
constexpr size_t D_AUX = D_COLD + offsetof(DEnvCold, cand);
constexpr size_t D_HS = D_AUX + up16(AUX_BYTES);
constexpr size_t D_REC = D_HS + 4 * sizeof(int32_t);
// continuous record
constexpr size_t C_A = sizeof(SnapHdr);
constexpr size_t C_B = C_A + offsetof(CEnv, ems_tmp);
constexpr size_t C_AUX = up16(C_B + offsetof(CEnv, cand) - offsetof(CEnv, e_off));
constexpr size_t C_HS = C_AUX + up16(AUX_BYTES);
constexpr size_t C_REC = C_HS + 4 * sizeof(double);
static_assert(D_COLD % 16 == 0 && D_AUX % 16 == 0 && D_REC % 16 == 0, "discrete record: 16-byte aligned regions");
static_assert(offsetof(DEnvCold, leaf) == 0 && offsetof(DEnvCold, density) < offsetof(DEnvCold, cand) &&
              offsetof(DEnvCold, e_st) < offsetof(DEnvCold, cand) && offsetof(DEnvCold, poly) < offsetof(DEnvCold, cand),
              "the persistent cold fields form the prefix of DEnvCold");
static_assert(C_B % 16 == offsetof(CEnv, e_off) % 16 && C_REC % 16 == 0, "continuous record: offsets congruent to the struct's modulo 16");
static_assert(offsetof(CEnv, ems_tmp) < offsetof(CEnv, e_off) && offsetof(CEnv, leaf) < offsetof(CEnv, cand) &&
              offsetof(CEnv, cand) < offsetof(CEnv, big) && offsetof(CEnv, big) < offsetof(CEnv, fbits),
              "transient continuous fields lie outside the two copied ranges");

struct SnapArgs {
    unsigned char *buf;       // records, `stride` bytes apart
    const int32_t *env, *rec; // nullptr: identity
    int n, n_envs;
    int64_t stride;
    uint64_t fp;
    DEnvHot *hot;
    DEnvCold *cold;
    CEnv *cenv;
    DEnvAux *aux;             // obs_prev of restored envs (nullptr: no delta rows); with `alias` also the EdgePoolA arrays
    int alias;
    void *hstate;
    int nb, nl;
};

// n bytes between two addresses that agree modulo sizeof(V): byte head, V vectors, byte tail
template <typename V>
__device__ __forceinline__ void span_v(unsigned char *dst, const unsigned char *src, int n, int tid) {
    constexpr int W = (int)sizeof(V);
    const int head = min(n, (int)((W - ((uintptr_t)src & (W - 1))) & (W - 1)));
    const int nv = (n - head) / W;
    for (int i = tid; i < head; i += SNAP_THREADS) dst[i] = src[i];
    const V *sv = (const V *)(src + head);
    V *dv = (V *)(dst + head);
    for (int i = tid; i < nv; i += SNAP_THREADS) dv[i] = sv[i];
    for (int i = head + W * nv + tid; i < n; i += SNAP_THREADS) dst[i] = src[i];
}
// The record mirrors the env structs modulo 16, so all but the DEnvAux fields of every other env (sizeof(DEnvAux) is a multiple of 8 only)
// move as 16-byte vectors
__device__ __forceinline__ void span(unsigned char *dst, const unsigned char *src, int n, int tid) {
    if (n <= 0) return;
    const uintptr_t d = (uintptr_t)dst ^ (uintptr_t)src;
    if ((d & 15) == 0) span_v<int4>(dst, src, n, tid);
    else if ((d & 7) == 0) span_v<int2>(dst, src, n, tid);
    else span_v<unsigned char>(dst, src, n, tid);
}
// SAVE: record <- object, else object <- record
template <bool SAVE>
__device__ __forceinline__ void xfer(unsigned char *rec, size_t roff, void *obj, size_t ooff, int n, int tid) {
    unsigned char *o = (unsigned char *)obj + ooff;
    if (SAVE) span(rec + roff, o, n, tid);
    else span(o, rec + roff, n, tid);
}
__device__ __forceinline__ int clampi(int v, int hi) { return v < 0 ? 0 : (v > hi ? hi : v); }

template <bool SAVE>
__device__ void move_aux(unsigned char *r, size_t base, const SnapArgs &a, int e, int nb, int ned, int tid) {
    if (!a.aux || !a.alias) return;
    DEnvAux *ax = a.aux + e;
    xfer<SAVE>(r, base + offsetof(DEnvAux, box_st), ax, offsetof(DEnvAux, box_st), nb * (int)sizeof(Stack4), tid);
    xfer<SAVE>(r, base + offsetof(DEnvAux, e_upper), ax, offsetof(DEnvAux, e_upper), ned, tid);
    xfer<SAVE>(r, base + offsetof(DEnvAux, e_alias), ax, offsetof(DEnvAux, e_alias), ((ned + 31) >> 5) * 4, tid);
}

// counts come from the header being copied (the env's when saving, the record's when restoring)
template <bool SAVE>
__device__ void move_discrete(unsigned char *r, const SnapArgs &a, int e, const DHdr &h, int tid) {
    const int nb = clampi(h.n_box, NB_MAX), ne = clampi(h.n_ems, E_MAX), ned = clampi(h.n_edge, EDGE_MAX), npo = clampi(h.n_poly, POLY_MAX),
              nl = clampi(h.n_leaf, NL_MAX);
    DEnvHot *hot = a.hot + e;
    DEnvCold *cold = a.cold + e;
#define HOT(f, bytes) xfer<SAVE>(r, D_HOT + offsetof(DEnvHot, f), hot, offsetof(DEnvHot, f), (bytes), tid)
#define COLD(f, bytes) xfer<SAVE>(r, D_COLD + offsetof(DEnvCold, f), cold, offsetof(DEnvCold, f), (bytes), tid)
    HOT(h, (int)sizeof(DHdr));
    HOT(box, nb * 12);
    HOT(ems, ne * 12);
    HOT(e_off, (nb + 1) * 2);     // CSR by box: off[0 .. n_box]
    HOT(e_lower, ned);
    HOT(e_next, ned);
    HOT(first_in, nb);
    HOT(last_in, nb);
    HOT(poly_off, (nb + 1) * 2);
    COLD(leaf, nl * 12);
    COLD(density, nb * 8);
    COLD(e_st, ned * (int)sizeof(Stack4));
    COLD(poly, npo * 16);
#undef HOT
#undef COLD
    move_aux<SAVE>(r, D_AUX, a, e, nb, ned, tid);
    xfer<SAVE>(r, D_HS, a.hstate, (size_t)e * 16, 16, tid);
}

template <bool SAVE>
__device__ void move_continuous(unsigned char *r, const SnapArgs &a, int e, const CHdr &h, int tid) {
    const int nb = clampi(h.n_box, NB_MAX), ne = clampi(h.n_ems, CE_MAX), ned = clampi(h.n_edge, EDGE_MAX), npo = clampi(h.n_poly, POLY_MAX),
              nl = clampi(h.n_leaf, NL_MAX);
    CEnv *ev = a.cenv + e;
#define FA(f, bytes) xfer<SAVE>(r, C_A + offsetof(CEnv, f), ev, offsetof(CEnv, f), (bytes), tid)
#define FB(f, bytes) xfer<SAVE>(r, C_B + offsetof(CEnv, f) - offsetof(CEnv, e_off), ev, offsetof(CEnv, f), (bytes), tid)
    FA(h, (int)sizeof(CHdr));
    FA(box, nb * 48);
    FA(den, nb * 8);
    FA(ems, ne * 48);
    FB(e_off, (nb + 1) * 2);
    FB(poly_off, (nb + 1) * 2);
    FB(e_lower, ned);
    FB(e_next, ned);
    FB(first_in, nb);
    FB(last_in, nb);
    FB(e_st, ned * (int)sizeof(Stack4));
    FB(poly, npo * 16);
    FB(leaf, nl * 48);
#undef FA
#undef FB
    move_aux<SAVE>(r, C_AUX, a, e, nb, ned, tid);
    xfer<SAVE>(r, C_HS, a.hstate, (size_t)e * 32, 32, tid);
}

template <bool CONT>
__global__ void __launch_bounds__(SNAP_THREADS) pct_snapshot_kernel(const SnapArgs a) {
    const int i = blockIdx.x, tid = threadIdx.x;
    const int e = a.env ? a.env[i] : i;
    unsigned char *r = a.buf + (size_t)i * (size_t)a.stride;
    if (e < 0 || e >= a.n_envs) {  // no such env: a header no restore accepts
        if (tid == 0) *(SnapHdr *)r = SnapHdr{0, 0, 0};
        return;
    }
    if (tid == 0) *(SnapHdr *)r = SnapHdr{SNAP_MAGIC, SNAP_VERSION, a.fp};
    if (CONT) move_continuous<true>(r, a, e, a.cenv[e].h, tid);
    else move_discrete<true>(r, a, e, a.hot[e].h, tid);
}

template <bool CONT, typename OT>
__global__ void __launch_bounds__(SNAP_THREADS) pct_restore_kernel(const SnapArgs a, const DParams pd, const CParams pc) {
    const int i = blockIdx.x, tid = threadIdx.x;
    const int e = a.env ? a.env[i] : i, k = a.rec ? a.rec[i] : i;
    if (e < 0 || e >= a.n_envs || k < 0) return;
    unsigned char *r = a.buf + (size_t)k * (size_t)a.stride;
    const SnapHdr sh = *(const SnapHdr *)r;
    if (sh.magic != SNAP_MAGIC || sh.version != SNAP_VERSION || sh.fingerprint != a.fp) {  // not this configuration's record: the env is left as it is
        if (tid == 0) {
            if (CONT) a.cenv[e].h.flags |= PCT_FLAG_BAD_SNAPSHOT;
            else a.hot[e].h.flags |= PCT_FLAG_BAD_SNAPSHOT;
        }
        return;
    }
    int n_leaf;
    if (CONT) {
        const CHdr h = *(const CHdr *)(r + C_A + offsetof(CEnv, h));
        move_continuous<false>(r, a, e, h, tid);
        n_leaf = clampi(h.n_leaf, NL_MAX);
    } else {
        const DHdr h = *(const DHdr *)(r + D_HOT + offsetof(DEnvHot, h));
        move_discrete<false>(r, a, e, h, tid);
        n_leaf = clampi(h.n_leaf, NL_MAX);
    }
    // the next step rewrites every row of whatever buffer it gets (include/pct_b200.h, delta rows)
    if (a.aux && tid == 0) { a.aux[e].obs_prev[0] = a.nb; a.aux[e].obs_prev[1] = a.nl; }
    if (!(CONT ? pc.obs : pd.obs)) return;
    __syncthreads();  // the restored record is complete before it is read back for the observation
    if (CONT) write_obs_c<OT>(pc, e, a.cenv + e, a.cenv[e].leaf, n_leaf, tid, SNAP_THREADS);
    else write_obs<OT, 0>(pd, e, a.hot + e, a.cold + e, a.cold[e].leaf, n_leaf, tid, SNAP_THREADS);
}

// ---- host side ----------------------------------------------------------------------------------------------
int64_t snapshot_record_bytes(const pct_env_batch *h) { return h->cfg.domain == PCT_CONTINUOUS ? (int64_t)C_REC : (int64_t)D_REC; }

// FNV-1a over everything that fixes the layout and the meaning of a record
uint64_t snapshot_fingerprint(const pct_env_batch *h) {
    uint64_t f = 0xcbf29ce484222325ull;
    auto mix = [&](const void *p, size_t n) {
        for (size_t i = 0; i < n; i++) { f ^= ((const unsigned char *)p)[i]; f *= 0x100000001b3ull; }
    };
    const int32_t v[6] = {h->cfg.domain, h->cfg.setting, h->cfg.internal_node_holder, h->cfg.leaf_node_holder, h->cfg.lnes, h->alias_mode ? 1 : 0};
    mix(v, sizeof v);
    mix(h->cfg.container_size, sizeof h->cfg.container_size);
    return f;
}

static SnapArgs snap_args(pct_env_batch *h, const int32_t *env, const int32_t *rec, int n, void *buf) {
    SnapArgs a{};
    a.buf = (unsigned char *)buf; a.env = env; a.rec = rec; a.n = n; a.n_envs = h->n_envs;
    a.stride = snapshot_record_bytes(h); a.fp = h->snap_fp;
    a.hot = h->d_hot; a.cold = h->d_cold; a.cenv = (CEnv *)h->c_state;
    a.aux = h->d_aux; a.alias = h->alias_mode ? 1 : 0;
    a.hstate = h->cfg.domain == PCT_CONTINUOUS ? (void *)h->d_hstate_c : (void *)h->d_hstate;
    a.nb = h->cfg.internal_node_holder; a.nl = h->cfg.leaf_node_holder;
    return a;
}

cudaError_t launch_snapshot(pct_env_batch *h, const int32_t *env, int n, void *buf, cudaStream_t st) {
    const SnapArgs a = snap_args(h, env, nullptr, n, buf);
    if (h->cfg.domain == PCT_CONTINUOUS) pct_snapshot_kernel<true><<<n, SNAP_THREADS, 0, st>>>(a);
    else pct_snapshot_kernel<false><<<n, SNAP_THREADS, 0, st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_restore(pct_env_batch *h, const int32_t *env, const int32_t *rec, int n, const void *buf, void *obs, cudaStream_t st) {
    const SnapArgs a = snap_args(h, env, rec, n, const_cast<void *>(buf));
    // the fields the row writers read (write_obs / write_obs_c)
    DParams pd{};
    CParams pc{};
    pd.obs = obs; pd.nb = pc.nb = h->cfg.internal_node_holder; pd.nl = pc.nl = h->cfg.leaf_node_holder;
    pd.setting = pc.setting = h->cfg.setting; pd.H = (int)h->cfg.container_size[2]; pc.H = h->cfg.container_size[2];
    pc.obs = obs;
    const bool f64 = h->cfg.obs_dtype == PCT_F64;
    if (h->cfg.domain == PCT_CONTINUOUS) {
        if (f64) pct_restore_kernel<true, double><<<n, SNAP_THREADS, 0, st>>>(a, pd, pc);
        else pct_restore_kernel<true, float><<<n, SNAP_THREADS, 0, st>>>(a, pd, pc);
    } else {
        if (f64) pct_restore_kernel<false, double><<<n, SNAP_THREADS, 0, st>>>(a, pd, pc);
        else pct_restore_kernel<false, float><<<n, SNAP_THREADS, 0, st>>>(a, pd, pc);
    }
    return cudaGetLastError();
}

}  // namespace pct
