// The ordered candidate list of the continuous env (C:space.py:531-568): candidate codes, their 6-tuples and hashes, and the CPython-set
// emulation with the keyed shuffle.  Shared by pctc_candidates_kernel (pct_continuous.cu) and the leaf expansion of caller-given items
// (pct_expand.cu).
#pragma once
#include "pct_common.cuh"
#include "pct_continuous.cuh"

namespace pct {

__device__ __forceinline__ bool rot_dims_c(const double nb[3], int rot, double &sx, double &sy, double &sz) {  // C:space.py:537-559
    switch (rot) {
    case 0: sx = nb[0]; sy = nb[1]; sz = nb[2]; return true;
    case 1: sx = nb[1]; sy = nb[0]; sz = nb[2]; return !(fabs(sx - sy) < 1e-6);
    case 2: sx = nb[0]; sy = nb[2]; sz = nb[1]; return !(fabs(sx - sy) < 1e-6 && fabs(sy - sz) < 1e-6);
    case 3: sx = nb[1]; sy = nb[2]; sz = nb[0]; return !(fabs(sx - sy) < 1e-6 && fabs(sy - sz) < 1e-6);
    case 4: sx = nb[2]; sy = nb[0]; sz = nb[1]; return !(fabs(sx - sy) < 1e-6);
    default: sx = nb[2]; sy = nb[1]; sz = nb[0]; return !(fabs(sx - sy) < 1e-6);
    }
}
// candidate code = ems_idx << 5 | rot << 2 | corner  ->  the 6-tuple the reference adds to its set (C:space.py:563-566)
__device__ __forceinline__ void cand_tuple(uint16_t code, const double (*ems)[6], const double nb[3], double t[6]) {
    const double *m = ems[code >> 5];
    double sx, sy, sz;
    rot_dims_c(nb, (code >> 2) & 7, sx, sy, sz);
    const int q = code & 3;
    if (q & 1) { t[0] = m[3] - sx; t[3] = m[3]; } else { t[0] = m[0]; t[3] = m[0] + sx; }
    if (q & 2) { t[1] = m[4] - sy; t[4] = m[4]; } else { t[1] = m[1]; t[4] = m[1] + sy; }
    t[2] = m[2]; t[5] = m[2] + sz;
}
__device__ __noinline__ inline uint64_t hash_double_call(double v) { return hash_double(v); }  // one copy of the routine for the three call sites of the candidates kernel
__device__ __noinline__ inline uint64_t cand_hash_c(const double t[6]) {
    uint64_t l[6];
#pragma unroll 1
    for (int i = 0; i < 6; i++) l[i] = hash_double(t[i]);
    return tuple_hash6(l);
}

// Table slots are 32 bits: candidate code | 16-bit tag (the top bits of the tuple hash — CPython compares the stored hash before the keys, setobject.c).
// A probe rejects a non-matching slot on the tag alone; the exact 6-double comparison (tuples rebuilt from the two codes) runs only on a tag match,
// i.e. practically only for true duplicates.  Round 1 rebuilt and compared the tuple of EVERY probed slot and broadcast the six doubles of every
// inserted key through shuffles (a large share of this kernel's instructions went to _Py_HashDouble's frexp loop — now an integer rotation,
// pct_pyhash.cuh — and to shuffles).
__device__ __forceinline__ bool cand_equal(uint16_t a, uint16_t b, const double (*ems)[6], const double nb[3]) {
    double u[6], v[6];
    cand_tuple(a, ems, nb, u);
    cand_tuple(b, ems, nb, v);
    return u[0] == v[0] && u[1] == v[1] && u[2] == v[2] && u[3] == v[3] && u[4] == v[4] && u[5] == v[5];
}

// The set emulation of one warp: the candidate codes of the item `nb` (R orientations) over the EMS list of `ev`, in CPython-set order, into
// ev->cand (`cnt` of them, declared here), then the keyed shuffle when p.shuffle is set (scratch: ev->ems_tmp).  Expanded in place (a macro, not
// an inlined function, so that pctc_candidates_kernel keeps its code).  Names it uses from the enclosing scope: p, e, lane, ev, h (the header),
// nb, R, n_ems, fl (capacity flags, ORed), and the warp's shared tables uint32_t tabA[CC_TAB], tabB[512].  The callers' staging arrays
// (uint64_t stg_h[32], rs_h[32], uint32_t rs_c[32], uint16_t stg_c[32]) belong to their shared-memory layouts; the body no longer uses them.
#define PCTC_CANDIDATES_BODY                                                                                                                                   \
    constexpr uint32_t EMPTY = 0xFFFFFFFFu;                                                                                                                    \
    uint32_t *tab = tabA;                                                                                                                                      \
    uint32_t mask = 7;                                                                                                                                         \
    int fill = 0;                                                                                                                                              \
    if (lane < 8) tab[lane] = EMPTY;                                                                                                                           \
    __syncwarp();                                                                                                                                              \
    /* the callers' staging arrays keep their places in the shared-memory layouts, unused */                                                                   \
    asm volatile("" ::"r"(smem_u32(stg_h)), "r"(smem_u32(rs_h)), "r"(smem_u32(rs_c)), "r"(smem_u32(stg_c)));                                                   \
    const int raw = n_ems * R * 4;                                                                                                                             \
    bool stop = false;                                                                                                                                         \
_Pragma("unroll 1")                                                                                                                                              \
    for (int base = 0; base < raw && !stop; base += 32) {                                                                                                      \
        const int r = base + lane;                                                                                                                             \
        bool valid = false;                                                                                                                                    \
        uint64_t hash = 0;                                                                                                                                     \
        uint16_t code = 0;                                                                                                                                     \
        /* The four corners of one (EMS, orientation) are four adjacent lanes and their 6-tuples draw on ten distinct coordinates (x: m0, m0 + sx, m3 - sx, */ \
        /* m3; y alike; z: m2, m2 + sz): every lane hashes two or three of them (_Py_HashDouble, the expensive part) and the group exchanges the results, */   \
        /* instead of six hashes per lane.  Same expressions as cand_tuple, so the same bits. */                                                               \
        uint64_t h0 = 0, h1 = 0, h2 = 0;                                                                                                                       \
        const int q = r & 3;                                                                                                                                   \
        if (r < raw) {                                                                                                                                         \
            const int er = r >> 2, rot = er % R, ei = er / R;                                                                                                  \
            double sx, sy, sz;                                                                                                                                 \
            if (rot_dims_c(nb, rot, sx, sy, sz)) {                                                                                                             \
                const double *m = ev->ems[ei];                                                                                                                 \
                if (m[3] - m[0] + 1e-6 >= sx && m[4] - m[1] + 1e-6 >= sy && m[5] - m[2] + 1e-6 >= sz) {                                                        \
                    valid = true;                                                                                                                              \
                    code = (uint16_t)((ei << 5) | (rot << 2) | q);                                                                                             \
                    double v0, v1, v2 = 0;                                                                                                                     \
                    if (q == 0) { v0 = m[0]; v1 = m[0] + sx; v2 = m[2]; }                                                                                      \
                    else if (q == 1) { v0 = m[3] - sx; v1 = m[3]; v2 = m[2] + sz; }                                                                            \
                    else if (q == 2) { v0 = m[1]; v1 = m[1] + sy; }                                                                                            \
                    else { v0 = m[4] - sy; v1 = m[4]; }                                                                                                        \
                    h0 = hash_double_call(v0);                                                                                                                 \
                    h1 = hash_double_call(v1);                                                                                                                 \
                    if (q < 2) h2 = hash_double_call(v2);                                                                                                      \
                }                                                                                                                                              \
            }                                                                                                                                                  \
        }                                                                                                                                                      \
        {                                                                                                                                                      \
            const int gb = lane & ~3, lx = gb + (q & 1), ly = gb + 2 + (q >> 1);                                                                               \
            uint64_t l6[6];                                                                                                                                    \
            l6[0] = __shfl_sync(FULL, h0, lx); l6[3] = __shfl_sync(FULL, h1, lx);                                                                              \
            l6[1] = __shfl_sync(FULL, h0, ly); l6[4] = __shfl_sync(FULL, h1, ly);                                                                              \
            l6[2] = __shfl_sync(FULL, h2, gb); l6[5] = __shfl_sync(FULL, h2, gb + 1);                                                                          \
            if (valid) hash = tuple_hash6(l6);                                                                                                                 \
        }                                                                                                                                                      \
        /* the chunk's new keys go in by claim rounds in lane (= reference) order, as in the discrete build_candidates (pct_cand.cuh).  The first pass */      \
        /* of the seek is the read-only lookup; a lane that lost a claim walks on with the same tag + exact comparison, so a value-equal tuple of a */         \
        /* lower lane (equal hash: the same sequence) is met where set_add_entry would meet it, and the higher code drops out */                               \
        SetProbe pr;                                                                                                                                           \
        pr.home(hash, mask);                                                                                                                                   \
        const uint32_t tag = (uint32_t)(hash >> 48);                                                                                                           \
_Pragma("unroll 1")                                                                                                                                              \
        for (;;) {                                                                                                                                             \
            if (valid && set_seek(tab, mask, pr, [&](uint32_t sl) { return (sl >> 16) == tag && cand_equal((uint16_t)sl, code, ev->ems, nb); }))               \
                valid = false;                                                                                                                                 \
            const uint32_t room = (mask * 3 + 4) / 5 - (uint32_t)fill;                                                                                         \
            const uint32_t cm = set_claim_round(valid, pr.slot(), lane, room);                                                                                 \
            if (!cm) break;                                                                                                                                    \
            if ((cm >> lane) & 1) { tab[pr.slot()] = (tag << 16) | code; valid = false; }                                                                      \
            fill += __popc(cm);                                                                                                                                \
            __syncwarp();                                                                                                                                      \
            if ((uint32_t)fill * 5 >= mask * 3) {                                                                                                              \
                uint32_t newsize = 8;                                                                                                                          \
                while (newsize <= (uint32_t)fill * 4) newsize <<= 1;                                                                                           \
                if (newsize > CC_TAB) { fl |= PCT_FLAG_CAND_OVERFLOW; stop = true; break; }                                                                    \
                uint32_t *nt = (tab == tabA) ? tabB : tabA;                                                                                                    \
                for (uint32_t t = lane; t < newsize; t += 32) nt[t] = EMPTY;                                                                                   \
                __syncwarp();                                                                                                                                  \
                /* set_table_resize: re-insert in slot order (set_insert_clean: no comparisons); the slots hold the tag only, so the hash is rebuilt */        \
                set_rehash(tab, mask, nt, newsize - 1, lane, [&](uint32_t c2) {                                                                                \
                    double u[6];                                                                                                                               \
                    cand_tuple((uint16_t)c2, ev->ems, nb, u);                                                                                                  \
                    return cand_hash_c(u);                                                                                                                     \
                });                                                                                                                                            \
                tab = nt;                                                                                                                                      \
                mask = newsize - 1;                                                                                                                            \
                pr.home(hash, mask);                                                                                                                           \
            }                                                                                                                                                  \
        }                                                                                                                                                      \
    }                                                                                                                                                          \
    __syncwarp();                                                                                                                                              \
    int cnt = 0;                                                                                                                                               \
_Pragma("unroll 1")                                                                                                                                              \
    for (uint32_t b2 = 0; b2 <= mask; b2 += 32) {                                                                                                              \
        const uint32_t s = b2 + lane;                                                                                                                          \
        const uint32_t c2 = s <= mask ? tab[s] : EMPTY;                                                                                                        \
        const uint32_t em = __ballot_sync(FULL, c2 != EMPTY);                                                                                                  \
        if (c2 != EMPTY) ev->cand[cnt + __popc(em & ((1u << lane) - 1))] = (uint16_t)c2;                                                                       \
        cnt += __popc(em);                                                                                                                                     \
    }                                                                                                                                                          \
    __syncwarp();                                                                                                                                              \
    if (p.shuffle) {  /* scratch: the GENEMS temp list (24 KB, idle between apply kernels): keys at 0, permuted codes at 10 KB */                              \
        static_assert(sizeof(ev->ems_tmp) >= 10240 + sizeof(ev->cand), "shuffle scratch fits");                                                                \
        shuffle_candidates<uint16_t>(ev->cand, cnt, (uint64_t *)ev->ems_tmp, (uint16_t *)((char *)ev->ems_tmp + 10240), p.seed, (uint64_t)(p.env_id_base + e), \
                                     (uint64_t)h.draw_pos, lane);                                                                                              \
    }

}  // namespace pct
