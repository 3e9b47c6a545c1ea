// The ordered candidate list of the discrete env: the CPython-set emulation (build_candidates) and the generators of the other leaf-node
// expansion schemes.  Shared by the candidates kernel (pct_discrete.cu, included at the place the definitions stood, so its code is
// unchanged) and the leaf expansion of caller-given items (pct_expand.cu).
#pragma once
#include "pct_common.cuh"
#include "pct_kernels.h"
#include "pct_geom.cuh"
#include "pct_rot.cuh"

namespace pct {

// ---- candidate leaves in CPython set order (EMSPoint, D:space.py:534-570) ---------------------------------
struct SetStage {  // per-warp staging area of the candidates kernel's shared-memory layout; build_candidates does not use it
    uint64_t h[32];
    uint32_t k[32];
};

// The ordered list: `n` keys at `keys` (one of the tables), `flags` the PCT_FLAG_* bits raised.  Results come back by value: an output
// argument taken by reference would pin the caller's variable to the stack frame.
template <typename SlotT>
struct CandList {
    SlotT *keys;
    int n, flags;
};

// Inserting a key that is already in the set is a no-op, so only FIRST occurrences change the table: duplicates inside the 32-wide chunk
// are collapsed onto their lowest lane with __match_any_sync, and every lane walks its key's probe sequence in the table as it stood at
// the chunk's start (a present key is found on exactly the sequence that placed it).  A new key's walk stops on the first empty slot of
// its sequence, which is where set_add_entry would put it if no lane below had gone first.  The new keys then go in by claim rounds
// (set_claim_round, pct_common.cuh): each round commits, in one step, the lanes whose serial insertion in lane (= reference) order
// would land on the slot they stand on, and the others walk on from there.  A resize re-inserts the old table 32 slots at a time by the
// same rounds (set_rehash), and the keys still pending walk the new table from their home slots.
template <typename SlotT>
__device__ __noinline__ CandList<SlotT> build_candidates(const int16_t (*ems)[6], int n_ems, const RotTab *rt, int R, SlotT *tabA, SlotT *tabB, SlotT *tabBig,
                                                         SetStage *stg, int lane, const uint32_t *raw_keys = nullptr, int n_raw = 0) {
    (void)stg;
    constexpr int BITS = sizeof(SlotT) == 2 ? 4 : 8;
    constexpr SlotT EMPTY = (SlotT)~(SlotT)0;
    SlotT *tab = tabA;
    uint32_t mask = 7;
    int fill = 0, flags = 0;
    if (lane < 8) tab[lane] = EMPTY;
    __syncwarp();
    const int raw = raw_keys ? n_raw : n_ems * R * 4;  // raw_keys: insertion sequence produced by an EV / EP / CP / FC generator
    bool stop = false;
#pragma unroll 1
    for (int base = 0; base < raw && !stop; base += 32) {
        const int r = base + lane;
        bool valid = false;
        uint64_t hash = 0;
        uint32_t key = 0xFFFFFFFFu;
        if (r < raw && raw_keys) {
            valid = true;
            key = raw_keys[r];
            hash = key_hash<BITS>(key, rt);
        } else if (r < raw) {
            const int q = r & 3, er = r >> 2;
            const int rot = er % R, ei = er / R;
            if (rt->valid & (1 << rot)) {
                const int sx = rt->d[rot][0], sy = rt->d[rot][1], sz = rt->d[rot][2];
                const int16_t *m = ems[ei];
                if (m[3] - m[0] >= sx && m[4] - m[1] >= sy && m[5] - m[2] >= sz) {
                    valid = true;
                    const int xs = (q & 1) ? m[3] - sx : m[0];
                    const int ys = (q & 2) ? m[4] - sy : m[1];
                    key = key_pack<BITS>(xs, ys, m[2], rt->canon[rot]);
                    hash = key_hash<BITS>(key, rt);
                }
            }
        }
        // first occurrence inside the chunk
        const uint32_t same = __match_any_sync(FULL, key);
        if (valid && (same & ((1u << lane) - 1))) valid = false;
        SetProbe pr;
        pr.home(hash, mask);
        // the first pass of the seek is the read-only lookup (a present key drops out); later passes walk on from a lost claim or, after a
        // resize, from the home slot: the chunk's keys differ from each other and from the table's, so those find nothing equal
#pragma unroll 1
        for (;;) {
            if (valid && set_seek(tab, mask, pr, [key](SlotT e) { return e == (SlotT)key; })) valid = false;
            const uint32_t room = (mask * 3 + 4) / 5 - (uint32_t)fill;  // insertions until fill * 5 >= mask * 3
            const uint32_t cm = set_claim_round(valid, pr.slot(), lane, room);
            if (!cm) break;
            if ((cm >> lane) & 1) { tab[pr.slot()] = (SlotT)key; valid = false; }
            fill += __popc(cm);
            __syncwarp();
            if ((uint32_t)fill * 5 >= mask * 3) {
                // set_table_resize(used * 4): smallest power of two > 4 * used, re-insert in slot order
                uint32_t newsize = 8;
                while (newsize <= (uint32_t)fill * 4) newsize <<= 1;
                if (newsize > TAB_A) { flags |= PCT_FLAG_CAND_OVERFLOW; stop = true; break; }
                SlotT *nt = newsize == TAB_A ? tabBig : ((tab == tabA) ? tabB : tabA);
                for (uint32_t t = lane; t < newsize; t += 32) nt[t] = EMPTY;
                __syncwarp();
                set_rehash(tab, mask, nt, newsize - 1, lane, [rt](SlotT e) { return key_hash<BITS>(e, rt); });
                tab = nt;
                mask = newsize - 1;
                pr.home(hash, mask);
            }
        }
    }
    __syncwarp();
    // iteration order = slot order: compact the keys in place
    int cnt = 0;
#pragma unroll 1
    for (uint32_t b2 = 0; b2 <= mask; b2 += 32) {
        const uint32_t s = b2 + lane;
        const SlotT e = s <= mask ? tab[s] : EMPTY;
        const uint32_t em = __ballot_sync(FULL, e != EMPTY);
        __syncwarp();
        if (e != EMPTY) tab[cnt + __popc(em & ((1u << lane) - 1))] = e;
        cnt += __popc(em);
        __syncwarp();
    }
    return CandList<SlotT>{tab, cnt, flags};
}

// ---- the other leaf-node expansion schemes (D:bin3D.py:101-112): generators of the set-insertion sequence --------------
constexpr int RAW_MAX = 2048;

struct RawList {  // a generator's insertion sequence: `n` keys in the caller's raw buffer, `flags` the PCT_FLAG_* bits raised
    int n, flags;
};

// FullCoord (D:space.py:573-610): every cell x valid rotation with lz = height of the cell, rot-major / lx / ly order
template <int BITS>
__device__ __noinline__ RawList gen_full_coord(const int16_t (*box)[6], int n_box, const RotTab *rt, int R, int W, int L, int H, uint32_t *raw,
                                               int lane) {
    int n = 0, flags = 0;
    const int cells = W * L;
#pragma unroll 1
    for (int rot = 0; rot < R; rot++) {
        if (!(rt->valid & (1 << rot))) continue;
        const int sx = rt->d[rot][0], sy = rt->d[rot][1], sz = rt->d[rot][2];
#pragma unroll 1
        for (int b = 0; b < cells; b += 32) {
            const int c = b + lane, lx = c / L, ly = c - lx * L;
            bool ok = false;
            int lz = 0;
            if (c < cells) {
                lz = rest_height(box, 0, n_box, 1, lx, ly, lx + 1, ly + 1);
                ok = lx + sx <= W && ly + sy <= L && lz + sz <= H;
            }
            const uint32_t m = __ballot_sync(FULL, ok);
            if (ok) {
                const int p = n + __popc(m & ((1u << lane) - 1));
                if (p < RAW_MAX) raw[p] = key_pack<BITS>(lx, ly, lz, rt->canon[rot]);
            }
            n += __popc(m);
        }
    }
    if (n > RAW_MAX) { flags |= PCT_FLAG_CAND_OVERFLOW; n = RAW_MAX; }
    __syncwarp();
    return RawList{n, flags};
}

// EventPoint (D:space.py:613-693) as the reference actually behaves: GENEMS (which maintains EMS and ZMAP) only runs for
// LNES == 'EMS' (D:bin3D.py:172-175), so ZMAP stays {0: x_up [0], y_left [0], x_bottom [W], y_right [L]} and the EMS list
// stays [whole bin]: four bin-corner placements per rotation at z = 0 (oversized rotations produce nothing valid).
template <int BITS>
__device__ __noinline__ int gen_event_point(const RotTab *rt, int R, int W, int L, uint32_t *raw, int lane) {
    int n = 0;
    if (lane == 0) {
        for (int rot = 0; rot < R; rot++) {
            if (!(rt->valid & (1 << rot))) continue;
            const int sx = rt->d[rot][0], sy = rt->d[rot][1], c = rt->canon[rot];
            if (sx > W || sy > L) continue;
            raw[n++] = key_pack<BITS>(0, 0, 0, c);
            raw[n++] = key_pack<BITS>(0, L - sy, 0, c);
            raw[n++] = key_pack<BITS>(W - sx, 0, 0, c);
            raw[n++] = key_pack<BITS>(W - sx, L - sy, 0, c);
        }
    }
    n = __shfl_sync(FULL, n, 0);
    __syncwarp();
    return n;
}

// ExtremePoint2D (ep = true, D:space.py:696-750 + PctTools.extreme2D :107-135) and CornerPoint (ep = false,
// D:space.py:752-806 + PctTools.corners2D :137-159): per distinct top level k, the 2-D points of the boxes whose top is
// above k; points new w.r.t. the previous level x rotations.  Small serial algorithms over <= 80 boxes: lane 0 runs them.
// Returns -2 for the empty-bin special case (two hard-coded placements, a list, no set).
template <int BITS>
__device__ __noinline__ RawList gen_level_points(const int16_t (*box)[6], int n_box, const RotTab *rt, int R, int W, int L, int H, bool ep,
                                                 uint32_t *raw, int lane) {
    if (n_box == 0) return RawList{-2, 0};
    int n = 0, flags = 0;
    if (lane == 0) {
        int16_t tset[NB_MAX + 1];
        int nt = 0;
        tset[nt++] = 0;
        for (int i = 0; i < n_box; i++) {
            const int16_t t = box[i][5];
            bool f = false;
            for (int k = 0; k < nt; k++) f |= tset[k] == t;
            if (!f) tset[nt++] = t;
        }
        for (int i = 1; i < nt; i++) { int16_t v = tset[i]; int j = i - 1; while (j >= 0 && tset[j] > v) { tset[j + 1] = tset[j]; j--; } tset[j + 1] = v; }
        uint8_t ord[NB_MAX], em[NB_MAX];
        int16_t cur[2 * NB_MAX + 2][2], last[2 * NB_MAX + 2][2];
        int nlast = 0;
        bool over = false;
        for (int ti = 0; ti < nt; ti++) {
            const int k = tset[ti];
            int nr = 0, nc = 0;
            for (int i = 0; i < n_box; i++)
                if (box[i][5] > k) ord[nr++] = (uint8_t)i;  // IK in box order
            if (nr == 0) { cur[0][0] = 0; cur[0][1] = 0; nc = 1; }
            else if (!ep) {
                // corners2D: stable sort by (y_end, x_end) descending, staircase of the items that extend x
                for (int i = 1; i < nr; i++) {
                    const uint8_t o = ord[i];
                    int j = i - 1;
                    while (j >= 0 && (box[ord[j]][4] < box[o][4] || (box[ord[j]][4] == box[o][4] && box[ord[j]][3] < box[o][3]))) { ord[j + 1] = ord[j]; j--; }
                    ord[j + 1] = o;
                }
                int xrec = 0, m = 0;
                for (int i = 0; i < nr; i++)
                    if (box[ord[i]][3] > xrec) { em[m++] = ord[i]; xrec = box[ord[i]][3]; }
                cur[nc][0] = 0; cur[nc][1] = box[ord[0]][4]; nc++;
                for (int i = 1; i < m; i++) { cur[nc][0] = box[em[i - 1]][3]; cur[nc][1] = box[em[i]][4]; nc++; }
                cur[nc][0] = box[em[m - 1]][3]; cur[nc][1] = 0; nc++;
            } else {
                // extreme2D: stable sort by (ly, x_end) ascending; the two `demo` walls use the reference's hard-coded 10
                for (int i = 1; i < nr; i++) {
                    const uint8_t o = ord[i];
                    int j = i - 1;
                    while (j >= 0 && (box[ord[j]][1] > box[o][1] || (box[ord[j]][1] == box[o][1] && box[ord[j]][3] > box[o][3]))) { ord[j + 1] = ord[j]; j--; }
                    ord[j + 1] = o;
                }
                for (int i = 0; i < nr; i++) {
                    const int16_t *ni = box[ord[i]];
                    int maxb0 = -10, maxb2 = -10, e0x = 0, e0y = 0, e2x = 0, e2y = 0;
                    bool has0 = false, has2 = false;
                    bool first2 = false;  // newEps is a dict: .values() lists key 2 before key 0 when newEps[2] was assigned first (D:PctTools.py:121-127)
                    for (int b = 0; b < 2 + i; b++) {
                        int bx2, bx3;
                        if (b == 0) { bx2 = 0; bx3 = 10; } else if (b == 1) { bx2 = 10; bx3 = 0; } else { bx2 = box[ord[b - 2]][3]; bx3 = box[ord[b - 2]][4]; }
                        if (ni[0] >= bx2 && ni[4] < bx3 && bx2 > maxb0) { e0x = bx2; e0y = ni[4]; maxb0 = bx2; has0 = true; }
                        if (ni[1] >= bx3 && ni[3] < bx2 && bx3 > maxb2) { e2x = ni[3]; e2y = bx3; maxb2 = bx3; if (!has2 && !has0) first2 = true; has2 = true; }
                    }
                    int w = 0;  // deleteEps2D
                    for (int q = 0; q < nc; q++)
                        if (!(cur[q][0] >= ni[0] && cur[q][0] < ni[3] && cur[q][1] >= ni[1] && cur[q][1] < ni[4])) { cur[w][0] = cur[q][0]; cur[w][1] = cur[q][1]; w++; }
                    nc = w;
                    if (has0 && has2 && !(e0x == e2x && e0y == e2y)) {
                        // list(set(newEps.values())): CPython order of two int 2-tuples in an 8-slot table; the values are inserted in the
                        // dict's key order, the first takes its home slot, the second probes from its own (perturb path); iteration = slot order
                        uint64_t l0[2] = {(uint64_t)e0x, (uint64_t)e0y}, l2[2] = {(uint64_t)e2x, (uint64_t)e2y};
                        const uint64_t h0 = tuple_hash_n(l0, 2), h2 = tuple_hash_n(l2, 2);
                        uint64_t s0 = h0 & 7, s2 = h2 & 7;
                        if (first2) { uint64_t pert = h0; while (s0 == s2) { pert >>= 5; s0 = (s0 * 5 + 1 + pert) & 7; } }
                        else { uint64_t pert = h2; while (s2 == s0) { pert >>= 5; s2 = (s2 * 5 + 1 + pert) & 7; } }
                        if (s0 < s2) { cur[nc][0] = e0x; cur[nc][1] = e0y; nc++; cur[nc][0] = e2x; cur[nc][1] = e2y; nc++; }
                        else { cur[nc][0] = e2x; cur[nc][1] = e2y; nc++; cur[nc][0] = e0x; cur[nc][1] = e0y; nc++; }
                    } else if (has0) { cur[nc][0] = e0x; cur[nc][1] = e0y; nc++; }
                    else if (has2) { cur[nc][0] = e2x; cur[nc][1] = e2y; nc++; }
                }
            }
            for (int q = 0; q < nc; q++) {
                bool f = false;
                for (int u = 0; u < nlast; u++) f |= last[u][0] == cur[q][0] && last[u][1] == cur[q][1];
                if (f) continue;
                for (int rot = 0; rot < R; rot++) {  // CI point x rotation -> insertion sequence of posVec
                    if (!(rt->valid & (1 << rot))) continue;
                    if (cur[q][0] + rt->d[rot][0] <= W && cur[q][1] + rt->d[rot][1] <= L && k + rt->d[rot][2] <= H) {
                        if (n < RAW_MAX && cur[q][0] >= 0 && cur[q][1] >= 0) raw[n++] = key_pack<BITS>(cur[q][0], cur[q][1], k, rt->canon[rot]);
                        else over = true;
                    }
                }
            }
            for (int q = 0; q < nc; q++) { last[q][0] = cur[q][0]; last[q][1] = cur[q][1]; }
            nlast = nc;
        }
        if (over) flags |= PCT_FLAG_CAND_OVERFLOW;
    }
    n = __shfl_sync(FULL, n, 0);
    __syncwarp();
    return RawList{n, flags};
}

}  // namespace pct
