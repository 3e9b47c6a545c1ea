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

// EventPoint over the maintained EMS list and ZMAP (LNES 'EVM', include/pct_b200.h): the reference's EventPoint (D:space.py:613-693) as it
// behaves when GENEMS runs after every placement.  The ZMAP is a pure function of the placed boxes in order: level 0 holds x_up {0}, y_left
// {0}, x_bottom {W}, y_right {L}; a box (x1,y1,z1,x2,y2,z2) adds x2 (if < W), y2 (if < L), x1, y1 to the four lists of level z1 and, if
// z2 < H, x1, y1, x2, y2 to those of level z2, a level created in placement order.  The lists are sorted sets.  Per level with an EMS at
// z == k, in level order: the CPython set of (xs, ys, k, xe, ye, k + sz) over rotation x {x_up, x_bottom - sx} x {y_left, y_right - sy},
// then the tuples inside some EMS of that level (2-D containment).  The set emulation keys are offset coordinates (xs and ys may be
// negative) with the rotation's canonical index; the kept tuples are written to `out` as candidate keys.  PCT_FLAG_CAND_OVERFLOW: a
// level's set beyond the emulation's 1228 entries (the levels from it on are dropped) or the list beyond EVM_LIST_MAX (truncated).
constexpr int EVM_LIST_MAX = 1228;

__device__ __forceinline__ uint64_t py_int_hash(int v) { return (uint64_t)(int64_t)(v == -1 ? -2 : v); }

// hash of the tuple a set key of level k stands for (noinline, as key_hash: it keeps the callers' register counts)
template <int F>
__device__ __noinline__ uint64_t evm_key_hash(uint32_t e, const RotTab *rt, int k) {
    constexpr int OFF = 1 << (F - 1);
    const int xs = (int)(e & ((1u << F) - 1)) - OFF, ys = (int)((e >> F) & ((1u << F) - 1)) - OFF, c = (int)(e >> (2 * F));
    const uint64_t l[6] = {py_int_hash(xs), py_int_hash(ys), (uint64_t)k, py_int_hash(xs + rt->d[c][0]), py_int_hash(ys + rt->d[c][1]),
                           (uint64_t)(k + rt->d[c][2])};
    return tuple_hash6(l);
}

// the four ZMAP lists of level k, sorted, at lists[0 / 256 / 512 / 768]: x_up, y_left, x_bottom, y_right -> their lengths
static __device__ __noinline__ int4 evm_level_lists(const int16_t (*box)[6], int n_box, int k, int W, int L, uint8_t *lists, int lane) {
    // bitmasks over 0..255: lane = list * 8 + word
    const int li = lane >> 3, lo = (lane & 7) * 32;
    uint32_t bits = 0;
    auto put = [&](int v) { if (v >= lo && v < lo + 32) bits |= 1u << (v - lo); };
    if (k == 0) put(li == 0 || li == 1 ? 0 : li == 2 ? W : L);
#pragma unroll 1
    for (int i = 0; i < n_box; i++) {
        const int16_t *b = box[i];
        if (b[2] == k) {  // maintainEventBottom
            if (li == 0) { if (b[3] < W) put(b[3]); } else if (li == 1) { if (b[4] < L) put(b[4]); } else put(b[li - 2]);
        }
        if (b[5] == k) put(li == 0 ? b[0] : li == 1 ? b[1] : b[li + 1]);  // AddNewEMSZ
    }
    const int cnt = __popc(bits);
    int pre = cnt;  // inclusive prefix inside the list's 8 lanes
#pragma unroll
    for (int d = 1; d < 8; d <<= 1) {
        const int t = __shfl_up_sync(FULL, pre, d);
        if ((lane & 7) >= d) pre += t;
    }
    const int tot = __shfl_sync(FULL, pre, li * 8 + 7);
    pre -= cnt;
    for (uint32_t m = bits; m; m &= m - 1) lists[li * 256 + pre++] = (uint8_t)(lo + __ffs(m) - 1);
    __syncwarp();
    return make_int4(__shfl_sync(FULL, tot, 0), __shfl_sync(FULL, tot, 8), __shfl_sync(FULL, tot, 16), __shfl_sync(FULL, tot, 24));
}

// one level's set of set keys, inserted as build_candidates inserts: the table it ends in (a stage of tabA / tabB / tabBig) and its mask;
// mask 0: the set outgrew the emulation, or a coordinate the key's range (PCT_FLAG_CAND_OVERFLOW)
template <typename SlotT>
struct EvmSet {
    SlotT *tab;
    uint32_t mask;
};
template <typename SlotT>
__device__ __forceinline__ EvmSet<SlotT> evm_level_set(const RotTab *rt, int R, int k, const uint8_t *lists, int4 ln, SlotT *tabA, SlotT *tabB,
                                                    SlotT *tabBig, int lane) {
    constexpr int F = sizeof(SlotT) == 2 ? 6 : 10;          // set key fields: xs + OFF, ys + OFF, canonical rotation
    constexpr int OFF = 1 << (F - 1);
    constexpr SlotT EMPTY = (SlotT)~(SlotT)0;
    const int nxu = ln.x, nyl = ln.y, ny = ln.y + ln.w, per = (ln.x + ln.z) * ny;
    int nrot = 0;
    for (int r = 0; r < R; r++) nrot += (rt->valid >> r) & 1;
    const int raw_n = nrot * per;
    auto hash_of = [rt, k](SlotT e) { return evm_key_hash<F>(e, rt, k); };
    SlotT *tab = tabA;
    uint32_t mask = 7;
    int fill = 0;
    if (lane < 8) tab[lane] = EMPTY;
    __syncwarp();
#pragma unroll 1
    for (int base = 0; base < raw_n; base += 32) {
        const int r = base + lane;
        bool valid = false, range = false;
        uint64_t hash = 0;
        uint32_t key = 0xFFFFFFFFu;
        if (r < raw_n) {
            int q = r / per, rot = 0;
            const int t = r - q * per, i = t / ny, j = t - i * ny;
            for (; rot < R; rot++)
                if (((rt->valid >> rot) & 1) && q-- == 0) break;
            const int xs = i < nxu ? lists[i] : lists[512 + i - nxu] - rt->d[rot][0];
            const int ys = j < nyl ? lists[256 + j] : lists[768 + j - nyl] - rt->d[rot][1];
            range = xs + OFF < 0 || xs + OFF >= (1 << F) || ys + OFF < 0 || ys + OFF >= (1 << F);  // an item beyond the key's range
            if (!range) {
                valid = true;
                key = (uint32_t)(xs + OFF) | ((uint32_t)(ys + OFF) << F) | ((uint32_t)rt->canon[rot] << (2 * F));
                hash = hash_of((SlotT)key);
            }
        }
        if (__any_sync(FULL, range)) return EvmSet<SlotT>{tab, 0};
        const uint32_t same = __match_any_sync(FULL, key);
        if (valid && (same & ((1u << lane) - 1))) valid = false;
        SetProbe pr;
        pr.home(hash, mask);
#pragma unroll 1
        for (;;) {
            if (valid && set_seek(tab, mask, pr, [key](SlotT e) { return e == (SlotT)key; })) valid = false;
            const uint32_t room = (mask * 3 + 4) / 5 - (uint32_t)fill;
            const uint32_t cm = set_claim_round(valid, pr.slot(), lane, room);
            if (!cm) break;
            if ((cm >> lane) & 1) { tab[pr.slot()] = (SlotT)key; valid = false; }
            fill += __popc(cm);
            __syncwarp();
            if ((uint32_t)fill * 5 >= mask * 3) {
                uint32_t newsize = 8;
                while (newsize <= (uint32_t)fill * 4) newsize <<= 1;
                if (newsize > TAB_A) return EvmSet<SlotT>{tab, 0};
                SlotT *nt = newsize == TAB_A ? tabBig : ((tab == tabA) ? tabB : tabA);
                for (uint32_t t = lane; t < newsize; t += 32) nt[t] = EMPTY;
                __syncwarp();
                set_rehash(tab, mask, nt, newsize - 1, lane, hash_of);
                tab = nt;
                mask = newsize - 1;
                pr.home(hash, mask);
            }
        }
    }
    __syncwarp();
    return EvmSet<SlotT>{tab, mask};
}

template <typename SlotT>
__device__ __noinline__ CandList<SlotT> gen_event_point_m(const DEnvHot *hot, const RotTab *rt, int R, int W, int L, int H, SlotT *tabA, SlotT *tabB,
                                                          SlotT *tabBig, uint32_t *raw, SlotT *out, int lane) {
    constexpr int KB = sizeof(SlotT) == 2 ? 4 : 8;          // candidate key fields (key_pack)
    constexpr int F = sizeof(SlotT) == 2 ? 6 : 10;
    constexpr int OFF = 1 << (F - 1);
    constexpr SlotT EMPTY = (SlotT)~(SlotT)0;
    const int16_t (*ems)[6] = hot->ems, (*box)[6] = hot->box;
    const int n_ems = hot->h.n_ems, n_box = hot->h.n_box;
    uint8_t *lists = (uint8_t *)raw;                        // x_up, y_left, x_bottom, y_right of the current level, 256 bytes each
    int n_out = 0;
#pragma unroll 1
    for (int lv = -1; lv < n_box; lv++) {
        // level keys: 0, then each top z2 < H not seen before, in placement order
        int k = 0;
        if (lv >= 0) {
            k = box[lv][5];
            bool seen = k >= H;
            for (int i = lane; i < lv && !seen; i += 32) seen = box[i][5] == k;
            if (__any_sync(FULL, seen)) continue;
        }
        bool has = false;
        for (int i = lane; i < n_ems; i += 32) has |= ems[i][2] == k;
        if (!__any_sync(FULL, has)) continue;
        const EvmSet<SlotT> st = evm_level_set<SlotT>(rt, R, k, lists, evm_level_lists(box, n_box, k, W, L, lists, lane), tabA, tabB, tabBig, lane);
        if (!st.mask) return CandList<SlotT>{out, n_out, PCT_FLAG_CAND_OVERFLOW};
        // slot order, kept if inside an EMS of the level (D:space.py:676-691)
#pragma unroll 1
        for (uint32_t b2 = 0; b2 <= st.mask; b2 += 32) {
            const uint32_t s = b2 + lane;
            const SlotT e = s <= st.mask ? st.tab[s] : EMPTY;
            bool keep = false;
            int xs = 0, ys = 0, c = 0;
            if (e != EMPTY) {
                xs = (int)(e & ((1u << F) - 1)) - OFF; ys = (int)((e >> F) & ((1u << F) - 1)) - OFF; c = (int)(e >> (2 * F));
                const int xe = xs + rt->d[c][0], ye = ys + rt->d[c][1];
                for (int i = 0; i < n_ems && !keep; i++) {
                    const int16_t *m = ems[i];
                    keep = m[2] == k && m[0] <= xs && m[1] <= ys && xe <= m[3] && ye <= m[4];
                }
            }
            const uint32_t km = __ballot_sync(FULL, keep);
            const int p = n_out + __popc(km & ((1u << lane) - 1));
            if (keep && p < EVM_LIST_MAX) out[p] = (SlotT)key_pack<KB>(xs, ys, k, c);
            n_out += __popc(km);
        }
        __syncwarp();
        if (n_out > EVM_LIST_MAX) return CandList<SlotT>{out, EVM_LIST_MAX, PCT_FLAG_CAND_OVERFLOW};
    }
    return CandList<SlotT>{out, n_out, 0};
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
