"""The claim rounds of the candidate lists' set emulation (csrc/pct_common.cuh set_claim_round / set_rehash, used by build_candidates in
pct_cand.cuh and PCTC_CANDIDATES_BODY in pct_cand_c.cuh), modelled in Python on cand_inputs' hashing.

The device inserts a chunk's new keys a warp at a time.  Every lane walks its key's probe sequence to the first empty slot (or to an
equal key, which drops it); a round then commits, at once, every pending lane below the lowest one whose slot a lower pending lane holds
too, up to the insertion that makes the set grow; the others walk on from where they stand.  A resize re-inserts the old table 32 slots
at a time by the same rounds, and the keys still pending walk the new table from their home slots.  RoundsModel below does the same
thing step for step; it must give `list(set(...))` on every input of cand_inputs (and the serial model's order at the 1229-key stop),
and the floors assert that the inputs reach what makes the rounds differ from a serial insertion: chunks of several rounds, a waiting
lane that walks on to a slot a higher lane stood on in the same round (a rule that let the lowest lane of each slot win would give it
to the higher lane), resizes with keys still pending, rounds into the 2048-slot stage, and value-equal continuous tuples that meet after
a lost claim.  The seeded adversarial inputs here (raw key sequences whose keys share home slots and probe runs) are fed to the device
by test_gpu_cand_rounds.py.
"""
import collections
import random
import sys

import pytest

import cand_inputs as ci

pytestmark = pytest.mark.skipif(sys.version_info[:2] != (3, 12), reason="the candidate order is CPython 3.12's set order (DESIGN section 6)")


# ============================================================ the model ============================================================
def _home(h, mask):
    return [h & mask, 0, h]  # window start, offset in the window, perturb


def _next(p, mask):
    if p[1] < 9 and p[0] + 9 <= mask:
        p[1] += 1
    else:
        p[1] = 0
        p[2] >>= 5
        p[0] = (p[0] * 5 + 1 + p[2]) & mask


def _seek(tab, mask, p, key):
    """walk on to the first empty slot (False) or the slot holding `key` (True); key None: no comparison"""
    while True:
        e = tab[p[0] + p[1]]
        if e is None:
            return False
        if key is not None and e[1] == key[1] and e[0] == key[0]:
            return True
        _next(p, mask)


def _claim(pend, slot, room):
    """set_claim_round: the committing lanes (in lane order) and the lowest lane that lost its slot to a lower one (32: none)"""
    seen, c = set(), 32
    for l in pend:
        if slot[l] in seen:
            c = l
            break
        seen.add(slot[l])
    return [l for l in pend if l < c][:room], c


def new_stats():
    return dict(rounds=collections.Counter(), walk_onto_higher=0, resize_pending=collections.Counter(), big_rounds=0, rehash_rounds=0,
                rehash_multi=0, equal_after_loss=0, chunks=0)


class RoundsModel:
    def __init__(self, st, cap=ci.TAB_MAX):
        self.tab, self.mask, self.fill, self.cap, self.overflow, self.st = [None] * 8, 7, 0, cap, False, st

    def _rehash(self, newsize):
        old, nt, nmask, st = self.tab, [None] * newsize, newsize - 1, self.st
        for b in range(0, len(old), 32):
            lanes = {l: old[b + l] for l in range(min(32, len(old) - b)) if old[b + l] is not None}
            p = {l: _home(e[1], nmask) for l, e in lanes.items()}
            pend, n = sorted(lanes), 0
            while pend:
                for l in pend:
                    _seek(nt, nmask, p[l], None)
                commit, _ = _claim(pend, {l: p[l][0] + p[l][1] for l in pend}, 32)
                for l in commit:
                    nt[p[l][0] + p[l][1]] = lanes[l]
                pend = [l for l in pend if l not in commit]
                n += 1
                st["rehash_rounds"] += 1
                st["big_rounds"] += newsize == ci.TAB_MAX
            st["rehash_multi"] += n >= 2
        self.tab, self.mask = nt, nmask

    def chunk(self, lanes):
        """lanes: {lane: (key, hash)} of the chunk's first occurrences"""
        st = self.st
        p = {l: _home(kv[1], self.mask) for l, kv in lanes.items()}
        pend, lost, rounds, prev = sorted(lanes), set(), 0, None
        while True:
            for l in list(pend):
                if _seek(self.tab, self.mask, p[l], lanes[l]):
                    pend.remove(l)
                    st["equal_after_loss"] += l in lost
            if prev is not None:  # a waiting lane walked on to a slot a higher lane stood on last round
                st["walk_onto_higher"] += any(prev.get(h) == p[w][0] + p[w][1] for w in pend for h in prev if h > w)
            slot = {l: p[l][0] + p[l][1] for l in pend}
            commit, _ = _claim(pend, slot, (self.mask * 3 + 4) // 5 - self.fill)
            if not commit:
                break
            rounds += 1
            st["big_rounds"] += self.mask == ci.TAB_MAX - 1
            for l in commit:
                self.tab[slot[l]] = lanes[l]
            pend = [l for l in pend if l not in commit]
            lost |= set(pend)
            self.fill += len(commit)
            prev = slot
            if self.fill * 5 >= self.mask * 3:
                newsize = 8
                while newsize <= self.fill * 4:
                    newsize <<= 1
                if pend:
                    st["resize_pending"][(self.mask + 1, newsize)] += 1
                if newsize > self.cap:
                    self.overflow = True
                    break
                self._rehash(newsize)
                for l in pend:
                    p[l] = _home(lanes[l][1], self.mask)
                lost, prev = set(), None
        if lanes:
            st["rounds"][rounds] += 1
            st["chunks"] += 1

    def order(self):
        return [e[0] for e in self.tab if e is not None]


def run_rounds(seq, n_raw, st=None, dedupe=True):
    """[(raw position, tuple)] through the claim rounds: (ordered tuples, overflow, stats).  dedupe: the discrete kernel first drops the
    repeats inside a chunk (__match_any_sync on the key); the continuous one sends them all to the lookup and the rounds"""
    st = st if st is not None else new_stats()
    model = RoundsModel(st)
    by_chunk = collections.defaultdict(list)
    for r, t in seq:
        by_chunk[r // 32].append((r, t))
    for base in range(0, n_raw, 32):
        lanes = {}
        for r, t in by_chunk.get(base // 32, []):
            if not dedupe or all(u != t for u, _ in lanes.values()):
                lanes[r % 32] = (t, ci.uhash(t))
        model.chunk(lanes)
        if model.overflow:
            break
    return model.order(), model.overflow, st


# ======================================================= adversarial inputs =======================================================
def _bits_cont(bits):
    return (16, 16, 16) if bits == 4 else (255, 255, 255)


def _pool(bits, item, R, n, rng):
    """n distinct keys of `item`"""
    cont = _bits_cont(bits)
    c = ci.canon(item, R)
    rots = sorted(set(c[r] for r in range(R) if ci.rot_dims_d(item, r)[3]))
    keys = set()
    while len(keys) < n:
        rot = rng.choice(rots)
        sx, sy, sz = (item[ci.PERM[rot][k]] for k in range(3))
        keys.add(ci.key_pack(bits, rng.randint(0, cont[0] - sx), rng.randint(0, cont[1] - sy), rng.randint(0, cont[2] - sz), rot))
    return sorted(keys)


def colliding_case(seed, bits):
    """a raw key sequence whose chunks gather keys of one or two home slots of the table size they meet (slots modulo 8, 32, 128, 512,
    2048 in turn as the set grows), so that lanes share slots and probe runs, with a few repeats"""
    rng = random.Random(6007 * seed + bits)
    item, R = (1, 2, 3) if bits == 4 else (3, 5, 7), 6
    keys = _pool(bits, item, R, 1600 if bits == 8 else 1200, rng)
    h = {k: ci.uhash(ci.key_tuple(bits, k, item)) for k in keys}
    rng.shuffle(keys)
    seq, used, size = [], set(), 8
    while len(seq) < ci.RAW_MAX - 32 and len(used) < len(keys) - 64:
        n_used = len(used)
        size = 8
        while size <= 4 * n_used:  # the table the set holds at this point (about: resizes come at fill * 5 >= mask * 3)
            size <<= 1
        size = min(size, ci.TAB_MAX)
        homes = rng.sample(range(size), 2)
        chunk = [k for k in keys if k not in used and h[k] % size in homes][:rng.randint(6, 32)]
        if len(chunk) < 32:
            chunk += [k for k in keys if k not in used and k not in chunk][:rng.randint(0, 32 - len(chunk))]
        rng.shuffle(chunk)
        while len(chunk) < 32:
            chunk.insert(rng.randrange(len(chunk) + 1), rng.choice(chunk) if chunk and rng.random() < 0.5 else rng.choice(keys))
        used |= set(chunk)
        seq += chunk
    return dict(kind="raw", cont=_bits_cont(bits), item=item, R=R, raw=seq[:ci.RAW_MAX])


N_COLLIDE = 12


def adversarial_cases():
    return [colliding_case(s, bits) for s in range(N_COLLIDE) for bits in (4, 8)]


def equal_tuples_case(seed):
    """a continuous EMS list of many EMS exactly one orientation's size (the four corners give one tuple), each EMS given two to four
    times in a row with -0.0 for 0.0 in some copies: value-equal tuples from different codes fill whole chunks"""
    rng = random.Random(7727 * seed + 1)
    cont = ci.BINS_C[seed % len(ci.BINS_C)]
    s = min(cont)
    item = (round(0.13 * s, 3), round(0.29 * s, 3), round(0.41 * s, 3))
    ems = []
    while len(ems) < ci.CE_MAX - 4:
        sx, sy, sz = (item[k] for k in ci.PERM[rng.randrange(6)])
        x0, y0 = (round(rng.uniform(0, v * 0.5), 2) for v in cont[:2])
        m = [x0, y0, 0.0, x0 + sx, y0 + sy, cont[2]]
        for _ in range(rng.randint(2, 4)):
            ems.append([-0.0 if v == 0.0 and rng.random() < 0.5 else v for v in m])
    return dict(cont=cont, item=item, R=6, ems=ems[:ci.CE_MAX])


N_EQUAL = 8


def adversarial_continuous_cases():
    return [equal_tuples_case(s) for s in range(N_EQUAL)]


# ============================================================= tests =============================================================
def _run(cases, seq_of, dedupe=True):
    st = new_stats()
    for k, c in enumerate(cases):
        seq, n = seq_of(c)
        order, over, _ = run_rounds(seq, n, st, dedupe)
        ref = ci.reference_order([t for _, t in seq])
        if len(ref) <= ci.CAND_CAP:
            assert not over and order == ref, "case %d: the rounds do not give CPython's order" % k
        else:
            sorder, sover, _ = ci.run_device_order(seq, n)
            assert over and sover and order == sorder and len(order) == ci.CAND_CAP + 1, "case %d: the rounds differ from the serial model" % k
    return st


@pytest.fixture(scope="module")
def discrete():
    return _run(ci.discrete_cases() + adversarial_cases(), ci.case_sequence)


@pytest.fixture(scope="module")
def continuous():
    return _run(ci.continuous_cases() + adversarial_continuous_cases(), ci.c_sequence, dedupe=False)


def test_discrete_rounds_reach_the_edges(discrete):
    st = discrete
    print({k: (dict(v) if isinstance(v, collections.Counter) else v) for k, v in st.items()})
    r = st["rounds"]
    assert r[2] >= 20 and r[3] >= 20 and sum(v for n, v in r.items() if n >= 5) >= 20
    assert st["walk_onto_higher"] >= 10
    assert st["resize_pending"][(8, 32)] >= 10 and st["resize_pending"][(128, 512)] >= 10
    assert st["resize_pending"][(512, 2048)] >= 5
    assert st["big_rounds"] >= 100
    assert st["rehash_multi"] >= 100


def test_adversarial_inputs_alone_reach_the_edges():
    st = _run(adversarial_cases(), ci.case_sequence)
    assert sum(v for n, v in st["rounds"].items() if n >= 5) >= 50
    assert st["walk_onto_higher"] >= 10
    assert st["resize_pending"][(8, 32)] >= 5 and st["resize_pending"][(128, 512)] >= 5
    assert st["big_rounds"] >= 50
    st = _run(adversarial_continuous_cases(), ci.c_sequence, dedupe=False)
    assert st["equal_after_loss"] >= 1000 and sum(v for n, v in st["rounds"].items() if n >= 5) >= 10


def test_continuous_rounds_reach_the_edges(continuous):
    st = continuous
    print({k: (dict(v) if isinstance(v, collections.Counter) else v) for k, v in st.items()})
    r = st["rounds"]
    assert r[2] >= 20 and r[3] >= 20 and sum(v for n, v in r.items() if n >= 5) >= 5
    assert st["walk_onto_higher"] >= 5
    assert st["resize_pending"][(8, 32)] >= 5 and st["resize_pending"][(128, 512)] >= 1
    assert st["big_rounds"] >= 10
    assert st["equal_after_loss"] >= 5


def test_claim_round_is_lane_order():
    # lanes 0 and 5 share a slot, lanes 3 and 4 share another: lanes 0..3 commit (lane 4 is the first loser), lane 5 waits although its
    # group's lowest lane committed; `room` cuts the commit at the insertion that makes the set grow
    slot = {0: 7, 1: 1, 2: 2, 3: 4, 4: 4, 5: 7, 6: 9}
    assert _claim(sorted(slot), slot, 32) == ([0, 1, 2, 3], 4)
    assert _claim(sorted(slot), slot, 2) == ([0, 1], 4)
    assert _claim([2, 6], slot, 32) == ([2, 6], 32)
