"""Inputs for the candidate lists' CPython-set emulation (csrc/pct_cand.cuh, pct_cand_c.cuh, pct_rot.cuh) and a pure-Python model of
CPython 3.12's setobject.c that says what each input reaches.

The tuples are the ones `EMSPoint` adds to `posVec` (D/C space.py), in its loop order: EMS x rotation (with its skip rules) x four corners.
The model follows set_add_entry / set_table_resize / set_insert_clean: tables of 8 slots growing to the smallest power of two above
4 x used when fill x 5 >= mask x 3, a linear window of 9 slots after the home slot unless it would pass the table end, perturb >>= 5.
It runs a sequence the way the device does: in chunks of 32 raw positions (one per lane), each key first looked up read-only in the
table as it stood at the chunk's start, the new ones then inserted in lane order.  That is the same sequence of set operations as
CPython's (the read-only lookup changes nothing), so its final slot order must be `list(set(...))`; test_candidate_inputs_cpu.py checks
this on every input, then asserts floors on what the inputs reach.  The continuous device compares a 16-bit tag (the hash's top bits)
before the tuples; the model counts tag matches between distinct tuples, which CPython never sees as anything but unequal hashes.

Generated inputs are seeded and deterministic; tests/test_gpu_candidate_units.py feeds the same inputs to the device.
"""
import math
import random
import struct

MASK64 = (1 << 64) - 1
E_MAX, RAW_MAX, CE_MAX = 128, 2048, 256
TAB_MAX, CAND_CAP = 2048, 1228  # the emulation's largest table; distinct keys it holds before the next resize would need 4096 slots
PERM = ((0, 1, 2), (1, 0, 2), (0, 2, 1), (1, 2, 0), (2, 0, 1), (2, 1, 0))  # 0 x y z, 1 y x z, 2 x z y, 3 y z x, 4 z x y, 5 z y x


def uhash(t):
    return hash(t) & MASK64


# ============================================= the tuples EMSPoint adds, in its order =============================================
def rot_dims_d(item, rot):
    """(sx, sy, sz, kept): D:space.py's orientation and its skip rule (rot 1/4/5 when sx == sy, rot 2/3 when all three are equal)"""
    sx, sy, sz = (item[PERM[rot][k]] for k in range(3))
    if rot in (1, 4, 5):
        return sx, sy, sz, sx != sy
    if rot in (2, 3):
        return sx, sy, sz, not (sx == sy and sy == sz)
    return sx, sy, sz, True


def rot_dims_c(item, rot):
    """C:space.py: the same with abs(a - b) < 1e-6 for equality"""
    sx, sy, sz = (item[PERM[rot][k]] for k in range(3))
    if rot in (1, 4, 5):
        return sx, sy, sz, not (abs(sx - sy) < 1e-6)
    if rot in (2, 3):
        return sx, sy, sz, not (abs(sx - sy) < 1e-6 and abs(sy - sz) < 1e-6)
    return sx, sy, sz, True


def corners(m, sx, sy, sz):
    """the four tuples of one (EMS, orientation), in posVec.add order"""
    return [(m[0], m[1], m[2], m[0] + sx, m[1] + sy, m[2] + sz),
            (m[3] - sx, m[1], m[2], m[3], m[1] + sy, m[2] + sz),
            (m[0], m[4] - sy, m[2], m[0] + sx, m[4], m[2] + sz),
            (m[3] - sx, m[4] - sy, m[2], m[3], m[4], m[2] + sz)]


def ems_sequence(ems, item, R, continuous):
    """[(raw position, tuple)] in EMSPoint's insertion order; raw position = (ems index x R + rotation) x 4 + corner, the device's lane order"""
    seq = []
    for ei, m in enumerate(ems):
        for rot in range(R):
            sx, sy, sz, kept = (rot_dims_c if continuous else rot_dims_d)(item, rot)
            if not kept:
                continue
            if continuous:
                fits = m[3] - m[0] + 1e-6 >= sx and m[4] - m[1] + 1e-6 >= sy and m[5] - m[2] + 1e-6 >= sz
            else:
                fits = m[3] - m[0] >= sx and m[4] - m[1] >= sy and m[5] - m[2] >= sz
            if fits:
                for q, t in enumerate(corners(m, sx, sy, sz)):
                    seq.append(((ei * R + rot) * 4 + q, t))
    return seq


# ====================================================== discrete keys ======================================================
def canon(item, R):
    """make_rot_tab's canonical index: the lowest rotation with the same oriented sizes"""
    d = [tuple(item[PERM[r][k]] for k in range(3)) for r in range(6)]
    return [min(q for q in range(r + 1) if d[q] == d[r]) for r in range(6)]


def key_bits(container):
    return 4 if max(container) <= 16 else 8


def key_pack(bits, xs, ys, zs, rot):
    return xs | (ys << bits) | (zs << (2 * bits)) | (rot << (3 * bits))


def key_tuple(bits, key, item):
    m = (1 << bits) - 1
    xs, ys, zs, rot = key & m, (key >> bits) & m, (key >> 2 * bits) & m, (key >> 3 * bits) & 7
    sx, sy, sz = (item[PERM[rot][k]] for k in range(3))
    return (xs, ys, zs, xs + sx, ys + sy, zs + sz)


def tuple_key(bits, t, item, R):
    """the key of a tuple: its rotation is the canonical one of its oriented sizes"""
    c = canon(item, R)
    size = (t[3] - t[0], t[4] - t[1], t[5] - t[2])
    rot = next(c[r] for r in range(6) if tuple(item[PERM[r][k]] for k in range(3)) == size)
    return key_pack(bits, t[0], t[1], t[2], rot)


# ================================================ the setobject.c model ================================================
class SetModel:
    """set_add_entry / set_table_resize / set_insert_clean of CPython 3.12 (no deletions, so no dummies); `cap`: the emulation's table
    limit, beyond which it stops with the overflow flag instead of resizing"""

    def __init__(self, stats, cap=TAB_MAX):
        self.tab = [None] * 8  # (key, hash)
        self.mask, self.fill, self.cap, self.overflow = 7, 0, cap, False
        self.st = stats

    def _probe(self, key, h, phase):
        """walk the probe sequence of (key, h): returns (slot index of key or of the first empty slot, found)"""
        tab, mask, st = self.tab, self.mask, self.st
        perturb, i, steps = h, h & mask, 0
        while True:
            n = 9 if i + 9 <= mask else 0
            if n == 0 and tab[i] is not None:
                st["wrap"] += 1
            for j in range(n + 1):
                e = tab[i + j]
                if e is None:
                    st["perturb_max"] = max(st["perturb_max"], steps)
                    st["perturb2"] += steps >= 2
                    st["window"] += j > 0
                    return i + j, False
                if e[1] >> 48 == h >> 48 and e[0] != key:
                    st["tag_" + phase] += 1
                    st["tag_" + phase + "_same_hash"] += e[1] == h
                if e[1] == h and e[0] == key:
                    st["window"] += j > 0
                    return i + j, True
            perturb >>= 5
            i = (i * 5 + 1 + perturb) & mask
            steps += 1

    def lookup(self, key, h):
        return self._probe(key, h, "probe")[1]

    def add(self, key, h):
        """returns (inserted, resized)"""
        s, found = self._probe(key, h, "insert")
        if found:
            return False, False
        self.tab[s] = (key, h)
        self.fill += 1
        if self.fill * 5 < self.mask * 3:
            return True, False
        newsize = 8
        while newsize <= self.fill * 4:
            newsize <<= 1
        if newsize > self.cap:
            self.overflow = True
            return True, True
        old = self.tab
        self.tab, self.mask = [None] * newsize, newsize - 1
        for e in old:  # set_insert_clean in slot order
            if e is not None:
                perturb, i = e[1], e[1] & self.mask
                while True:
                    n = 9 if i + 9 <= self.mask else 0
                    j = next((j for j in range(n + 1) if self.tab[i + j] is None), None)
                    if j is not None:
                        self.tab[i + j] = e
                        break
                    perturb >>= 5
                    i = (i * 5 + 1 + perturb) & self.mask
        return True, True

    def order(self):
        return [e[0] for e in self.tab if e is not None]


def new_stats():
    st = {k: 0 for k in ("wrap", "perturb2", "perturb_max", "window", "tag_probe", "tag_insert", "tag_probe_same_hash", "tag_insert_same_hash",
                         "tag_insert_same_chunk", "dup_in_chunk", "dup_in_chunk_lane0", "dup_in_chunk_lane31", "dup_across_chunks")}
    st["resizes"] = []  # (fill, lane, pending staged keys after it in the chunk)
    return st


def run_device_order(seq, n_raw, stats=None):
    """Run [(raw position, tuple)] as the device does (chunks of 32 raw positions, read-only lookup, first occurrences in lane order).
    Returns (ordered tuples, overflow, stats)."""
    st = stats if stats is not None else new_stats()
    model = SetModel(st)
    by_chunk = {}
    for r, t in seq:
        by_chunk.setdefault(r // 32, []).append((r, t))
    for base in range(0, n_raw, 32):
        chunk = by_chunk.get(base // 32, [])
        first = {}
        for r, t in chunk:
            if t in first:
                st["dup_in_chunk"] += 1
                st["dup_in_chunk_lane0"] += first[t] % 32 == 0
                st["dup_in_chunk_lane31"] += r % 32 == 31
            else:
                first[t] = r
        staged = []
        for r, t in chunk:
            if first[t] != r:
                continue
            if model.lookup(t, uhash(t)):
                st["dup_across_chunks"] += 1
            else:
                staged.append((r, t))
        in_chunk = set()
        for k, (r, t) in enumerate(staged):
            before = st["tag_insert"]
            ins, resized = model.add(t, uhash(t))
            if st["tag_insert"] > before and any(uhash(u) >> 48 == uhash(t) >> 48 for u in in_chunk):
                st["tag_insert_same_chunk"] += 1
            in_chunk.add(t)
            if resized:
                st["resizes"].append((model.fill, r % 32, len(staged) - k - 1))
            if model.overflow:
                return model.order(), True, st
    return model.order(), False, st


def reference_order(tuples):
    """CPython's own order"""
    return list(set(tuples))


# ================================================ discrete inputs ================================================
CONTAINERS_D = ((10, 10, 10), (16, 16, 16), (17, 16, 16), (255, 255, 255), (20, 18, 24))
SHAPES = ("xyz", "x=y", "y=z", "x=z", "x=y=z")


def _item_d(rng, shape, top):
    a, b, c = (rng.randint(1, top) for _ in range(3))
    if shape == "x=y": b = a
    elif shape == "y=z": c = b
    elif shape == "x=z": c = a
    elif shape == "x=y=z": b = c = a
    return (a, b, c)


def _ems_d(rng, cont, item, exact):
    W, L, H = cont
    while True:
        x0, y0, z0 = rng.randrange(W), rng.randrange(L), rng.randrange(H)
        if rng.random() < exact:  # a side of the EMS equal to a side of the item: corners coincide
            sx, sy = rng.choice(item), rng.choice(item)
            x1 = min(W, x0 + sx if rng.random() < 0.6 else rng.randint(x0 + 1, W))
            y1 = min(L, y0 + sy if rng.random() < 0.6 else rng.randint(y0 + 1, L))
        else:
            x1, y1 = rng.randint(x0 + 1, W), rng.randint(y0 + 1, L)
        return [x0, y0, z0, x1, y1, H]


def discrete_case(seed):
    """one random EMS-mode case: container, item, R, EMS list"""
    rng = random.Random(1000003 * seed + 17)
    cont = CONTAINERS_D[seed % len(CONTAINERS_D)]
    R = 6 if rng.random() < 0.6 else 2
    shape = SHAPES[(seed // len(CONTAINERS_D)) % len(SHAPES)]
    top = max(1, min(cont) // rng.choice((2, 3, 5)))
    item = _item_d(rng, shape, top)
    n = rng.choice((1, 2, 3, 5, 8, 13, 21, 40, 80, 128))
    exact = rng.choice((0.0, 0.3, 0.8))
    ems = [_ems_d(rng, cont, item, exact) for _ in range(n)]
    return dict(kind="ems", cont=cont, item=item, R=R, ems=ems)


def _grow_to(rng, case, target, draw, continuous):
    """append EMS drawn by `draw` until the case holds exactly `target` distinct tuples (an EMS that would pass it is not taken; after
    many misses the last EMS is taken back)"""
    seen, added = set(), []
    for m in case["ems"]:
        added.append(set(t for _, t in ems_sequence([m], case["item"], case["R"], continuous)) - seen)
        seen |= added[-1]
    misses = 0
    while len(seen) != target:
        m = _ems_fit(rng, case["cont"], case["item"], continuous) if target - len(seen) < 24 and rng.random() < 0.5 else draw()
        new = set(t for _, t in ems_sequence([m], case["item"], case["R"], continuous)) - seen
        if new and len(seen) + len(new) <= target and len(case["ems"]) < (CE_MAX if continuous else E_MAX):
            case["ems"].append(m)
            added.append(new)
            seen |= new
            misses = 0
        else:
            misses += 1
            if misses > 300 and case["ems"]:
                case["ems"].pop()
                seen -= added.pop()
                misses = 0
    return case


def _ems_fit(rng, cont, item, continuous):
    """an EMS of exactly one orientation's sizes: its four corners coincide, so it adds one tuple (or a few, where rounding parts them)"""
    sx, sy, sz = (item[k] for k in PERM[rng.randrange(6)])
    if continuous:
        x0, y0, z0 = (round(rng.uniform(0, v * 0.8), 3) for v in cont)
    else:
        x0, y0, z0 = (rng.randrange(max(1, v - 15)) for v in cont)
    return [x0, y0, z0, x0 + sx, y0 + sy, z0 + sz]


def discrete_sized_case(seed, target):
    """an EMS-mode case with exactly `target` distinct tuples (E_MAX EMS at most; 6 orientations of an item with three distinct sides)"""
    rng = random.Random(7919 * seed + target)
    if seed % 2:
        cont, item = (255, 255, 255), (rng.randint(1, 5), rng.randint(6, 9), rng.randint(10, 14))
    else:  # 16-bit keys
        cont, item = (16, 16, 16), (1, 2, 3)
    case = dict(kind="ems", cont=cont, item=item, R=6, ems=[])
    return _grow_to(rng, case, target, lambda: _ems_d(rng, cont, item, 0.0), False)


def raw_case(seed):
    """a raw key sequence (the EV / EP / CP / FC path): keys drawn from a pool with many repeats, repeats placed at lanes 0 and 31"""
    rng = random.Random(4099 * seed + 5)
    cont = CONTAINERS_D[seed % len(CONTAINERS_D)]
    bits = key_bits(cont)
    R = 6 if seed % 3 else 2
    item = _item_d(rng, SHAPES[seed % len(SHAPES)], max(1, min(cont) // 3))
    c = canon(item, R)
    rots = sorted(set(c[r] for r in range(R) if rot_dims_d(item, r)[3]))
    pool_n = rng.choice((3, 30, 300, 1000, 1300))
    pool = set()
    for _ in range(4 * pool_n):
        if len(pool) == pool_n:
            break
        rot = rng.choice(rots)
        sx, sy, sz = (item[PERM[rot][k]] for k in range(3))
        W, L, H = cont
        if sx > W or sy > L or sz > H:
            continue
        pool.add(key_pack(bits, rng.randint(0, W - sx), rng.randint(0, L - sy), rng.randint(0, H - sz), rot))
    pool = sorted(pool)
    n = rng.randint(1, RAW_MAX)
    seq = [rng.choice(pool) for _ in range(n)] if pool else []
    for b in range(0, len(seq) - 32, 32):  # a key repeated at lane 31 of its chunk, a lane-0 key repeated later in its chunk
        if rng.random() < 0.3:
            seq[b + 31] = seq[b + rng.randrange(31)]
        if rng.random() < 0.3:
            seq[b + rng.randint(1, 31)] = seq[b]
    return dict(kind="raw", cont=cont, item=item, R=R, raw=seq)


def raw_sized_case(target, cont):
    """a raw sequence with exactly `target` distinct keys, each repeated (<= RAW_MAX keys in all)"""
    rng = random.Random(target * 31 + cont[0])
    item, R = (3, 5, 7), 6
    bits = key_bits(cont)
    c = canon(item, R)
    keys = set()
    while len(keys) < target:
        rot = c[rng.randrange(6)]
        keys.add(key_pack(bits, rng.randint(0, cont[0] - 7), rng.randint(0, cont[1] - 7), rng.randint(0, cont[2] - 7), rot))
    keys = sorted(keys)
    rng.shuffle(keys)
    seq = list(keys)
    while len(seq) < RAW_MAX:
        seq.insert(rng.randrange(len(seq) + 1), rng.choice(keys))
    return dict(kind="raw", cont=cont, item=item, R=R, raw=seq)


def raw_resize_case(fill, lane, cont):
    """a raw sequence whose `fill`-th distinct key (a resize threshold) sits on `lane` of its chunk, with new keys staged after it on the
    lanes above and repeats of the first key everywhere else"""
    base = raw_sized_case(fill + 40, cont)["raw"]
    keys = list(dict.fromkeys(base))
    p = fill - 1
    while p % 32 != lane:
        p += 1
    seq = keys[:fill - 1] + [keys[0]] * (p - fill + 1) + [keys[fill - 1]]
    seq += keys[fill:fill + 31 - lane] + keys[:8]
    return dict(kind="raw", cont=cont, item=(3, 5, 7), R=6, raw=seq)


def case_sequence(case):
    """[(raw position, tuple)] and the number of raw positions of a discrete case"""
    if case["kind"] == "raw":
        bits = key_bits(case["cont"])
        return [(r, key_tuple(bits, k, case["item"])) for r, k in enumerate(case["raw"])], len(case["raw"])
    return ems_sequence(case["ems"], case["item"], case["R"], False), len(case["ems"]) * case["R"] * 4


N_RANDOM_D, N_RAW = 400, 60
EXTRA_D = (491, 571)  # discrete_case seeds past N_RANDOM_D whose 307th key lands on lane 0 (searched; the CPU test asserts it)
SIZED_D = (1, 4, 5, 6, 18, 19, 20, 76, 77, 78, 306, 307, 308, 1227, 1228, 1229, 1300)


def discrete_cases():
    cases = [discrete_case(s) for s in list(range(N_RANDOM_D)) + list(EXTRA_D)]
    cases += [discrete_sized_case(s, t) for t in SIZED_D for s in (0, 1)]  # 16-bit and 32-bit keys
    cases += [raw_case(s) for s in range(N_RAW)]
    cases += [raw_sized_case(t, cont) for t in (1228, 1229) for cont in ((16, 16, 16), (255, 255, 255))]
    cases += [raw_resize_case(f, lane, cont) for f in (5, 19, 77, 307) for lane in (0, 13, 31) for cont in ((16, 16, 16), (255, 255, 255))]
    cases.append(dict(kind="ems", cont=(10, 10, 10), item=(2, 3, 4), R=6, ems=[]))  # empty EMS list
    cases.append(dict(kind="raw", cont=(10, 10, 10), item=(2, 3, 4), R=6, raw=[]))  # empty raw sequence
    return cases


# ================================================ continuous inputs ================================================
BINS_C = ((1.0, 1.0, 1.0), (1.2, 0.8, 1.0), (10.0, 10.0, 10.0), (2400.0, 1700.0, 2300.0))


def _item_c(rng, cont, mode):
    s = min(cont)
    a, b, c = (round(rng.uniform(0.1, 0.5) * s, rng.choice((1, 2, 6, 17))) for _ in range(3))
    if mode == "apart":  # sides 0, 5e-7, 1e-6 and 2e-6 apart, on each pair of axes
        d = rng.choice((0.0, 5e-7, 1e-6, 2e-6, 1e-6 + 1e-12, 1e-6 - 1e-12))
        pair = rng.randrange(4)
        if pair == 0: b = a + d
        elif pair == 1: c = b + d
        elif pair == 2: c = a + d
        else: b = a + d; c = a + rng.choice((0.0, d, -d))
    return (a, b, c)


def _ems_c(rng, cont, item, mode):
    W, L, H = cont
    x0, y0, z0 = (round(rng.uniform(0, v * 0.9), rng.choice((1, 3, 6, 17))) for v in (W, L, H))
    if mode == "exact":  # width exactly a side: corners 0 / 1 (2 / 3) give equal tuples from different codes
        x1, y1 = x0 + rng.choice(item), y0 + rng.choice(item)
    elif mode == "edge":  # width at side - 1e-6 and an ulp or two either side: the fit test's boundary
        sx, sy = rng.choice(item), rng.choice(item)
        x1, k = x0 + (sx - 1e-6), rng.randint(-2, 2)
        for _ in range(abs(k)):
            x1 = math.nextafter(x1, math.inf if k > 0 else -math.inf)
        y1 = y0 + (sy - 1e-6) if rng.random() < 0.5 else rng.uniform(y0, L)
    elif mode == "decimal":  # widths equal to a side in decimal but not in binary
        x0 = rng.choice((0.1, 0.2, 0.7, 1.1))
        x1 = x0 + rng.choice(item)
        x1 = float(repr(x1)[:8]) if rng.random() < 0.5 else x1
        y1 = rng.uniform(y0, L)
    else:
        x1, y1 = rng.uniform(x0, W), rng.uniform(y0, L)
    return [x0, y0, z0, min(x1, 2 * W), min(y1, 2 * L), H]


def continuous_case(seed):
    rng = random.Random(1000033 * seed + 3)
    cont = BINS_C[seed % len(BINS_C)]
    R = 6 if rng.random() < 0.6 else 2
    imode = "apart" if seed % 3 == 0 else "plain"
    item = _item_c(rng, cont, imode)
    n = rng.choice((1, 2, 3, 6, 10, 20, 40, 60))
    modes = rng.choice((("plain",), ("exact", "plain"), ("edge", "plain"), ("decimal", "exact")))
    ems = [_ems_c(rng, cont, item, rng.choice(modes)) for _ in range(n)]
    if seed % 7 == 0 and ems:  # value-equal coordinates: -0.0 next to 0.0, 0.1 + 0.2 next to 0.3 (unequal, like every binary neighbour)
        m = list(ems[0])
        m[0], m[1] = 0.0, -0.0
        ems.append(m)
        ems.append([-0.0, 0.0] + m[2:])
        ems.append([0.1 + 0.2, 0.3] + m[2:])
        ems.append([0.3, 0.1 + 0.2] + m[2:])
    return dict(cont=cont, item=item, R=R, ems=ems)


def continuous_sized_case(seed, target):
    rng = random.Random(104729 * seed + target)
    cont = BINS_C[seed % len(BINS_C)]
    s = min(cont)
    item = (0.11 * s, 0.23 * s, 0.37 * s)
    case = dict(cont=cont, item=item, R=6, ems=[])
    return _grow_to(rng, case, target, lambda: _ems_c(rng, cont, item, rng.choice(("plain", "exact"))), True)


# seeds of continuous_case whose lists hold tag matches between distinct tuples (found by searching seeds 0 ..; the CPU test asserts the
# matches are still there, so this list cannot go stale)
TAG_SEEDS = (1008, 2881, 4028, 4387, 8962, 16839)
N_RANDOM_C = 300
SIZED_C = (5, 19, 77, 307, 1228, 1229)


def continuous_cases():
    cases = [continuous_case(s) for s in range(N_RANDOM_C)]
    cases += [continuous_case(s) for s in TAG_SEEDS]
    cases += [continuous_sized_case(s, t) for s, t in enumerate(SIZED_C)]
    cases.append(dict(cont=(1.0, 1.0, 1.0), item=(0.2, 0.3, 0.4), R=6, ems=[]))
    return cases


def c_sequence(case):
    return ems_sequence(case["ems"], case["item"], case["R"], True), len(case["ems"]) * case["R"] * 4


def bits_of(t):
    return tuple(struct.unpack("<Q", struct.pack("<d", v))[0] for v in t)
