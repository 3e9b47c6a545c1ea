"""The candidate lists' CPython-set emulation on the device, against CPython's own set.

tests/device_units/cand_units.cu includes the product headers unchanged and runs make_rot_tab / key_hash / tuple_hash6 (pct_rot.cuh,
pct_common.cuh), cand_tuple / cand_hash_c / rot_dims_c (pct_cand_c.cuh), build_candidates<uint16_t / uint32_t> (pct_cand.cuh) one warp
per case in both shared-memory layouts of the step's candidates kernel (the 2048-slot stage in shared memory, and settings 1/3's 128
shared slots with the 2048 stage in a global buffer), PCTC_CANDIDATES_BODY on a CEnv in global memory with the shuffle off and on, and
shuffle_candidates on caller lists.  The inputs are tests/cand_inputs.py's (their reach is asserted by test_candidate_inputs_cpu.py).

For each case the reference is CPython: the tuples EMSPoint adds, in its loop order, go into a real `set`, and `list(s)` must equal the
device's order mapped back to tuples, bit for bit; every device hash must equal `hash()` of its tuple.  At 1229 distinct keys the
emulation stops with PCT_FLAG_CAND_OVERFLOW and returns the 1229 keys in the order of its 2048-slot table (DESIGN section 7); that list
is compared with cand_inputs' setobject model, which the CPU test holds to `list(set(...))` below the limit.
"""
import ctypes as C
import os
import random
import sys

import numpy as np
import pytest

import cand_inputs as ci
from test_shuffle import _expected_order

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "tests", "device_units", "_build", "libcand_units.so")
FLAG_CAND_OVERFLOW = 8
pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(sys.version_info[:2] != (3, 12), reason="the candidate order is CPython 3.12's set order (DESIGN section 6)")]


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(LIB):
        raise RuntimeError("%s is missing: build() (make -C tests/device_units) builds it" % LIB)
    L = C.CDLL(LIB)
    L.cu_cenv_bytes.restype = C.c_size_t
    return L


def _torch():
    return pytest.importorskip("torch")


def _dev(a, dtype):
    return _torch().from_numpy(np.ascontiguousarray(np.asarray(a, dtype=dtype))).cuda()


def _run(fn, *args):
    torch = _torch()
    conv = []
    for a in args:
        if torch.is_tensor(a):
            conv.append(C.c_void_p(a.data_ptr()))
        elif isinstance(a, tuple):  # ("u64", value)
            conv.append(C.c_ulonglong(a[1]) if a[0] == "u64" else C.c_longlong(a[1]))
        else:
            conv.append(C.c_int(a))
    rc = fn(*conv)
    assert rc == 0, "CUDA error %d" % rc


def _u64(a):
    return a.cpu().numpy().view(np.uint64)


def _expected(seq):
    """(ordered tuples, overflow): CPython's list(set(...)) below the limit, the model's 2048-slot order at it"""
    ref = ci.reference_order([t for _, t in seq])
    if len(ref) <= ci.CAND_CAP:
        return ref, False
    order, over, _ = ci.run_device_order(seq, max(r for r, _ in seq) + 1)
    assert over and len(order) == ci.CAND_CAP + 1
    return order, True


# ======================================================== rotation table, hashes ========================================================
def test_rot_tab_matches_the_reference_skip_rules(lib):
    items = [(a, b, c) for a in range(1, 5) for b in range(1, 5) for c in range(1, 5)] + [(255, 255, 1), (16, 1, 16), (17, 17, 17)]
    rows = [(it, R) for it in items for R in (2, 6)]
    out = _torch().zeros((len(rows), 25), dtype=_torch().int32, device="cuda")
    _run(lib.cu_rot_tab, _dev([it for it, _ in rows], np.int32), _dev([R for _, R in rows], np.int32), len(rows), out)
    got = out.cpu().numpy()
    for k, (it, R) in enumerate(rows):
        dims = [tuple(it[ci.PERM[r][c]] for c in range(3)) for r in range(6)]
        valid = sum(1 << r for r in range(6) if r < R and ci.rot_dims_d(it, r)[3])
        assert [tuple(got[k, 3 * r:3 * r + 3]) for r in range(6)] == dims, (it, R)
        assert got[k, 18] == valid, (it, R)
        assert list(got[k, 19:25]) == ci.canon(it, R), (it, R)


def test_tuple_hash6_is_pythons_tuple_hash(lib):
    rng = random.Random(5)
    tuples = []
    for _ in range(20000):
        kind = rng.randrange(3)
        if kind == 0:
            t = tuple(rng.randint(0, 300) for _ in range(6))
        elif kind == 1:
            t = tuple(rng.choice((-1, -2, 0, 2 ** 61 - 2, 2 ** 61, -2 ** 62, rng.randint(-2 ** 63, 2 ** 63))) for _ in range(6))
        else:
            t = tuple(rng.choice((0.0, -0.0, 0.1 + 0.2, 0.3, 1e-6, 2400.0 - 1e-6, rng.uniform(-3000, 3000), 5e-324, 1e300)) for _ in range(6))
        tuples.append(t)
    lanes = np.array([[hash(v) & ci.MASK64 for v in t] for t in tuples], dtype=np.uint64)
    out = _torch().zeros(len(tuples), dtype=_torch().int64, device="cuda")
    _run(lib.cu_tuple_hash6, _dev(lanes.view(np.int64), np.int64), len(tuples), out)
    assert list(_u64(out)) == [ci.uhash(t) for t in tuples]


# =========================================================== discrete ===========================================================
@pytest.fixture(scope="module")
def discrete_runs(lib):
    """every case of cand_inputs.discrete_cases through build_candidates, per key width and layout: {(bits, bigsm): [(case, keys, cnt, flags)]}"""
    torch = _torch()
    cases = ci.discrete_cases()
    res = {}
    for bits in (4, 8):
        sel = [c for c in cases if ci.key_bits(c["cont"]) == bits]
        n = len(sel)
        ems = np.zeros((n, ci.E_MAX, 6), np.int16)
        raw = np.zeros((n, ci.RAW_MAX), np.uint32)
        n_ems, n_raw = np.zeros(n, np.int32), np.full(n, -1, np.int32)
        for k, c in enumerate(sel):
            if c["kind"] == "raw":
                raw[k, :len(c["raw"])] = c["raw"]
                n_raw[k] = len(c["raw"])
            elif c["ems"]:
                ems[k, :len(c["ems"])] = c["ems"]
                n_ems[k] = len(c["ems"])
        args = (_dev(ems, np.int16), _dev(n_ems, np.int32), _dev([c["item"] for c in sel], np.int32), _dev([c["R"] for c in sel], np.int32),
                _dev(raw.view(np.int32), np.int32), _dev(n_raw, np.int32), n)
        for bigsm in (0, 1):
            keys = torch.full((n, ci.TAB_MAX), -1, dtype=torch.int32, device="cuda")
            cnt = torch.zeros(n, dtype=torch.int32, device="cuda")
            flags = torch.zeros(n, dtype=torch.int32, device="cuda")
            big = torch.zeros((n, ci.TAB_MAX), dtype=torch.int32, device="cuda")
            _run(lib.cu_build_d, 16 if bits == 4 else 32, bigsm, *args, keys, cnt, flags, big)
            kk, cc, ff = keys.cpu().numpy().view(np.uint32), cnt.cpu().numpy(), flags.cpu().numpy()
            res[(bits, bigsm)] = [(c, kk[k, :cc[k]].tolist(), int(cc[k]), int(ff[k])) for k, c in enumerate(sel)]
    return res


@pytest.mark.parametrize("bigsm", [1, 0], ids=["2048-stage-shared", "2048-stage-global"])
@pytest.mark.parametrize("bits", [4, 8], ids=["16-bit", "32-bit"])
def test_discrete_order_count_and_flags_equal_cpython(discrete_runs, bits, bigsm):
    runs = discrete_runs[(bits, bigsm)]
    assert len(runs) >= 100
    n_over = 0
    for k, (c, keys, cnt, flags) in enumerate(runs):
        seq, _ = ci.case_sequence(c)
        want, over = _expected(seq)
        n_over += over
        got = [ci.key_tuple(bits, key, c["item"]) for key in keys]
        tag = "case %d (%s, %s, R %d, item %s)" % (k, c["kind"], c["cont"], c["R"], c["item"])
        assert flags == (FLAG_CAND_OVERFLOW if over else 0), tag
        assert cnt == len(want), tag
        assert got == want, tag
        assert keys == [ci.tuple_key(bits, t, c["item"], c["R"]) for t in want], tag + ": keys are not the canonical ones"
    assert n_over >= 2


@pytest.mark.parametrize("bits", [4, 8], ids=["16-bit", "32-bit"])
def test_discrete_key_hash_is_pythons_hash(lib, discrete_runs, bits):
    keys, items, Rs, want = [], [], [], []
    for c, ks, _, _ in discrete_runs[(bits, 1)]:
        for key in ks:
            keys.append(key); items.append(c["item"]); Rs.append(c["R"])
            want.append(ci.uhash(ci.key_tuple(bits, key, c["item"])))
    out = _torch().zeros(len(keys), dtype=_torch().int64, device="cuda")
    _run(lib.cu_key_hash, bits, _dev(np.array(keys, np.uint32).view(np.int32), np.int32), _dev(items, np.int32), _dev(Rs, np.int32), len(keys), out)
    assert len(keys) > 10000
    assert list(_u64(out)) == want


# ========================================================== continuous ==========================================================
def _c_tuple(case, code):
    m = case["ems"][code >> 5]
    sx, sy, sz, _ = ci.rot_dims_c(case["item"], (code >> 2) & 7)
    return ci.corners(m, sx, sy, sz)[code & 3]


SEED, ENV_BASE = 0x1234ABCD, 1000


@pytest.fixture(scope="module")
def continuous_runs(lib):
    """every case of cand_inputs.continuous_cases through PCTC_CANDIDATES_BODY, shuffle off and on: {shuffle: [(case, codes, cnt, flags)]}"""
    torch = _torch()
    cases = ci.continuous_cases()
    n = len(cases)
    off = np.zeros(n + 1, np.int32)
    off[1:] = np.cumsum([len(c["ems"]) for c in cases])
    ems = np.array([m for c in cases for m in c["ems"]], np.float64).reshape(-1, 6)
    draws = np.array([(37 * k) % 500 for k in range(n)], np.int64)
    env = torch.zeros(n * lib.cu_cenv_bytes() // 8 + 2, dtype=torch.float64, device="cuda")
    res = {}
    for shuffle in (0, 1):
        codes = torch.zeros((n, ci.TAB_MAX), dtype=torch.int16, device="cuda")
        cnt = torch.zeros(n, dtype=torch.int32, device="cuda")
        flags = torch.zeros(n, dtype=torch.int32, device="cuda")
        _run(lib.cu_build_c, _dev(ems, np.float64), _dev(off, np.int32), _dev([c["item"] for c in cases], np.float64),
             _dev([c["R"] for c in cases], np.int32), _dev(draws, np.int64), n, env, shuffle, ("u64", SEED), ("ll", ENV_BASE), codes, cnt, flags)
        cc, ff, kk = cnt.cpu().numpy(), flags.cpu().numpy(), codes.cpu().numpy().view(np.uint16)
        res[shuffle] = [(c, kk[k, :cc[k]].tolist(), int(cc[k]), int(ff[k]), int(draws[k])) for k, c in enumerate(cases)]
    res["arrays"] = (ems, off)
    return res


@pytest.mark.parametrize("shuffle", [0, 1], ids=["shuffle-off", "shuffle-on"])
def test_continuous_order_count_and_flags_equal_cpython(continuous_runs, shuffle):
    n_over = 0
    for k, (c, codes, cnt, flags, draw) in enumerate(continuous_runs[shuffle]):
        seq, _ = ci.c_sequence(c)
        want, over = _expected(seq)
        n_over += over
        if shuffle:
            want = [want[i] for i in _expected_order(len(want), SEED, ENV_BASE + k, draw)]
        tag = "case %d (%s, R %d, item %r)" % (k, c["cont"], c["R"], c["item"])
        assert flags == (FLAG_CAND_OVERFLOW if over else 0), tag
        assert cnt == len(want), tag
        got = [_c_tuple(c, code) for code in codes]
        assert [ci.bits_of(t) for t in got] == [ci.bits_of(t) for t in want], tag
    assert n_over >= 1


def test_continuous_tuples_hashes_and_rotations(lib, continuous_runs):
    ems, off = continuous_runs["arrays"]
    runs = continuous_runs[0]
    q_case, q_code = [], []
    for k, (c, codes, _, _, _) in enumerate(runs):
        q_case += [k] * len(codes)
        q_code += codes
        for code in range(0, len(c["ems"]) * 32, 37):  # codes the list does not hold too: every rotation, unfitting EMS
            if (code >> 2) & 7 < 6:
                q_case.append(k); q_code.append(code)
    n = len(q_code)
    torch = _torch()
    tup = torch.zeros((n, 6), dtype=torch.float64, device="cuda")
    hsh = torch.zeros(n, dtype=torch.int64, device="cuda")
    dims = torch.zeros((n, 3), dtype=torch.float64, device="cuda")
    valid = torch.zeros(n, dtype=torch.int32, device="cuda")
    _run(lib.cu_cand_c, _dev(ems, np.float64), _dev(off, np.int32), _dev([c["item"] for c, *_ in runs], np.float64), _dev(q_case, np.int32),
         _dev(q_code, np.int32), n, tup, hsh, dims, valid)
    tup, hsh, dims, valid = tup.cpu().numpy(), _u64(hsh), dims.cpu().numpy(), valid.cpu().numpy()
    assert n > 10000
    for i in range(n):
        c = runs[q_case[i]][0]
        want = _c_tuple(c, q_code[i])
        assert ci.bits_of(tuple(float(v) for v in tup[i])) == ci.bits_of(want), (q_case[i], q_code[i])
        assert int(hsh[i]) == ci.uhash(want), (q_case[i], q_code[i])
        sx, sy, sz, kept = ci.rot_dims_c(c["item"], (q_code[i] >> 2) & 7)
        assert tuple(dims[i]) == (sx, sy, sz) and bool(valid[i]) == kept, (q_case[i], q_code[i])


# =========================================================== shuffle ===========================================================
@pytest.mark.parametrize("bits", [16, 32])
def test_shuffle_candidates_is_the_keyed_permutation(lib, bits):
    torch = _torch()
    rng = random.Random(bits)
    ns = [0, 1, 2, 3, 31, 32, 33, 63, 64, 65, 100, 511, 512, 1000, 1227, 1228] + [rng.randint(0, 1228) for _ in range(240)]
    n_case, out_max = len(ns), ci.TAB_MAX
    dt = np.uint16 if bits == 16 else np.uint32
    lists = np.zeros((n_case, out_max), dt)
    for k, n in enumerate(ns):
        lists[k, :n] = [rng.randrange(1 << bits) for _ in range(n)]
    gid = np.array([rng.randrange(1 << 40) for _ in ns], np.uint64)
    draws = np.array([rng.randrange(1 << 20) for _ in ns], np.uint64)
    seed = rng.randrange(1 << 63)
    sdt = np.int16 if bits == 16 else np.int32
    dl = _dev(lists.view(sdt), sdt)
    keys = torch.zeros((n_case, out_max), dtype=torch.int64, device="cuda")
    tmp = torch.zeros_like(dl)
    _run(lib.cu_shuffle, bits, dl, _dev(ns, np.int32), _dev(gid.view(np.int64), np.int64), _dev(draws.view(np.int64), np.int64), ("u64", seed),
         n_case, keys, tmp)
    got = dl.cpu().numpy().view(dt)
    for k, n in enumerate(ns):
        perm = _expected_order(n, seed, int(gid[k]), int(draws[k]))
        assert got[k, :n].tolist() == [int(lists[k, i]) for i in perm], "n = %d" % n
