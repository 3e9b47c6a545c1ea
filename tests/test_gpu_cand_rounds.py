"""The claim rounds of the candidate lists' set emulation on the device, on the adversarial inputs of test_cand_rounds_cpu.py.

The raw key sequences whose chunks gather keys of shared home slots go through build_candidates (tests/device_units/cand_units.cu,
cu_build_d) with 16-bit and 32-bit keys, with the 2048-slot stage in shared memory and in a global buffer; the EMS lists full of
value-equal tuples from different codes go through PCTC_CANDIDATES_BODY (cu_build_c).  Each list must equal CPython's `list(set(...))`
of the same tuples bit for bit, as in test_gpu_candidate_units.py (at the 1229-key stop: the serial model's order and the overflow flag).
"""
import sys

import numpy as np
import pytest

import cand_inputs as ci
import test_cand_rounds_cpu as rounds
from test_gpu_candidate_units import FLAG_CAND_OVERFLOW, _c_tuple, _dev, _expected, _run, _torch, lib  # noqa: F401  (lib: the fixture)

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(sys.version_info[:2] != (3, 12), reason="the candidate order is CPython 3.12's set order (DESIGN section 6)")]


@pytest.mark.parametrize("bigsm", [1, 0], ids=["2048-stage-shared", "2048-stage-global"])
@pytest.mark.parametrize("bits", [4, 8], ids=["16-bit", "32-bit"])
def test_colliding_raw_keys_equal_cpython(lib, bits, bigsm):
    torch = _torch()
    sel = [c for c in rounds.adversarial_cases() if ci.key_bits(c["cont"]) == bits]
    n = len(sel)
    assert n == rounds.N_COLLIDE
    raw = np.zeros((n, ci.RAW_MAX), np.uint32)
    for k, c in enumerate(sel):
        raw[k, :len(c["raw"])] = c["raw"]
    keys = torch.full((n, ci.TAB_MAX), -1, dtype=torch.int32, device="cuda")
    cnt = torch.zeros(n, dtype=torch.int32, device="cuda")
    flags = torch.zeros(n, dtype=torch.int32, device="cuda")
    big = torch.zeros((n, ci.TAB_MAX), dtype=torch.int32, device="cuda")
    _run(lib.cu_build_d, 16 if bits == 4 else 32, bigsm, _dev(np.zeros((n, ci.E_MAX, 6)), np.int16), _dev(np.zeros(n), np.int32),
         _dev([c["item"] for c in sel], np.int32), _dev([c["R"] for c in sel], np.int32), _dev(raw.view(np.int32), np.int32),
         _dev([len(c["raw"]) for c in sel], np.int32), n, keys, cnt, flags, big)
    kk, cc, ff = keys.cpu().numpy().view(np.uint32), cnt.cpu().numpy(), flags.cpu().numpy()
    for k, c in enumerate(sel):
        seq, _ = ci.case_sequence(c)
        want, over = _expected(seq)
        got = [ci.key_tuple(bits, int(key), c["item"]) for key in kk[k, :cc[k]]]
        assert int(ff[k]) == (FLAG_CAND_OVERFLOW if over else 0), "case %d" % k
        assert got == want, "case %d" % k


def test_equal_tuples_equal_cpython(lib):
    torch = _torch()
    cases = rounds.adversarial_continuous_cases()
    n = len(cases)
    off = np.zeros(n + 1, np.int32)
    off[1:] = np.cumsum([len(c["ems"]) for c in cases])
    ems = np.array([m for c in cases for m in c["ems"]], np.float64).reshape(-1, 6)
    env = torch.zeros(n * lib.cu_cenv_bytes() // 8 + 2, dtype=torch.float64, device="cuda")
    codes = torch.zeros((n, ci.TAB_MAX), dtype=torch.int16, device="cuda")
    cnt = torch.zeros(n, dtype=torch.int32, device="cuda")
    flags = torch.zeros(n, dtype=torch.int32, device="cuda")
    _run(lib.cu_build_c, _dev(ems, np.float64), _dev(off, np.int32), _dev([c["item"] for c in cases], np.float64),
         _dev([c["R"] for c in cases], np.int32), _dev(np.zeros(n), np.int64), n, env, 0, ("u64", 0), ("ll", 0), codes, cnt, flags)
    cc, ff, kk = cnt.cpu().numpy(), flags.cpu().numpy(), codes.cpu().numpy().view(np.uint16)
    for k, c in enumerate(cases):
        seq, _ = ci.c_sequence(c)
        want, over = _expected(seq)
        got = [_c_tuple(c, int(code)) for code in kk[k, :cc[k]]]
        assert int(ff[k]) == (FLAG_CAND_OVERFLOW if over else 0), "case %d" % k
        assert [ci.bits_of(t) for t in got] == [ci.bits_of(t) for t in want], "case %d" % k
