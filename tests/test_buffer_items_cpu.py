"""CPU: item preview and item override of the buffered env on the oracle (ItemsOracle.preview / set_items, tests/buffer_items.py), which
tests/test_gpu_buffer_items.py holds pct_buffer_preview_items / pct_buffer_set_items against.

- Identity: set_items with the env's own buffer changes nothing (observation, counts, flags).
- Stream twin: overriding slot j with X at step t gives, from t on, the observations of a twin whose stream holds X at the draw position
  that filled slot j (tracked by the refill rule on a position array; trajectories shorter than the stream, so no position is reused).
- Preview: preview(k) is what the next k placing steps put into the slots they empty.
Both domains, settings 1-3, B in {1, 3, 16}, and a discrete bin under the CP leaf scheme.
"""
import numpy as np
import pytest

from buffer_items import ItemsOracle
from buffer_oracle import config, refill

PSEED = 61
CFGS = [(nm, B) for nm in ("d1", "d2", "d3", "c1", "c2", "c3") for B in (1, 3, 16)] + [("cp_big_s1", 3), ("ep_big_s2", 3)]
IDS = ["%s-B%d" % c for c in CFGS]


def _steps(B):
    return 12 if B == 16 else 30


def _flat_slot(f, B, nl):
    return f // nl if 0 <= f < B * nl else 0


@pytest.mark.parametrize("name,B", CFGS, ids=IDS)
def test_identity(name, B):
    c, mk = config(name, 64 if B == 16 else 50)
    m = ItemsOracle(c, mk(5, 0, 400), B)
    m.reset()
    for t in range(_steps(B)):
        obs, nl, nc, fl, sticky = m.obs.copy(), m.n_leaf.copy(), m.n_cand.copy(), m.slot_fl.copy(), m.sticky
        obs2, rec = m.set_items(m.buf.copy())
        assert np.array_equal(obs2.view(np.uint64), obs.view(np.uint64)), t
        assert np.array_equal(m.n_leaf, nl) and np.array_equal(m.n_cand, nc) and np.array_equal(m.slot_fl, fl) and m.sticky == sticky, t
        assert (rec["n_leaf"], rec["n_cand"], rec["flags"]) == (int(nl.sum()), int(nc.sum()), sticky), t
        m.step(m.policy(PSEED, 0, t))


@pytest.mark.parametrize("name,B", CFGS, ids=IDS)
def test_stream_twin(name, B):
    c, mk = config(name, 64 if B == 16 else 50)
    L, T = 400, _steps(B)
    st, other = mk(7, 1, L), mk(9, 2, L)
    t0 = T // 2
    rng = np.random.RandomState(B)
    A = ItemsOracle(c, st, B)
    A.reset()
    ids = np.arange(L, dtype=np.float64)[:, None].repeat(4, 1)
    posbuf = np.zeros((B, 4))
    pos = refill(posbuf, 0, ids, True, 0)
    flats, obs = [], []
    for t in range(T):
        if t == t0:
            j = rng.randint(B)
            X = other[rng.randint(L)]
            p = int(posbuf[j, 0])
            buf = A.buf.copy()
            buf[j] = X
            obs.append(A.set_items(buf)[0].copy())
        f = A.policy(PSEED, 0, t)
        _, _, d, _ = A.step(f)
        flats.append(f)
        if t >= t0:
            obs.append(A.obs.copy())
        pos = refill(posbuf, pos, ids, d, _flat_slot(f, B, c["nl"]))
    assert pos < L
    twin = st.copy()
    twin[p] = X
    Z = ItemsOracle(c, twin, B)
    Z.reset()
    for t in range(T):
        if t == t0:
            assert np.array_equal(Z.obs.view(np.uint64), obs[0].view(np.uint64)), "the override"
        Z.step(flats[t])
        if t >= t0:
            assert np.array_equal(Z.obs.view(np.uint64), obs[t - t0 + 1].view(np.uint64)), t


@pytest.mark.parametrize("name,B", CFGS, ids=IDS)
def test_preview(name, B):
    c, mk = config(name, 64 if B == 16 else 50)
    m = ItemsOracle(c, mk(11, 3, 400), B)
    m.reset()
    k, checked = 4, 0
    for t0 in range(0, 2 * _steps(B), k):
        pv = m.preview(k)
        got = []
        for t in range(t0, t0 + k):
            f = m.policy(PSEED, 0, t)
            _, _, d, _ = m.step(f)
            if d:  # the reset refilled the buffer: the rest of this preview is stale
                break
            got.append(m.buf[_flat_slot(f, B, c["nl"])].copy())
        assert np.array_equal(np.array(got).reshape(-1, 4), pv[:len(got)]), t0
        checked += len(got)
    assert checked >= _steps(B) // 2
