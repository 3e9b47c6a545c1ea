"""CPU: the row-selection rule of the opt-in delta observation writes (csrc/pct_discrete.cu write_obs_delta, PCT_B200_OBS_DELTA=1),
restated in numpy and run over oracle trajectories with episode ends and resets: a buffer that only ever receives the rows the rule
selects must equal the full observation after every step — including when the buffer is swapped for one full of garbage (the host
then resets the row counts to "all", begin_obs / pct_fill_prev_kernel in csrc/pct_api.cu).  This checks the algorithm and its
invariant (rows at or above the stored counts are all-zero), not the CUDA code; tests/test_zzz_gpu_obs_delta.py does that on an H100."""
import numpy as np
import pytest

from harness import make_stream, policy_pick
from pct_oracle import OracleDiscrete

NB, NL = 80, 50


def delta_write(buf, prev, full):
    """one write_obs_delta call: buf / full are (NB + NL + 1, 9); prev = [internal rows, leaf rows] that may be non-zero in buf"""
    n_box = int((full[:NB, 8] == 1).sum()) if full[0, :6].any() or full[1:NB, 8].any() else 0  # row 0 carries its flag even when empty
    n_leaf = int((full[NB:NB + NL, 8] == 1).sum())
    pb, pl = min(prev[0], NB), min(prev[1], NL)
    wb, wl = max(n_box, pb, 1), max(n_leaf, pl)
    buf[:wb] = full[:wb]
    buf[NB:NB + wl] = full[NB:NB + wl]
    buf[NB + NL] = full[NB + NL]
    prev[0], prev[1] = max(n_box, 1), n_leaf
    return wb + wl + 1


@pytest.mark.parametrize("setting", [1, 2, 3])
def test_delta_rule_reproduces_full_observation(setting):
    seed = 70 + setting
    env = OracleDiscrete(setting, stream=make_stream(seed, 0, 600, setting))
    rng = np.random.default_rng(1)
    buf, prev = rng.normal(size=(NB + NL + 1, 9)), [NB, NL]  # a fresh buffer: garbage, counts = all rows
    o = env.reset()
    rows_written, episodes = [], 0
    for t in range(400):
        full = o.reshape(NB + NL + 1, 9)
        rows_written.append(delta_write(buf, prev, full))
        assert np.array_equal(buf, full), "step %d" % t
        assert not buf[prev[0]:NB].any() and not buf[NB + prev[1]:NB + NL].any()  # the invariant the next call relies on
        if t % 97 == 96:  # the caller switches to another buffer: the host resets the counts
            buf, prev = rng.normal(size=(NB + NL + 1, 9)), [NB, NL]
        _, row = policy_pick(o, NB, NL, seed, 0, t)
        o, r, d, info = env.step(row)
        if d:  # auto-reset semantics: the next observation written is the reset one
            o = env.reset()
            episodes += 1
    assert episodes >= 8
    assert np.mean(rows_written) < 0.45 * (NB + NL + 1)  # the point of the exercise: well under half of the 131 rows per step
