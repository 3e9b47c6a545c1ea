"""CPU: the reference's item overrides (tests/golden/items_s*.npz / citems_s*.npz, made by tests/golden/make_item_golden.py) equal stream
items at those draws.  The oracle runs each record's EFFECTIVE stream (the override written into the stream position of the item it
replaced) and must reproduce every observation the policy saw, every reward, done and counter, and every observation after a step.

The observation a step returns shows the source's next item, recorded before the caller overrode it; it is compared where that draw was
not overridden.  This also covers the one documented difference (include/pct_b200.h, pct_set_items): after a FAILED step at an override,
the reference's terminal observation re-reads the source's head, the replaced item, while an env whose item was overridden keeps it."""
import glob
import os

import numpy as np
import pytest

from pct_oracle import OracleContinuous, OracleDiscrete

G = os.path.join(os.path.dirname(__file__), "golden")
GOLD = sorted(glob.glob(os.path.join(G, "items_s*.npz"))) + sorted(glob.glob(os.path.join(G, "citems_s*.npz")))


def effective_stream(g):
    s = g["stream"].copy()
    for t in np.nonzero(g["override"])[0]:
        s[int(g["draw"][t])] = g["item"][t]
    return s


def test_item_goldens_present():
    assert len(GOLD) == 6


@pytest.mark.parametrize("path", GOLD, ids=[os.path.basename(p) for p in GOLD])
def test_oracle_replays_overrides_as_stream_items(path):
    g = np.load(path)
    setting, continuous = int(g["setting"]), os.path.basename(path).startswith("c")
    env = (OracleContinuous if continuous else OracleDiscrete)(setting, stream=effective_stream(g))
    o = env.reset()
    overridden = {int(g["draw"][t]) for t in np.nonzero(g["override"])[0]}
    compared = differences = n_done = 0
    for t in range(len(g["rows"])):
        assert np.array_equal(o, g["seen"][t]), "observation seen at step %d (override=%s)" % (t, bool(g["override"][t]))
        o, r, d, info = env.step(g["rows"][t])
        assert r == g["reward"][t] and d == bool(g["done"][t]) and info["counter"] == g["counter"][t], t
        if d:
            assert info["ratio"] == g["ratio"][t]
        if d:
            term = g["terminal"][n_done]
            n_done += 1
            if int(g["draw"][t]) not in overridden:  # a terminal observation shows the source's head
                assert np.array_equal(o, term), "terminal observation of step %d" % t
                compared += 1
            if g["override"][t]:  # the documented difference: the reference's terminal observation shows the replaced item
                replaced = g["stream"][int(g["draw"][t])][:3]
                assert list(term[-6:-3]) == sorted(replaced if continuous else np.trunc(replaced)), t
                differences += 1
            o = env.reset()
        if int(g["draw"][t]) + 1 not in overridden:  # the observation a step (and a reset after it) leaves shows the next draw
            assert np.array_equal(o, g["after"][t]), "observation after step %d" % t
            compared += 1
    assert g["override"].sum() > len(g["rows"]) // 3 and g["done"].sum() >= 5 and compared > len(g["rows"]) // 4
    assert differences >= 1  # the records contain failed steps at overrides
