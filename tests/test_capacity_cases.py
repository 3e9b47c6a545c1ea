"""The capacity cases of tests/golden/capacity_cases.npz (made by tests/golden/make_capacity_cases.py) still do what they are named for:
every expectation the GPU test relies on (t*, the flag bits, the peaks before t*) is re-derived here from the oracle, so the fixture
cannot go stale.  Each case reports the boundary it reaches (its peak counts against the capacities, or t*): in every assertion message,
and for passing cases in the captured output that `pytest -rP` (or -s) shows."""
import pytest

from harness import CAPS, capacity_trace, load_capacity_cases

CASES = load_capacity_cases()


@pytest.mark.parametrize("name", sorted(CASES))
def test_capacity_case(name):
    c = CASES[name]
    tr = capacity_trace(c)
    caps = {k: cap for k, (_, cap) in CAPS[c["domain"]].items()}
    caps["boxes"] = c["nb"]
    reached = "%s: %s; peaks before it: %s" % (
        name, "t* = %d (flag %d, counts %s)" % (tr["t_star"], tr["flag"], tr["star"]) if tr["t_star"] >= 0 else "no flag in %d steps" % tr["n_steps"],
        ", ".join("%s %d/%d" % (k, v, caps[k]) for k, v in sorted(tr["peak"].items()) if k in caps))
    print(reached)
    assert tr["reset_flags"] == 0, "the first observation already crosses a capacity: " + reached
    assert (tr["t_star"], tr["flag"], tr["n_steps"]) == (c["t_star"], c["flag"], c["n_steps"]), reached
    assert tr["peak"] == c["peak"], reached
    if c["flag"]:
        assert bin(c["flag"]).count("1") == 1, "one capacity at a time: " + reached
    else:
        assert tr["done"] or tr["n_steps"] == c["steps"], reached
    for k, (lo, hi) in c["require"].items():
        assert lo <= tr["peak"][k] <= hi, "%s peak not in [%d, %d]: %s" % (k, lo, hi, reached)
    for k, (lo, hi) in c["require_star"].items():
        assert lo <= tr["star"][k] <= hi, "%s at t* not in [%d, %d]: %s" % (k, lo, hi, reached)
    for k, v in tr["peak"].items():  # nothing before t* crosses a capacity: the steps the GPU test compares are exact
        assert v <= caps.get(k, v), "%s over its capacity before t*: %s" % (k, reached)
    if name == "d_side255_s1":
        assert (c["stream"][:c["n_steps"], :3] == 255).any(), reached
