"""CPU: the torch composition of DBL / HM on height_maps + query_placements (tests/query_compose.py), with the two calls answered by
OracleDiscrete, chooses what the oracle restatement of the reference's heuristics chooses, on whole episodes."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
import pct_oracle_heuristics as H  # noqa: E402
from harness import CASES, ITEM_SET, OracleDiscrete, case_stream, make_stream  # noqa: E402
from query_compose import composed_rows, grid_queries  # noqa: E402


class OracleQueries(object):
    """stand-in for a PctBatch: query_placements / height_maps of n oracle envs (drop_box_virtual with each env's item density)"""

    def __init__(self, envs):
        self.envs = envs
        self.container_size = envs[0].container
        self.setting = envs[0].setting

    def height_maps(self):
        return torch.from_numpy(np.stack([e.plain() for e in self.envs]).astype(np.int32))

    def query_placements(self, queries):
        q = queries.numpy()
        feas = np.zeros(q.shape[:2], dtype=bool)
        rest = np.zeros(q.shape[:2], dtype=np.int32)
        for r, e in enumerate(self.envs):
            for j in range(q.shape[1]):
                feas[r, j], rest[r, j] = e.drop_box_virtual(q[r, j, :3], q[r, j, 3], q[r, j, 4])
        return torch.from_numpy(feas), torch.from_numpy(rest)


def test_grid_order_is_the_reference_loop():
    nb = [3, 5, 2]
    q, inside = grid_queries(torch.tensor([nb]), 10, 8, 2)
    want = [H.rot_dims(nb, r) + [lx, ly] for lx in range(10 - nb[0] + 1) for ly in range(8 - nb[1] + 1) for r in range(6)]
    assert q[0][inside[0]].tolist() == want


@pytest.mark.parametrize("name", ["DBL", "HM"])
@pytest.mark.parametrize("which", ["s1", "s2", "s3", "flat_s1"])
def test_composed_choice_equals_the_oracle_heuristic(name, which):
    if which == "flat_s1":
        c = CASES["flat_s1"]
        envs = [OracleDiscrete(1, container_size=c["container"], internal_node_holder=c["nb"], leaf_node_holder=c["nl"],
                               stream=case_stream(c, 5, e, 400)) for e in range(3)]
    else:
        setting = int(which[1])
        envs = [OracleDiscrete(setting, stream=make_stream(5, e, 400, setting)) for e in range(3)]
    view = OracleQueries(envs)
    for e in envs:
        e.reset()
    episodes, steps = np.zeros(len(envs), dtype=int), 0
    while (episodes < 2).any():
        rows = composed_rows(view, name, torch.tensor([e.next_box for e in envs])).numpy()
        for i, e in enumerate(envs):
            want = H.action_row(H.choose(name, e, None))
            assert np.array_equal(rows[i], want.astype(np.float32)), "env %d step %d: %s vs %s" % (i, steps, rows[i], want)
            _, _, done, _ = e.step(want)
            if done:
                episodes[i] += 1
                e.reset()
        steps += 1
        assert steps < 500
    assert ITEM_SET  # the default streams draw from the 125-item set
