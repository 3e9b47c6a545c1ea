"""Records the reference's UNMODIFIED heuristic baselines (heuristic.py: LASH, OnlineBPH, BR, MACS, DBL, heightmap_min) on containers
other than 10x10x10 -> tests/golden/heur_case_<case>.npz (the heur_s*.npz format plus `container` and `items`).  Needs the
reference checkout that oracle/ref_shim.py loads (PCT_REFERENCE_ROOT).

    python tests/golden/make_heuristic_golden_cases.py [case ...]        (default: every case; one process per case runs them in parallel)

big_s1..3:  20 x 18 x 24 with the `_BIG` items of tests/harness.py (the big_* step cases): below the 32-cell side of the static height map.
big40_s1..3: 40 x 36 x 16 with the BIG40 items of tests/test_gpu_queries.py: above it.  H = 16 keeps every episode far below the 80 boxes of
            internal_node_holder (the reference raises IndexError at 81); trajectories of 70 items cannot reach it either.
MACS re-scans the whole voxel grid per level per candidate in Python, so it plays fewer episodes.
"""
import contextlib
import io
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import ref_shim  # noqa: E402
from harness import _BIG  # noqa: E402
from pct_oracle import rnd_u64  # noqa: E402

BIG40_ITEMS = [(i, j, k) for i in (3, 7, 12) for j in (4, 9) for k in (3, 8, 11)]  # BIG40 of tests/test_gpu_queries.py
N_TRAJ = 12
CASES = {
    "big_s1": dict(setting=1, container=(20, 18, 24), items=_BIG, traj_len=60),
    "big_s2": dict(setting=2, container=(20, 18, 24), items=_BIG, traj_len=60),
    "big_s3": dict(setting=3, container=(20, 18, 24), items=_BIG, traj_len=60),
    "big40_s1": dict(setting=1, container=(40, 36, 16), items=BIG40_ITEMS, traj_len=70),
    "big40_s2": dict(setting=2, container=(40, 36, 16), items=BIG40_ITEMS, traj_len=70),
    "big40_s3": dict(setting=3, container=(40, 36, 16), items=BIG40_ITEMS, traj_len=70),
}
EPISODES = {"LSAH": 4, "OnlineBPH": 4, "BR": 4, "MACS": 2, "DBL": 4, "HM": 3}


def dataset(case, seed=4242):
    """N_TRAJ trajectories over the case's item set (setting 3: densities in (0, 1])"""
    s = case["setting"]
    d = np.ones((N_TRAJ, case["traj_len"], 4 if s == 3 else 3))
    for t in range(N_TRAJ):
        for k in range(case["traj_len"]):
            d[t, k, :3] = case["items"][rnd_u64(seed + s, t, k) % len(case["items"])]
            if s == 3:
                d[t, k, 3] = (1 + rnd_u64(seed ^ 0x5555, t, k) % 999) / 1000.0
    return d


def record(name_case):
    case = CASES[name_case]
    D, _ = ref_shim.load_reference()
    sys.argv = [sys.argv[0]]
    import heuristic as H  # the reference module, unmodified (imports givenData / tools from the reference checkout)
    fns = {"LSAH": H.LASH, "OnlineBPH": H.OnlineBPH, "BR": H.BR, "MACS": H.MACS, "DBL": H.DBL, "HM": H.heightmap_min}

    class Recording(D.PackingDiscrete):
        def reset(self):
            if hasattr(self, "packed"):
                self.log.append([list(p) for p in self.packed])
            return super().reset()

    setting, data = case["setting"], dataset(case)
    rec = {}
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "set.pt")
        torch.save([t.tolist() for t in data], path)
        for name, fn in fns.items():
            n_ep = EPISODES[name]
            env = Recording(setting=setting, container_size=list(case["container"]), item_set=case["items"], data_name=path,
                            load_test_data=True, internal_node_holder=80, leaf_node_holder=50)
            env.log = []
            with contextlib.redirect_stdout(io.StringIO()):
                fn(env, n_ep)
            eps = env.log[:n_ep]
            assert len(eps) == n_ep
            rec["len_" + name] = np.array([len(e) for e in eps])
            rec["flat_" + name] = np.array([p for e in eps for p in e], dtype=np.int64).reshape(-1, 7)
            print(name_case, name, "lengths", rec["len_" + name].tolist(), flush=True)
    out = os.path.join(HERE, "heur_case_%s.npz" % name_case)
    np.savez_compressed(out, setting=setting, data=data, container=np.array(case["container"]), items=np.array(case["items"]), **rec)
    print(out, os.path.getsize(out), "B")


if __name__ == "__main__":
    for c in sys.argv[1:] or list(CASES):
        record(c)
