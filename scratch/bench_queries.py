"""Batched placement queries and height maps (pct_query_placements(_f64) / pct_height_maps) next to the paths a user has without them.

For 1024 and 4096 envs, settings 1 and 2, both domains, after 40 random-policy steps: CUDA-event timing of CUDA-graph replays of
  query_placements with k = 64 and 256 random placements per env (grid positions / positions in the bin, rotated item sizes),
  height_maps of every env (discrete),
and, in the same run,
  1000 single query_placement calls (synchronous, host clock),
  one heuristic_actions("DBL") (discrete; it evaluates the W x L x rotations grid of every env; continuous: "LSAH" over the EMS),
  one step of DBL composed in torch on query_placements (tests/query_compose.py; eager, the current items are passed in).
Reports µs per call and millions of queries/s, with the card and its power limit.  python scratch/bench_queries.py [--iters 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import pct_b200  # noqa: E402
from query_compose import ROT, composed_rows  # noqa: E402

ITEMS = [(i, j, k) for i in range(1, 6) for j in range(1, 6) for k in range(1, 6)]


def timed(fn, iters, graph=True):
    """seconds per call: `iters` calls captured in one CUDA graph and replayed 5 times; graph=False: eager calls between two events"""
    fn()
    torch.cuda.synchronize()
    a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if graph:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(iters):
                fn()
        g.replay()
        torch.cuda.synchronize()
        a.record()
        for _ in range(5):
            g.replay()
        z.record()
        torch.cuda.synchronize()
        return a.elapsed_time(z) / (5 * iters) * 1e-3
    a.record()
    for _ in range(iters):
        fn()
    z.record()
    torch.cuda.synchronize()
    return a.elapsed_time(z) / iters * 1e-3


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        pl = "unavailable (%s)" % e
    return name, pl


def random_queries(n, k, continuous, rng):
    if continuous:
        q = np.concatenate([np.round(rng.uniform(0.1, 0.5, (n, k, 3)), 3), np.round(rng.uniform(0.0, 1.0, (n, k, 2)), 3)], axis=2)
        return torch.as_tensor(q, dtype=torch.float64, device="cuda")
    it = np.asarray(ITEMS)[rng.integers(0, len(ITEMS), (n, k))]
    perm = np.asarray(ROT)[rng.integers(0, 6, (n, k))]
    dims = np.take_along_axis(it, perm, axis=2)
    q = np.concatenate([dims, rng.integers(0, 10, (n, k, 2))], axis=2)
    return torch.as_tensor(q, dtype=torch.int32, device="cuda")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    name, pl = card()
    print(json.dumps(dict(card=name, power_limit_and_max_sm_clock=pl)))
    rng = np.random.default_rng(0)
    for continuous in (False, True):
        for setting in (1, 2):
            for n in (1024, 4096):
                if continuous:
                    b = pct_b200.PctBatch(n, setting, container_size=(1.0, 1.0, 1.0), continuous=True, sample_from_distribution=True, seed=1234)
                else:
                    b = pct_b200.PctBatch(n, setting, item_set=ITEMS, seed=1234)
                b.reset()
                for t in range(40):
                    _, _, _, info = b.step(leaf_idx=b.random_policy(4321, t))
                b.check_flags(info[:, 1].cpu().numpy())
                out = dict(domain="continuous" if continuous else "discrete", setting=setting, n_envs=n)
                for k in (64, 256):
                    q = random_queries(n, k, continuous, rng)
                    f, h = b.query_placements(q)
                    sec = timed(lambda: b.query_placements(q, out=(f, h)), args.iters)
                    out["queries_k%d" % k] = dict(us=round(sec * 1e6, 1), Mqueries_per_s=round(n * k / sec / 1e6, 1), feasible=round(float(f.float().mean()), 3))
                if not continuous:
                    hm = b.height_maps()
                    sec = timed(lambda: b.height_maps(out=hm), args.iters)
                    out["height_maps"] = dict(us=round(sec * 1e6, 1))
                # 1000 single synchronous queries (the path without the batched call)
                qh = random_queries(1, 1000, continuous, rng)[0].cpu().numpy()
                b.query_placement(0, qh[0, :3], qh[0, 3], qh[0, 4])
                t0 = time.perf_counter()
                for j in range(1000):
                    b.query_placement(j % n, qh[j, :3], qh[j, 3], qh[j, 4])
                sec = (time.perf_counter() - t0) / 1000
                out["single_query"] = dict(us=round(sec * 1e6, 1), Mqueries_per_s=round(1 / sec / 1e6, 4))
                heur = "LSAH" if continuous else "DBL"
                rows = b.heuristic_actions(heur)
                sec = timed(lambda: b.heuristic_actions(heur, out=rows), args.iters)
                out["heuristic_" + heur] = dict(us=round(sec * 1e6, 1))
                if not continuous:  # the same DBL in torch: grid enumeration + query_placements + first minimum (current items given)
                    nb = torch.as_tensor(np.asarray([b.state(e)["next_box"] for e in range(n)], dtype=np.int64), device=b.device)
                    ok = torch.equal(composed_rows(b, "DBL", nb), b.heuristic_actions("DBL"))
                    sec = timed(lambda: composed_rows(b, "DBL", nb), args.iters, graph=False)
                    R = 6 if setting == 2 else 2
                    out["composed_DBL"] = dict(us=round(sec * 1e6, 1), queries_per_env=100 * R, equals_builtin=ok)
                print(json.dumps(out), flush=True)
                b.close()


if __name__ == "__main__":
    main()
