"""Item preview and item override (pct_preview_items / pct_set_items) against one pct_step of the same batch.

For 1024 and 4096 envs, settings 1 and 2, both domains, after 40 random-policy steps: CUDA-event timing of CUDA-graph replays of
  preview_items with k = 1 and k = 8,
  set_items on every env (each env's own current item: the state does not drift between replays),
  steady-state steps of the random policy (minus the policy kernel), on the same observation buffer as set_items,
and one decision of the buffer driver with B = 3 (tests/buffer_compose.py: fan-out into 3 children, set_items, heuristic rows,
query_placements, set_items + step of the parent; eager calls between two events).  Reports µs per call, with the card and its power
limit.  python scratch/bench_items.py [--iters 20]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scratch"))
import pct_b200  # noqa: E402
from bench_queries import card, timed  # noqa: E402
from buffer_compose import BufferDriver  # noqa: E402

ITEMS = [(i, j, k) for i in range(1, 6) for j in range(1, 6) for k in range(1, 6)]


def make(n, setting, continuous):
    if continuous:
        return pct_b200.PctBatch(n, setting, container_size=(1.0, 1.0, 1.0), continuous=True, sample_from_distribution=True, seed=1234)
    return pct_b200.PctBatch(n, setting, item_set=ITEMS, seed=1234)


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
                b = make(n, setting, continuous)
                b.reset()
                for t in range(40):
                    _, _, _, info = b.step(leaf_idx=b.random_policy(4321, t))
                b.check_flags(info[:, 1].cpu().numpy())
                out = dict(domain="continuous" if continuous else "discrete", setting=setting, n_envs=n)
                for k in (1, 8):
                    pv = b.preview_items(k)
                    sec = timed(lambda: b.preview_items(k, out=pv), args.iters)
                    out["preview_k%d_us" % k] = round(sec * 1e6, 1)
                cur = b.preview_items(1)[:, 0].clone()
                items = cur[:, :3].to(torch.float64 if continuous else torch.int32).contiguous()
                den = cur[:, 3].contiguous()
                sec = timed(lambda: b.set_items(items, density=den), args.iters)
                out["set_items_all_us"] = round(sec * 1e6, 1)
                # steady-state steps on the same observation buffer (delta rows, as set_items above): random policy + step, minus the policy
                # alone; the batch moves on, so its state is saved and restored around this
                snap = b.snapshot()
                idx = torch.zeros((n,), dtype=torch.int32, device=b.device)

                def step():
                    b.random_policy(4321, 40, out=idx)
                    b.step(leaf_idx=idx)
                sec_ps = timed(step, args.iters)
                sec_p = timed(lambda: b.random_policy(4321, 40, out=idx), args.iters)
                out["step_us"] = round((sec_ps - sec_p) * 1e6, 1)
                out["set_items_over_step"] = round(out["set_items_all_us"] / out["step_us"], 2)
                b.restore(snap, write_obs=False)
                # buffer driver, B = 3
                B = 3
                child = make(n * B, setting, continuous)
                child.reset()
                src = np.stack([np.asarray(ITEMS, dtype=np.float64)[rng.integers(0, len(ITEMS), 64)] for _ in range(n)])
                if continuous:
                    src = np.round(rng.uniform(0.1, 0.5, (n, 64, 3)), 3)
                src = np.concatenate([src, np.ones(src.shape[:2] + (1,))], axis=2)
                drv = BufferDriver(b, child, torch.as_tensor(src), B)
                sec = timed(drv.step, max(4, args.iters // 4), graph=False)
                out["buffer_decision_B3_us"] = round(sec * 1e6, 1)
                print(json.dumps(out), flush=True)
                child.close()
                b.close()


if __name__ == "__main__":
    main()
