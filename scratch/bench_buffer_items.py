"""Item preview and item override of buffered batches (pct_buffer_preview_items, pct_buffer_set_items; DESIGN.md section 21).

For discrete settings 1 and 2 and the continuous domain (setting 1), at 4096 envs, B in {3, 16}, after 40 random-policy steps:
CUDA-event timing of CUDA-graph replays (bench_queries.timed) of
  set_all    pct_buffer_set_items of every env, with the envs' own buffers (the rows an override writes; the expansion's work is that of a step's);
  set_1%     pct_buffer_set_items of 1 % of the envs (an index list);
  step       pct_buffer_step of every env with the policy's flat indices (the reference: select, apply, refill, expansion);
  preview    pct_buffer_preview_items(k = 1) of every env.
Reports µs per call, with the card, its power limit and max SM clock.
python scratch/bench_buffer_items.py [--iters 20] [--domains d1,d2,c1]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scratch"))
from bench_buffer_envs import SEED, make, warm  # noqa: E402
from bench_queries import card, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--domains", default="d1,d2,c1", help="comma-separated subset of d1, d2, c1")
    args = ap.parse_args()
    name, pl = card()
    print(json.dumps(dict(card=name, power_limit_and_max_sm_clock=pl)), flush=True)
    n = args.n
    for d in args.domains.split(","):
        continuous, setting = d[0] == "c", int(d[1])
        for B in (3, 16):
            P = make(n, setting, continuous, buffer=B)
            t = warm(P, continuous)
            flat = P.random_policy_dev(SEED, t).clone()
            items = P.buffer_items()
            k = max(1, n // 100)
            sel = torch.as_tensor(np.sort(np.random.RandomState(k).permutation(n)[:k]).astype(np.int32), device=P.device)
            few = items[sel.long()].contiguous()
            pv = torch.zeros((n, 1, 4), dtype=torch.float64, device=P.device)
            torch.cuda.synchronize()
            set_all = timed(lambda: P.buffer_set_items(items), args.iters) * 1e6
            set_few = timed(lambda: P.buffer_set_items(few, env_idx=sel), args.iters) * 1e6
            prev = timed(lambda: P.buffer_preview_items(1, out=pv), args.iters) * 1e6
            step = timed(lambda: P.step(leaf_idx=flat), args.iters) * 1e6
            print(json.dumps(dict(domain=d, n_envs=n, B=B, set_all_us=round(set_all, 1), set_1pct_us=round(set_few, 1), set_1pct_envs=k,
                                  buffer_step_us=round(step, 1), set_all_over_step=round(set_all / step, 3), preview_k1_us=round(prev, 1))), flush=True)
            P.close()


if __name__ == "__main__":
    main()
