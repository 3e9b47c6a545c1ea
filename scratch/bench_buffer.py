"""Buffered packing (pct_buffer_step, DESIGN.md section 18) against the same decision composed from plain calls, and against a plain step.

For discrete settings 1 and 2 and the continuous domain (setting 1), at 1024 and 4096 envs, B in {1, 3, 5, 10}, after 40 random-policy steps:
CUDA-event timing of CUDA-graph replays (bench_queries.timed) of
  buffer    pct_buffer_policy_random + pct_buffer_step (the policy kernel alone is reported as `policy`);
  composed  expand_items of B items + set_items_only of the chosen one + step_envs of every env, on a plain batch;
  plain     the random policy + pct_step, on a plain batch (once per configuration).
Reports µs per call, with the card, its power limit and max SM clock.  --only-buffer: the buffered step alone (A/B of builds through
PCT_B200_LIB, e.g. the in-turn slot layout: UNIT=pct_buffer scratch/mkvariant.sh inturn -DBUF_SLOTS_INTURN=1).
python scratch/bench_buffer.py [--iters 20] [--only-buffer]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scratch"))
import pct_b200  # noqa: E402
from bench_queries import card, timed  # noqa: E402

ITEMS = [(i, j, k) for i in range(1, 6) for j in range(1, 6) for k in range(1, 6)]
SEED = 5


def make(n, setting, continuous, buffer=None):
    if continuous:
        return pct_b200.PctBatch(n, setting, container_size=(1.0, 1.0, 1.0), continuous=True, sample_from_distribution=True, seed=1234, buffer=buffer)
    return pct_b200.PctBatch(n, setting, item_set=ITEMS, seed=1234, buffer=buffer)


def warm(b, continuous, steps=40):
    b.reset()
    t = torch.zeros((), dtype=torch.int64, device=b.device)
    for i in range(steps):
        idx = b.random_policy_dev(SEED, t) if (b.buffer is not None or not continuous) else b.random_policy(SEED, i)
        b.step(leaf_idx=idx)
        t += 1
    torch.cuda.synchronize()
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--only-buffer", action="store_true")
    args = ap.parse_args()
    name, pl = card()
    print(json.dumps(dict(card=name, power_limit_and_max_sm_clock=pl, lib=os.environ.get("PCT_B200_LIB", "default"))), flush=True)
    for continuous, setting in ((False, 1), (False, 2), (True, 1)):
        dom = "c%d" % setting if continuous else "d%d" % setting
        for n in (1024, 4096):
            plain_us = None
            if not args.only_buffer:
                Q = make(n, setting, continuous)
                t = warm(Q, continuous)
                if continuous:
                    plain_us = timed(lambda: Q.step(leaf_idx=Q.random_policy(SEED, 0)), args.iters) * 1e6
                else:
                    plain_us = timed(lambda: Q.step(leaf_idx=Q.random_policy_dev(SEED, t)), args.iters) * 1e6
            for B in (1, 3, 5, 10):
                P = make(n, setting, continuous, buffer=B)
                t = warm(P, continuous)
                pol_us = timed(lambda: P.random_policy_dev(SEED, t), args.iters) * 1e6
                buf_us = timed(lambda: P.step(leaf_idx=P.random_policy_dev(SEED, t)), args.iters) * 1e6
                row = dict(domain=dom, n_envs=n, B=B, buffer_us=round(buf_us, 1), policy_us=round(pol_us, 1))
                P.close()
                if not args.only_buffer:
                    items = Q.preview_items(B)
                    qd = torch.float64 if continuous else torch.int32
                    it3 = items[:, :, :3].to(qd).contiguous()
                    den = items[:, :, 3].contiguous()
                    first, den0 = it3[:, 0].contiguous(), den[:, 0].contiguous()
                    lv = torch.empty((n, B, Q.nl, 9), dtype=Q.obs_dtype, device=Q.device)
                    li = torch.empty((n, B, 8), dtype=torch.int32, device=Q.device)
                    obs = torch.empty((n, Q.obs_len), dtype=Q.obs_dtype, device=Q.device)
                    leaf = torch.zeros(n, dtype=torch.int32, device=Q.device)
                    ar = torch.arange(n, dtype=torch.int32, device=Q.device)

                    def composed():
                        Q.expand_items(it3, density=den, out=(lv, li))
                        Q.set_items(first, density=den0, out=obs, whole_batch=False)
                        Q.step(leaf_idx=leaf, env_idx=ar, out=obs)
                    row.update(composed_us=round(timed(composed, args.iters) * 1e6, 1), plain_step_us=round(plain_us, 1))
                print(json.dumps(row), flush=True)
            if not args.only_buffer:
                Q.close()


if __name__ == "__main__":
    main()
