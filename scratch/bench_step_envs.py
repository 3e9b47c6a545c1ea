"""Selected-env calls (pct_step_envs, pct_reset_envs_only, pct_set_items_only) against their whole-batch counterparts.

For discrete settings 1 and 2 and the continuous domain (setting 1), at 1024 and 4096 envs, after 40 random-policy steps: CUDA-event timing of
CUDA-graph replays (bench_queries.timed) of
  the random policy + pct_step, and the random policy + pct_step_envs of 1 env, 1 %, 10 %, 50 % and all envs, by list and by mask
  (the policy kernel alone is reported too);
  pct_reset_envs_only / pct_set_items_only of 1 env and of 1 % of the envs against pct_reset_envs / pct_set_items;
  the gym loop "policy -> step -> reset(mask=done, whole_batch=False)" (auto_reset=False) against "policy -> step" of the auto-reset twin.
Every measurement starts from the same restored state.  Reports µs per call, with the card, its power limit and max SM clock.
python scratch/bench_step_envs.py [--iters 20]
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


def make(n, setting, continuous, auto_reset=True):
    if continuous:
        return pct_b200.PctBatch(n, setting, container_size=(1.0, 1.0, 1.0), continuous=True, sample_from_distribution=True, seed=1234,
                                 auto_reset=auto_reset)
    return pct_b200.PctBatch(n, setting, item_set=ITEMS, seed=1234, auto_reset=auto_reset)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    name, pl = card()
    print(json.dumps(dict(card=name, power_limit_and_max_sm_clock=pl)), flush=True)
    gen = torch.Generator().manual_seed(7)
    for continuous, setting in ((False, 1), (False, 2), (True, 1)):
        for n in (1024, 4096):
            A, B = make(n, setting, continuous), make(n, setting, continuous, auto_reset=False)
            A.reset(); B.reset()
            for t in range(40):
                A.step(leaf_idx=A.random_policy(4321, t))
                B.step(leaf_idx=B.random_policy(4321, t))
                B.reset(mask=B._done, whole_batch=False)
            assert torch.equal(A._obs, B._obs)
            snap_a, snap_b = A.snapshot(), B.snapshot()
            dev = A.device
            idx = torch.zeros((n,), dtype=torch.int32, device=dev)
            out = dict(domain="continuous" if continuous else "discrete", setting=setting, n_envs=n)

            def run(key, fn, b=A, snap=snap_a):
                b.restore(snap)
                out[key] = round(timed(fn, args.iters) * 1e6, 2)

            run("policy_us", lambda: A.random_policy(4321, 40, out=idx))
            run("step_us", lambda: A.step(leaf_idx=A.random_policy(4321, 40, out=idx)))
            for frac, k in (("1", 1), ("1pct", max(1, n // 100)), ("10pct", n // 10), ("50pct", n // 2), ("all", n)):
                sel = torch.randperm(n, generator=gen)[:k].sort().values.to(dtype=torch.int32, device=dev)
                m = torch.zeros(n, dtype=torch.bool, device=dev)
                m[sel.long()] = True
                run("step_envs_list_%s_us" % frac, lambda: A.step(leaf_idx=A.random_policy(4321, 40, out=idx), env_idx=sel))
                run("step_envs_mask_%s_us" % frac, lambda: A.step(leaf_idx=A.random_policy(4321, 40, out=idx), mask=m))
                if frac in ("1", "1pct"):
                    run("reset_envs_%s_us" % frac, lambda: A.reset(env_idx=sel))
                    run("reset_envs_only_%s_us" % frac, lambda: A.reset(env_idx=sel, whole_batch=False))
                    items = (torch.full((k, 3), 0.2, dtype=torch.float64, device=dev) if continuous
                             else torch.full((k, 3), 2, dtype=torch.int32, device=dev))
                    run("set_items_%s_us" % frac, lambda: A.set_items(items, env_idx=sel))
                    run("set_items_only_%s_us" % frac, lambda: A.set_items(items, env_idx=sel, whole_batch=False))
            run("auto_reset_loop_us", lambda: A.step(leaf_idx=A.random_policy(4321, 40, out=idx)))

            def gym():
                B.random_policy(4321, 40, out=idx)
                B.step(leaf_idx=idx)
                B.reset(mask=B._done, whole_batch=False)
            run("gym_loop_reset_only_us", gym, B, snap_b)
            print(json.dumps(out), flush=True)
            A.close(); B.close()


if __name__ == "__main__":
    main()
