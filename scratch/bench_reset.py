"""Per-env reset (pct_reset_envs) against one pct_step of the same batch, and the gym loop it enables against the auto-reset step.

For 1024 and 4096 envs, settings 1 and 2, both domains, after 40 random-policy steps: CUDA-event timing of CUDA-graph replays of
  reset(env_idx=...) of 1 env, of 1 % of the envs and of every env, and reset(mask=all zeros); a replayed reset of every env resets
  empty bins from the second call on, so it is also timed from the mid-episode state every time (restore + reset minus restore),
  steady-state steps of the random policy (minus the policy kernel), on the same observation buffer as the resets,
  the graphed loop "random policy -> step -> reset(mask=done)" of a batch without auto-reset against "random policy -> step" of its
  auto-reset twin (same items and actions, so both loops compute the same observations; checked after the timing).
The batch state is saved before and restored after each reset measurement.  Reports µs per call, with the card and its power limit.
python scratch/bench_reset.py [--iters 20]
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
    print(json.dumps(dict(card=name, power_limit_and_max_sm_clock=pl)))
    for continuous in (False, True):
        for setting in (1, 2):
            for n in (1024, 4096):
                A, B = make(n, setting, continuous), make(n, setting, continuous, auto_reset=False)
                A.reset(); B.reset()
                for t in range(40):
                    _, _, _, info = A.step(leaf_idx=A.random_policy(4321, t))
                    B.step(leaf_idx=B.random_policy(4321, t))
                    B.reset(mask=B._done)
                A.check_flags(info[:, 1].cpu().numpy())
                assert torch.equal(A._obs, B._obs)
                out = dict(domain="continuous" if continuous else "discrete", setting=setting, n_envs=n)
                idx = torch.zeros((n,), dtype=torch.int32, device=A.device)

                def step():
                    A.random_policy(4321, 40, out=idx)
                    A.step(leaf_idx=idx)
                snap = A.snapshot()
                sec_ps = timed(step, args.iters)
                sec_p = timed(lambda: A.random_policy(4321, 40, out=idx), args.iters)
                out["step_us"] = round((sec_ps - sec_p) * 1e6, 1)
                A.restore(snap, write_obs=False)
                A.step(leaf_idx=A.random_policy(4321, 40))  # rewrites every row of the restored envs: the resets below see the delta rows of a step
                snap = A.snapshot()
                lists = dict(one=torch.tensor([n // 2], dtype=torch.int32, device=A.device),
                             pct1=torch.arange(0, n, 100, dtype=torch.int32, device=A.device),
                             all=torch.arange(n, dtype=torch.int32, device=A.device))
                for key, lst in lists.items():
                    sec = timed(lambda: A.reset(env_idx=lst), args.iters)
                    out["reset_%s_us" % key] = round(sec * 1e6, 1)
                    A.restore(snap, write_obs=False)
                    A.step(leaf_idx=A.random_policy(4321, 40))
                    snap = A.snapshot()
                zero = torch.zeros((n,), dtype=torch.uint8, device=A.device)
                out["reset_mask0_us"] = round(timed(lambda: A.reset(mask=zero), args.iters) * 1e6, 1)
                # every env reset from the mid-episode state each time: restore + reset minus restore alone (the reset after a restore
                # without observation rows writes every row of every env)
                A.restore(snap, write_obs=False)
                sec_rr = timed(lambda: (A.restore(snap, write_obs=False), A.reset(env_idx=lists["all"])), args.iters)
                sec_r = timed(lambda: A.restore(snap, write_obs=False), args.iters)
                out["reset_all_mid_us"] = round((sec_rr - sec_r) * 1e6, 1)
                A.step(leaf_idx=A.random_policy(4321, 40))
                for key in ("one", "pct1", "all", "all_mid", "mask0"):
                    out["reset_%s_over_step" % key] = round(out["reset_%s_us" % key] / out["step_us"], 2)
                # the graphed gym loop against the auto-reset step: both twins from the same state (B follows A's restores)
                A.restore(snap)
                B.restore(snap)
                ia, ib = torch.zeros_like(idx), torch.zeros_like(idx)

                def auto():
                    A.random_policy(4321, 41, out=ia)
                    A.step(leaf_idx=ia)

                def gym():
                    B.random_policy(4321, 41, out=ib)
                    B.step(leaf_idx=ib)
                    B.reset(mask=B._done)
                out["loop_auto_reset_us"] = round(timed(auto, args.iters) * 1e6, 1)
                out["loop_step_reset_mask_us"] = round(timed(gym, args.iters) * 1e6, 1)
                out["loop_ratio"] = round(out["loop_step_reset_mask_us"] / out["loop_auto_reset_us"], 2)
                out["loop_outputs_equal"] = bool(torch.equal(A._obs, B._obs))
                print(json.dumps(out), flush=True)
                A.close(); B.close()


if __name__ == "__main__":
    main()
