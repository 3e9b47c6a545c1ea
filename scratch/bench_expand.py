"""Read-only leaf expansion of caller-given items (pct_expand_items) against set_items on every env and one pct_step of the same batch.

For 1024 and 4096 envs, settings 1 and 2, both domains, after 40 random-policy steps: CUDA-event timing of CUDA-graph replays of
  expand_items with k = 1, 3 and 8 items per env (random items of the batch's kind),
  set_items on every env (each env's own current item) and steady-state steps, measured as scratch/bench_items.py measures them,
and one B = 3 buffer decision two ways (eager calls between two events): on expand_items (expand the buffer, pick the item with the
most leaves and its first leaf, set_items + step) and as BufferDriver.step() (tests/buffer_compose.py: fan-out into 3 children).
Reports µs per call, with the card and its power limit.  python scratch/bench_expand.py [--iters 20]
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


def item_source(n, length, continuous, rng):
    if continuous:
        src = np.round(rng.uniform(0.1, 0.5, (n, length, 3)), 3)
    else:
        src = np.stack([np.asarray(ITEMS, dtype=np.float64)[rng.integers(0, len(ITEMS), length)] for _ in range(n)])
    return np.concatenate([src, np.ones(src.shape[:2] + (1,))], axis=2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    name, pl = card()
    print(json.dumps(dict(card=name, power_limit_and_max_sm_clock=pl)), flush=True)
    rng = np.random.default_rng(0)
    for continuous in (False, True):
        for setting in (1, 2):
            for n in (1024, 4096):
                b = make(n, setting, continuous)
                b.reset()
                for t in range(40):
                    _, _, _, info = b.step(leaf_idx=b.random_policy(4321, t))
                b.check_flags(info[:, 1].cpu().numpy())
                qd = torch.float64 if continuous else torch.int32
                out = dict(domain="continuous" if continuous else "discrete", setting=setting, n_envs=n)
                src = torch.as_tensor(item_source(n, 8, continuous, rng)[:, :, :3]).to(device=b.device, dtype=qd)
                for k in (1, 3, 8):
                    items = src[:, :k].contiguous()
                    o = b.expand_items(items)
                    sec = timed(lambda: b.expand_items(items, out=o), args.iters)
                    out["expand_k%d_us" % k] = round(sec * 1e6, 1)
                cur = b.preview_items(1)[:, 0].clone()
                items1 = cur[:, :3].to(qd).contiguous()
                den = cur[:, 3].contiguous()
                sec = timed(lambda: b.set_items(items1, density=den), args.iters)
                out["set_items_all_us"] = round(sec * 1e6, 1)
                snap = b.snapshot()
                idx = torch.zeros((n,), dtype=torch.int32, device=b.device)

                def step():
                    b.random_policy(4321, 40, out=idx)
                    b.step(leaf_idx=idx)
                sec_ps = timed(step, args.iters)
                sec_p = timed(lambda: b.random_policy(4321, 40, out=idx), args.iters)
                out["step_us"] = round((sec_ps - sec_p) * 1e6, 1)
                for k in (1, 3, 8):
                    out["expand_k%d_over_step" % k] = round(out["expand_k%d_us" % k] / out["step_us"], 2)
                out["expand_k1_over_set_items"] = round(out["expand_k1_us"] / out["set_items_all_us"], 2)
                b.restore(snap, write_obs=False)
                # one B = 3 buffer decision on expand_items: expand, choose, set_items, step, refill
                B = 3
                bsrc = torch.as_tensor(item_source(n, 64, continuous, rng)).to(b.device)
                st = dict(buf=bsrc[:, :B].clone(), pos=B)
                ar = torch.arange(n, device=b.device)
                lv = torch.empty((n, B, b.nl, 9), dtype=b.obs_dtype, device=b.device)
                inf = torch.empty((n, B, 8), dtype=torch.int32, device=b.device)

                def decide_expand():
                    buf = st["buf"]
                    b.expand_items(buf[:, :, :3], density=buf[:, :, 3].contiguous(), out=(lv, inf))
                    j = inf[:, :, 5].argmax(1)
                    chosen = buf[ar, j]
                    b.set_items(chosen[:, :3], density=chosen[:, 3].contiguous())
                    b.step(leaf_idx=idx)
                    buf[ar, j] = bsrc[:, st["pos"] % 64]
                    st["pos"] += 1
                sec = timed(decide_expand, max(4, args.iters // 4), graph=False)
                out["buffer_decision_B3_expand_us"] = round(sec * 1e6, 1)
                b.restore(snap, write_obs=False)
                child = make(n * B, setting, continuous)
                child.reset()
                drv = BufferDriver(b, child, bsrc.cpu(), B)
                sec = timed(drv.step, max(4, args.iters // 4), graph=False)
                out["buffer_decision_B3_driver_us"] = round(sec * 1e6, 1)
                print(json.dumps(out), flush=True)
                child.close()
                b.close()


if __name__ == "__main__":
    main()
