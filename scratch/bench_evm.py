"""Step time of LNES='EVM' (EventPoint over the maintained EMS list and ZMAP) against 'EMS' and the reference's degenerate 'EV'.

For 1024 and 4096 envs, settings 1 and 2, 10x10x10 bin, the 125-item set: reset, 20 random-policy steps, then `--steps` random-policy steps
timed between two CUDA events (auto-reset on).  Reports ms per step, the mean number of valid leaves per observation, and the share of envs
whose record carries the candidate-overflow flag at the end, with the card and its power limit.  python scratch/bench_evm.py [--steps 50]
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
from bench_queries import card  # noqa: E402

ITEMS = [(i, j, k) for i in range(1, 6) for j in range(1, 6) for k in range(1, 6)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    a = ap.parse_args()
    name, pl = card()
    print(json.dumps(dict(card=name, power_limit_and_max_sm_clock=pl)), flush=True)
    for setting in (1, 2):
        for n in (1024, 4096):
            for lnes in ("EMS", "EV", "EVM"):
                b = pct_b200.PctBatch(n, setting, item_set=ITEMS, seed=1234, LNES=lnes)
                b.reset()
                for t in range(20):
                    b.step(leaf_idx=b.random_policy(4321, t))
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for t in range(a.steps):
                    obs, _, _, info = b.step(leaf_idx=b.random_policy(4321, 20 + t))
                e1.record()
                torch.cuda.synchronize()
                leaves = float(obs.view(n, -1, 9)[:, 80:130, 8].sum(1).float().mean())  # 80 internal / 50 leaf rows (the defaults)
                flagged = sum(1 for e in range(0, n, max(1, n // 256)) if b.state(e)["flags"] & 8) / len(range(0, n, max(1, n // 256)))
                print(json.dumps(dict(setting=setting, n_envs=n, lnes=lnes, ms_per_step=round(e0.elapsed_time(e1) / a.steps, 3),
                                      mean_leaves_last_obs=round(leaves, 1), cand_overflow_share=round(flagged, 3))), flush=True)
                b.close()


if __name__ == "__main__":
    main()
