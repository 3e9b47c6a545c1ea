"""Heuristic baselines of buffered envs (pct_buffer_heuristic_actions + pct_buffer_step_rows, DESIGN.md section 22) against the plain baseline
step (pct_heuristic_actions + pct_step) and against the same decision composed from plain calls.

LSAH, DBL and HM on discrete settings 1 and 2, LSAH on the continuous domain (setting 1); 4096 envs, B in {1, 3, 16}, after 30 baseline steps.
CUDA-event timing of CUDA-graph replays (bench_queries.timed) of
  buffer    buffer_heuristic_actions + buffer_step_rows (the heuristic call alone is reported as `heur`);
  plain     heuristic_actions + step(actions=rows), on a plain batch (once per configuration);
  composed  B x (set_items of one item + heuristic_actions) + set_items + step(actions=rows) on a plain batch: the device work of composing the
            decision from plain calls, without the host's pick between them (a lower bound of that route).
Reports µs per step, with the card, its power limit and max SM clock.
python scratch/bench_buffer_heuristics.py [--iters 20]
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
CITEMS = [(round(0.1 * i, 1), round(0.1 * j, 1), round(0.1 * k, 1)) for i in range(1, 6) for j in range(1, 6) for k in range(1, 6)]
SEED, N = 5, 4096


def make(setting, continuous, buffer=None):
    if continuous:
        return pct_b200.PctBatch(N, setting, container_size=(1.0, 1.0, 1.0), continuous=True, sample_from_distribution=True, item_set=CITEMS,
                                 seed=1234, buffer=buffer)
    return pct_b200.PctBatch(N, setting, item_set=ITEMS, seed=1234, buffer=buffer)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    name, pl = card()
    print(json.dumps(dict(card=name, power_limit_and_max_sm_clock=pl)), flush=True)
    for continuous, setting, heur in ((False, 1, "LSAH"), (False, 1, "DBL"), (False, 1, "HM"), (False, 2, "LSAH"), (False, 2, "DBL"),
                                      (False, 2, "HM"), (True, 1, "LSAH")):
        dom = "c%d" % setting if continuous else "d%d" % setting
        P = make(setting, continuous)
        P.reset()
        for t in range(30):
            P.step(actions=P.heuristic_actions(heur, seed=SEED, t=t))
        plain_us = timed(lambda: P.step(actions=P.heuristic_actions(heur, seed=SEED)), args.iters) * 1e6
        for B in (1, 3, 16):
            if continuous:
                it = torch.rand((N, 3), dtype=torch.float64, device=P.device).mul(0.4).add(0.1).mul(1000).round().div(1000)
            else:
                it = torch.randint(1, 6, (N, 3), dtype=torch.int32, device=P.device)

            def composed():
                for _ in range(B):
                    P.set_items(it)
                    P.heuristic_actions(heur, seed=SEED)
                P.set_items(it)
                P.step(actions=P.heuristic_actions(heur, seed=SEED))
            comp_us = timed(composed, max(2, args.iters // B)) * 1e6
            Q = make(setting, continuous, buffer=B)
            Q.reset()
            for t in range(30):
                Q.buffer_step_rows(*Q.buffer_heuristic_actions(heur, seed=SEED, t=t))
            torch.cuda.synchronize()
            heur_us = timed(lambda: Q.buffer_heuristic_actions(heur, seed=SEED), args.iters) * 1e6
            buf_us = timed(lambda: Q.buffer_step_rows(*Q.buffer_heuristic_actions(heur, seed=SEED)), args.iters) * 1e6
            print(json.dumps(dict(domain=dom, heuristic=heur, envs=N, B=B, buffer_us=round(buf_us, 1), heur_us=round(heur_us, 1),
                                  plain_us=round(plain_us, 1), composed_us=round(comp_us, 1), buffer_over_plain=round(buf_us / plain_us, 2),
                                  composed_over_buffer=round(comp_us / buf_us, 2))), flush=True)
            Q.close()
        P.close()


if __name__ == "__main__":
    main()
