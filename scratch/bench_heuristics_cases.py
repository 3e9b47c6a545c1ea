"""Heuristic baselines per container: selection-kernel time per call (CUDA events around pct_heuristic_actions) and the time of a
whole step (selection + pct_step), setting 2, on 10^3, 20x18x24, 40x36x16 and the 255^3 limit container (DESIGN.md section 14).
Prints one line per (container, baseline) and, with --json PATH, writes the table with the card name and power limit.

    python scratch/bench_heuristics_cases.py [--json heur_cases.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pct_b200  # noqa: E402

ITEMS = [(i, j, k) for i in range(1, 6) for j in range(1, 6) for k in range(1, 6)]
BIG = [(i, j, k) for i in (4, 6, 9) for j in (5, 8) for k in (3, 7, 10)]
BIG40 = [(i, j, k) for i in (3, 7, 12) for j in (4, 9) for k in (3, 8, 11)]
LIMIT = [(255, 255, 255), (250, 60, 6), (40, 40, 5), (200, 180, 120), (90, 240, 100)]
CONTAINERS = [("10x10x10", (10, 10, 10), ITEMS), ("20x18x24", (20, 18, 24), BIG), ("40x36x16", (40, 36, 16), BIG40),
              ("255x255x255", (255, 255, 255), LIMIT)]
NAMES = ("LSAH", "OnlineBPH", "BR", "MACS", "DBL", "HM", "RANDOM")


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                            timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def one(name, container, items, n, warm, steps):
    b = pct_b200.PctBatch(n, 2, container_size=container, item_set=items, seed=3)
    b.reset()
    for t in range(warm):
        b.step(actions=b.heuristic_actions(name, t=t))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    sel = 0.0
    t0 = time.perf_counter()
    for t in range(steps):
        e0.record()
        rows = b.heuristic_actions(name, t=warm + t)
        e1.record()
        b.step(actions=rows)
        e1.synchronize()
        sel += e0.elapsed_time(e1)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    b.close()
    return sel / steps, dt / steps * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--macs-envs", type=int, default=256)
    a = ap.parse_args()
    gpu, pl = card()
    print("card: %s, power limit %s" % (gpu, pl), flush=True)
    rows = []
    for cname, container, items in CONTAINERS:
        limit = container[0] > 100
        for name in NAMES:
            n = a.macs_envs if name == "MACS" else a.envs
            if limit and name == "MACS":
                n = min(n, 64)
            warm, steps = (3, 5) if limit else (10, 30)
            sel, step = one(name, container, items, n, warm, steps)
            rows.append(dict(container=cname, heuristic=name, setting=2, envs=n, selection_ms=round(sel, 4), step_ms=round(step, 4)))
            print("%-12s %-9s %5d envs: selection %.3f ms/call, step (selection + pct_step) %.3f ms" % (cname, name, n, sel, step), flush=True)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(dict(card=gpu, power_limit=pl, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
