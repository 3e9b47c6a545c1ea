"""Claim rounds per 32-key chunk of the discrete candidate list (csrc/pct_common.cuh set_claim_round), counted by the CPU model of
tests/test_cand_rounds_cpu.py on the EMS lists of bench.py's item streams: oracle envs (OracleDiscrete) fed uniform items over bench's
ITEM_SET, driven by the synthetic policy (policy_pick), the candidate list of every step rebuilt through the model.

    python scratch/cand_rounds_stats.py [--setting S] [--envs N] [--steps K]

Prints the histogram of rounds per chunk that holds new keys, the mean, and the rounds of the resize rehashes.  CPU only.
"""
import argparse
import collections
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]

import bench  # noqa: E402
import cand_inputs as ci  # noqa: E402
import test_cand_rounds_cpu as rounds  # noqa: E402
from pct_oracle import OracleDiscrete, policy_pick  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--setting", type=int, default=1)
    ap.add_argument("--envs", type=int, default=16)
    ap.add_argument("--steps", type=int, default=300)
    a = ap.parse_args()
    R = 6 if a.setting == 2 else 2
    st = rounds.new_stats()
    lists, keys = 0, 0
    for e in range(a.envs):
        rng = random.Random(e)
        stream = [list(rng.choice(bench.ITEM_SET)) + [1.0] for _ in range(a.steps + 1)]
        env = OracleDiscrete(a.setting, stream=stream)
        obs = env.reset()
        for t in range(a.steps):
            ems = [list(map(int, m)) for m in env.ems()]
            seq = ci.ems_sequence(ems, tuple(env.next_box), R, False)
            order, _, _ = rounds.run_rounds(seq, len(ems) * R * 4, st)
            lists += 1
            keys += len(order)
            _, row = policy_pick(obs, 80, 50, 99, e, t)
            obs, _, done, _ = env.step(row)
            if done:
                obs = env.reset()
    h = st["rounds"]
    n = sum(v for r, v in h.items() if r > 0)
    print("setting %d: %d lists, %.1f keys per list, %d chunks with new keys" % (a.setting, lists, keys / lists, n))
    print("rounds per chunk:", {r: h[r] for r in sorted(h) if r > 0}, "mean %.2f" % (sum(r * v for r, v in h.items()) / n))
    print("rehash rounds: %d (%d of the 32-slot groups took 2 or more)" % (st["rehash_rounds"], st["rehash_multi"]))
    print("resizes with keys pending:", dict(st["resize_pending"]))


if __name__ == "__main__":
    main()
