"""Selected envs and snapshots of buffered batches (pct_buffer_step_envs, pct_buffer_reset_envs, pct_buffer_snapshot / _restore; DESIGN.md
section 20).

For discrete settings 1 and 2 and the continuous domain (setting 1), at 1024 and 4096 envs, B in {3, 5}, after 40 random-policy steps:
CUDA-event timing of CUDA-graph replays (bench_queries.timed) of
  step_envs   pct_buffer_step_envs of a selection of 1 env, 1 %, 10 %, 50 % and 100 % (an index list; the flat indices of the policy kernel);
  full        pct_buffer_step of every env (the same flat indices);
  plain       pct_step_envs of the same selection on a plain batch (once per configuration and selection);
  reset       pct_buffer_reset_envs of 4 envs and of 10 %;
  snapshot / restore of every env (restore with and without rows), and a 512 x 8 fan-out (512 records, each into 8 envs; at 1024 envs the
              first 1024 destinations), with GB/s of the record bytes moved: the nonzero bytes of one zero-filled snapshot (a lower bound of the
              live prefixes), plus the observation rows for a restore with rows.
Reports µs per call, with the card, its power limit and max SM clock.
python scratch/bench_buffer_envs.py [--iters 20] [--quick] [--domains d1,d2,c1]
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
import pct_b200  # noqa: E402
from bench_queries import card, timed  # noqa: E402

ITEMS = [(i, j, k) for i in range(1, 6) for j in range(1, 6) for k in range(1, 6)]
SEED = 5
FRACS = (("1", None), ("1%", 0.01), ("10%", 0.10), ("50%", 0.50), ("100%", 1.0))


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


def selection(n, frac, dev):
    k = 1 if frac is None else max(1, int(round(n * frac)))
    return torch.as_tensor(np.sort(np.random.RandomState(k).permutation(n)[:k]).astype(np.int32), device=dev)


def live_bytes(snap):
    """nonzero bytes of a zero-filled snapshot: a lower bound of the bytes its live prefixes move"""
    return int((snap.cpu().numpy() != 0).sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--quick", action="store_true", help="1024 envs, B = 3, discrete setting 1 only")
    ap.add_argument("--domains", default="d1,d2,c1", help="comma-separated subset of d1, d2, c1")
    args = ap.parse_args()
    name, pl = card()
    print(json.dumps(dict(card=name, power_limit_and_max_sm_clock=pl)), flush=True)
    doms = ((False, 1),) if args.quick else tuple((d[0] == "c", int(d[1])) for d in args.domains.split(","))
    for continuous, setting in doms:
        dom = "c%d" % setting if continuous else "d%d" % setting
        for n in ((1024,) if args.quick else (1024, 4096)):
            Q = make(n, setting, continuous)
            tq = warm(Q, continuous)
            qidx = Q.random_policy(SEED, 0) if continuous else Q.random_policy_dev(SEED, tq)
            plain = {}
            for lab, frac in FRACS:
                sel = selection(n, frac, Q.device)
                plain[lab] = timed(lambda: Q.step(leaf_idx=qidx, env_idx=sel), args.iters) * 1e6
            Q.close()
            for B in ((3,) if args.quick else (3, 5)):
                P = make(n, setting, continuous, buffer=B)
                t = warm(P, continuous)
                flat = P.random_policy_dev(SEED, t).clone()
                full = timed(lambda: P.step(leaf_idx=flat), args.iters) * 1e6
                for lab, frac in FRACS:
                    sel = selection(n, frac, P.device)
                    us = timed(lambda: P.buffer_step_envs(flat, env_idx=sel), args.iters) * 1e6
                    print(json.dumps(dict(domain=dom, n_envs=n, B=B, call="buffer_step_envs", selection=lab, us=round(us, 1),
                                          full_buffer_step_us=round(full, 1), plain_step_envs_us=round(plain[lab], 1))), flush=True)
                for lab, sel in (("4 envs", torch.as_tensor([3, 100, 500, n - 1], dtype=torch.int32, device=P.device)),
                                 ("10%", selection(n, 0.10, P.device))):
                    us = timed(lambda: P.buffer_reset_envs(env_idx=sel), args.iters) * 1e6
                    print(json.dumps(dict(domain=dom, n_envs=n, B=B, call="buffer_reset_envs", selection=lab, us=round(us, 1))), flush=True)
                snap = torch.zeros((n, P.buffer_snapshot_bytes), dtype=torch.uint8, device=P.device)
                P.buffer_snapshot(out=snap)
                torch.cuda.synchronize()
                live = live_bytes(snap)
                s_us = timed(lambda: P.buffer_snapshot(out=snap), args.iters) * 1e6
                r_us = timed(lambda: P.buffer_restore(snap), args.iters) * 1e6
                r0_us = timed(lambda: P.buffer_restore(snap, write_obs=False), args.iters) * 1e6
                rows = n * P.obs_len * P._obs.element_size()
                rec = torch.arange(512, device=P.device, dtype=torch.int32).repeat_interleave(8) % n
                dst = torch.arange(min(4096, n), device=P.device, dtype=torch.int32)
                fan = rec[:len(dst)]
                f_us = timed(lambda: P.buffer_restore(snap, env_idx=dst, rec_idx=fan, write_obs=False), args.iters) * 1e6
                print(json.dumps(dict(domain=dom, n_envs=n, B=B, record_bytes=P.buffer_snapshot_bytes, live_bytes_per_env=round(live / n),
                                      snapshot_us=round(s_us, 1), snapshot_GBps=round(live / s_us / 1e3, 1),
                                      restore_rows_us=round(r_us, 1), restore_rows_GBps=round((live + rows) / r_us / 1e3, 1),
                                      restore_us=round(r0_us, 1), restore_GBps=round(live / r0_us / 1e3, 1),
                                      fanout_512x8_envs=len(dst), fanout_us=round(f_us, 1), full_buffer_step_us=round(full, 1))), flush=True)
                P.close()


if __name__ == "__main__":
    main()
