"""Snapshot / restore throughput (pct_snapshot / pct_restore) on mid-episode batches, next to one pct_step of the same batch.

For 4096 and 8192 envs of both domains (setting 1), after 100 random-policy steps: CUDA-event timing of CUDA-graph replays of many calls of
  snapshot of every env, restore of every env (with and without observation rows), fan-out of 512 parents x 8 children,
and one pct_step.  Bytes moved are computed from the live counts in the records (read + write of the live parts; plus the observation
rows written), and reported as GB/s and as a fraction of the H100 SXM data-sheet bandwidth (3.35 TB/s).  Prints the card and its power
limit in the same run.  python scratch/bench_snapshot.py [--iters 50]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pct_b200  # noqa: E402

PEAK = 3.35e12
ITEMS = [(i, j, k) for i in range(1, 6) for j in range(1, 6) for k in range(1, 6)]
# header fields of a record (pct_snapshot.cu): the env header starts at byte 16 with n_box, n_ems, n_leaf; n_edge / n_poly per domain
EDGE_POLY_OFF = {False: (16 + 44, 16 + 68), True: (16 + 80, 16 + 84)}


def live_bytes(snap, continuous, alias):
    """bytes of the live parts of every record (what one gather reads, or one scatter writes)"""
    r = snap.cpu().numpy()
    i32 = lambda off: r[:, off:off + 4].copy().view(np.int32)[:, 0].astype(np.int64)  # noqa: E731
    nb, ne, nl = i32(16), i32(20), i32(24)
    ned, npo = i32(EDGE_POLY_OFF[continuous][0]), i32(EDGE_POLY_OFF[continuous][1])
    if continuous:
        b = 16 + 88 + nb * 48 + nb * 8 + ne * 48 + 2 * (nb + 1) * 2 + 2 * ned + 2 * nb + ned * 32 + npo * 16 + nl * 48 + 32
    else:
        b = 16 + 80 + nb * 12 + ne * 12 + 2 * (nb + 1) * 2 + 2 * ned + 2 * nb + nl * 12 + nb * 8 + ned * 32 + npo * 16 + 16
    if alias:
        b = b + nb * 32 + ned + (ned + 31) // 32 * 4
    return b


def timed(fn, iters, graph=True):
    """seconds per call: `iters` calls captured in one CUDA graph and replayed (no host overhead in the number); graph=False: eager calls"""
    fn()
    torch.cuda.synchronize()
    a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if graph:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(iters):
                fn()
        g.replay()
        torch.cuda.synchronize()
        a.record()
        for _ in range(5):
            g.replay()
        z.record()
        torch.cuda.synchronize()
        return a.elapsed_time(z) / (5 * iters) * 1e-3
    a.record()
    for _ in range(iters):
        fn()
    z.record()
    torch.cuda.synchronize()
    return a.elapsed_time(z) / iters * 1e-3


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                            timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        pl = "unavailable (%s)" % e
    return name, pl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    name, pl = card()
    print(json.dumps(dict(card=name, power_limit=pl)))
    for continuous in (False, True):
        for n in (4096, 8192):
            if continuous:
                b = pct_b200.PctBatch(n, 1, container_size=(1.0, 1.0, 1.0), continuous=True, sample_from_distribution=True, seed=1234)
            else:
                b = pct_b200.PctBatch(n, 1, item_set=ITEMS, seed=1234)
            b.reset()
            for t in range(100):
                _, _, _, info = b.step(leaf_idx=b.random_policy(4321, t))
            b.check_flags(info[:, 1].cpu().numpy())
            snap = b.snapshot()
            live = live_bytes(snap, continuous, alias=True)
            obs_row = b.obs_len * 4
            buf = torch.empty_like(snap)
            t_snap = timed(lambda: b.snapshot(out=buf), args.iters)
            t_rest = timed(lambda: b.restore(snap, write_obs=False), args.iters)
            t_rest_obs = timed(lambda: b.restore(snap), args.iters)
            parents = snap[torch.arange(0, n, n // 512, device=snap.device)][:512].contiguous()
            rec = torch.arange(512, dtype=torch.int32, device=snap.device).repeat_interleave(8)
            env = torch.arange(4096, dtype=torch.int32, device=snap.device)
            # the C call itself: PctBatch.restore would add its device-side range check of rec_idx (one elementwise kernel) to the number
            fan = lambda: b.L.pct_restore(b.h, C.c_void_p(env.data_ptr()), C.c_void_p(rec.data_ptr()), 4096, C.c_void_p(parents.data_ptr()),  # noqa: E731
                                          C.c_void_p(b._obs.data_ptr()), b._stream())
            t_fan = timed(fan, args.iters)
            live_par = live_bytes(parents, continuous, alias=True)
            idx = b.random_policy(4321, 100).clone()
            t_step = timed(lambda: b.step(leaf_idx=idx), 20, graph=False)  # eager, as bench.py steps
            rows = []
            for what, sec, moved in (("snapshot", t_snap, 2 * live.sum()), ("restore", t_rest, 2 * live.sum()),
                                     ("restore+obs", t_rest_obs, 2 * live.sum() + n * obs_row),
                                     ("fanout512x8", t_fan, 8 * 2 * live_par.sum() + 4096 * obs_row)):
                rows.append(dict(op=what, us=round(sec * 1e6, 1), MB=round(moved / 1e6, 2), GBps=round(moved / sec / 1e9, 1),
                                 frac_peak=round(moved / sec / PEAK, 3)))
            print(json.dumps(dict(domain="continuous" if continuous else "discrete", setting=1, n_envs=n, record_bytes=b.snapshot_bytes,
                                  mean_live_bytes=int(live.mean()), step_us=round(t_step * 1e6, 1), ops=rows)))
            b.close()


if __name__ == "__main__":
    main()
