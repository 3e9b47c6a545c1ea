"""Per-kernel durations of the discrete step on bench.py's headline workload, from a torch.profiler trace (CUDA activities).

    [PCT_B200_LIB=<lib>] python scratch/stage_times.py [--steps K] [--setting S] [--envs N] [--out FILE.json]

Same batch as bench.py's `value` (make_batch, PREROLL steps of the synthetic policy before anything is recorded), the L2 flushed
between steps outside the recorded kernels.  Two traced runs, each on a fresh batch: the default launch sequence (the candidates
kernel overlaps the apply kernel's tail through programmatic dependent launch, so those two durations overlap) and the serialised
one (PCT_B200_OVERLAP=0: every kernel starts after the previous one ended).  Per kernel: mean duration, launches per step, registers,
grid, block and dynamic shared memory as the trace records them.  The card's name, power limit and max SM clock are read in the
same call.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), (s.strip() for s in out.strip().split(","))))


def traced(setting, n, K, overlap):
    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    if overlap is not None:
        os.environ["PCT_B200_OVERLAP"] = "1" if overlap else "0"
    batch = bench.make_batch(setting, False, n, 0, 0)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda:0")
    batch.reset()
    T0 = bench.PREROLL + 64
    for t in range(T0):
        batch.step(leaf_idx=batch.random_policy(bench.POLICY_SEED, t))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for t in range(K):
            flush.zero_()
            batch.step(leaf_idx=batch.random_policy(bench.POLICY_SEED, T0 + t))
        torch.cuda.synchronize()
    batch.close()
    os.environ.pop("PCT_B200_OVERLAP", None)
    fd, path = tempfile.mkstemp(suffix=".json")
    os.close(fd)
    prof.export_chrome_trace(path)
    with open(path) as f:
        ev = json.load(f)["traceEvents"]
    os.remove(path)
    kern = sorted((e for e in ev if e.get("cat") == "kernel" and "pct" in e["name"]), key=lambda e: e["ts"])
    rows = {}
    for e in kern:
        name = e["name"].split("(")[0].replace("void ", "").replace("pct::", "")
        a = e["args"]
        r = rows.setdefault(name, {"n": 0, "us": 0.0, "regs": a.get("registers per thread"), "grid": a.get("grid"), "block": a.get("block"),
                                   "smem": a.get("shared memory"), "first_ts": e["ts"]})
        r["n"] += 1
        r["us"] += e["dur"]
    # step span: first kernel start of a step to the last kernel end, per step (steps are separated by the flush memset)
    spans, cur = [], None
    for e in sorted((e for e in ev if e.get("cat") == "kernel"), key=lambda e: e["ts"]):
        if "pct" not in e["name"]:
            if cur:
                spans.append(cur[1] - cur[0])
            cur = None
            continue
        cur = [e["ts"], e["ts"] + e["dur"]] if cur is None else [cur[0], max(cur[1], e["ts"] + e["dur"])]
    if cur:
        spans.append(cur[1] - cur[0])
    out = []
    for name, r in sorted(rows.items(), key=lambda kv: kv[1]["first_ts"]):
        out.append({"kernel": name, "ms_mean": r["us"] / r["n"] / 1e3, "per_step": r["n"] / K, "regs": r["regs"], "grid": r["grid"],
                    "block": r["block"], "smem": r["smem"]})
    return {"kernels": out, "step_span_ms_mean": sum(spans) / len(spans) / 1e3 if spans else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--setting", type=int, default=1)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import pct_b200
    doc = {"card": card(), "lib": pct_b200.LIB_PATH, "setting": a.setting, "envs": a.envs, "steps": a.steps,
           "default": traced(a.setting, a.envs, a.steps, None), "serialised": traced(a.setting, a.envs, a.steps, False)}
    print("card:", json.dumps(doc["card"]))
    for mode in ("default", "serialised"):
        print("%s launch sequence: step span %.4f ms (first kernel start to last kernel end, mean)" % (mode, doc[mode]["step_span_ms_mean"]))
        for k in doc[mode]["kernels"]:
            print("  %-48s %8.4f ms  x%.2f/step  regs %-4s grid %-16s block %-14s smem %s" % (
                k["kernel"][:48], k["ms_mean"], k["per_step"], k["regs"], k["grid"], k["block"], k["smem"]))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
