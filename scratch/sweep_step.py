"""A/B of launch-shape variants on bench.py's headline workload: the `value` measurement of bench.py (its `measure`, L2 flushed between
steps, PREROLL steps first) for several library builds and environment knobs, alternated round by round in one call.

    python scratch/sweep_step.py --out FILE.json --rounds R --steps K NAME=LIB[:VAR=VAL,...] ...

Each (round, variant) runs in a fresh process, since the library is chosen at import (PCT_B200_LIB); the variants of a round run in a
rotated order.  Prints one line per measurement and, at the end, per variant: median / min / max of env-steps/s.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHILD = r"""
import json, sys, torch
sys.path.insert(0, %r)
import bench
cx = bench.Ctx()
cx.rank, cx.local, cx.world, cx.dist = 0, 0, 1, None
cx.dev = torch.device("cuda:0")
cx.flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=cx.dev)
cx.barrier = torch.cuda.synchronize
rec = bench.measure(cx, %d, False, %d, %d, %d, bench.PREROLL, kernels=False)
print("RESULT", json.dumps({"value": rec["value"], "ms_per_step": rec["ms_per_step"], "p50": rec["ms_per_step_p50"]}))
"""


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=100)
    ap.add_argument("--setting", type=int, default=1)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--out", default=None)
    ap.add_argument("variants", nargs="+")
    a = ap.parse_args()
    vs = []
    for v in a.variants:
        name, spec = v.split("=", 1)
        lib, _, envs = spec.partition(":")
        env = dict(kv.split("=", 1) for kv in envs.split(",")) if envs else {}
        vs.append((name, os.path.join(ROOT, lib), env))
    res = {name: [] for name, _, _ in vs}
    for r in range(a.rounds):
        order = vs[r % len(vs):] + vs[:r % len(vs)]
        for name, lib, env in order:
            e = dict(os.environ, PCT_B200_LIB=lib, **env)
            out = subprocess.run([sys.executable, "-c", CHILD % (ROOT, a.setting, a.envs, a.steps, a.warmup)], env=e, capture_output=True,
                                 text=True, cwd=ROOT)
            line = [l for l in out.stdout.splitlines() if l.startswith("RESULT ")]
            if out.returncode != 0 or not line:
                print("FAILED", name, out.returncode, out.stderr[-2000:], flush=True)
                continue
            rec = json.loads(line[0][7:])
            res[name].append(rec)
            print("round %d %-10s %.4e env-steps/s  %.4f ms/step" % (r, name, rec["value"], rec["ms_per_step"]), flush=True)
    summ = {}
    for name, recs in res.items():
        v = [x["value"] for x in recs]
        if v:
            summ[name] = {"median": statistics.median(v), "min": min(v), "max": max(v), "n": len(v),
                          "ms_median": statistics.median(x["ms_per_step"] for x in recs)}
            print("%-10s median %.4e  min %.4e  max %.4e  (%d runs)  %.4f ms/step" % (name, summ[name]["median"], summ[name]["min"],
                                                                                    summ[name]["max"], len(v), summ[name]["ms_median"]))
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"runs": res, "summary": summ}, f, indent=1)


if __name__ == "__main__":
    main()
