"""Launch sequence of every public call, for comparing two builds of the library (PCT_B200_LIB selects the one under test).

Runs a fixed call sequence per configuration (both domains, settings 1-3, float32 / float64 observations, the defaults and the launch
variants) under torch.profiler and writes, per call, the kernels it enqueued (name, grid, block, dynamic shared memory, registers) in
stream order per stream, pct_kernel_launches after the call, and a digest of what the call produced.  Two builds that enqueue the same
kernels the same way and compute the same results give identical files.
    PCT_B200_LIB=<lib> python scratch/launch_trace.py <out.json>
"""
import hashlib
import json
import os
import sys

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pct_b200  # noqa: E402

N = 1030  # >= 1024: the staged pct_step_host path cuts the discrete batch into 4 uneven env ranges
D_ITEMS = [(i, j, k) for i in range(1, 6) for j in range(1, 6) for k in range(1, 6)]
C_ITEMS = [(0.1 * i, 0.1 * j, 0.1 * k) for i in range(1, 6) for j in range(1, 6) for k in range(1, 6)]
VARIANTS = [{}, {"PCT_B200_OVERLAP": "0"}, {"PCT_B200_OVERLAP_CONT": "1"}, {"PCT_B200_K3": "block"}, {"PCT_B200_WALK": "fork"},
            {"PCT_B200_GROUPS": "2"}]


def digest(*xs):
    h = hashlib.sha1()
    for x in xs:
        if torch.is_tensor(x):
            x = x.detach().cpu().numpy()
        if isinstance(x, dict):
            for k in sorted(x):
                h.update(k.encode())
                h.update(digest(x[k]).encode())
        elif isinstance(x, np.ndarray):
            h.update(np.ascontiguousarray(x).tobytes())
        else:
            h.update(repr(x).encode())
    return h.hexdigest()[:16]


def calls(b, cont, setting):
    """(name, fn) pairs; fn runs one public call and returns what it produced"""
    dev, n = b.device, b.n_envs
    ft = b.obs_dtype
    idx0 = torch.zeros(n, dtype=torch.int32, device=dev)
    pin = lambda a: torch.from_numpy(a).pin_memory().numpy()
    host = lambda: (np.zeros((n, b.obs_len), dtype=np.float64 if ft == torch.float64 else np.float32), np.zeros(n, np.float32),
                    np.zeros(n, np.uint8), np.zeros((n, 8), np.int32))

    def step_host(pinned):
        o, r, d, i = host()
        if pinned:
            o, r, d, i = pin(o), pin(r), pin(d), pin(i)
        b.step_host(o, r, d, i, leaf_idx=np.zeros(n, np.int32))
        return digest(o, r, d, i)

    def step_actions():
        rows = b._obs.view(n, -1, 9)[:, b.nb, :].contiguous()  # each env's first leaf row
        return digest(*b.step(actions=rows))

    def captured_step():
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            b.step(leaf_idx=idx0)
        g.replay()
        return digest(b._obs, b._rew, b._done, b._info)

    def snapshot_restore():
        snap = b.snapshot(out=torch.zeros((n, b.snapshot_bytes), dtype=torch.uint8, device=dev))
        b.step(leaf_idx=idx0)
        return digest(snap, b.restore(snap))

    sz = (lambda v: 0.1 * v) if cont else (lambda v: v)
    q = torch.tensor([[[sz(2), sz(3), sz(1), sz(j), sz(k)] for j in range(3) for k in range(2)] for _ in range(8)], dtype=torch.float64)
    heur = ["LSAH", "OnlineBPH", "BR"] if cont else ["LSAH", "OnlineBPH", "BR", "MACS", "DBL", "HM", "RANDOM"]
    out = [("reset", lambda: digest(b.reset()))]
    for t in range(4):
        out.append(("step_leaf_%d" % t, lambda t=t: digest(*b.step(leaf_idx=b.random_policy(11, t).clone()))))
    out += [
        ("step_actions", step_actions),
        ("step_leaf", lambda: digest(*b.step(leaf_idx=idx0))),
        ("step_host_pinned", lambda: step_host(True)),
        ("step_host_unpinned", lambda: step_host(False)),
        ("random_policy", lambda: digest(b.random_policy(3, 9))),
        ("set_items", lambda: digest(b.set_items([[sz(2), sz(2), sz(3)]] * 4, env_idx=[0, 2, 4, 6]), b._info)),
        ("reset_env_idx", lambda: digest(b.reset(env_idx=[1, 3, 5]))),
        ("reset_mask", lambda: digest(b.reset(mask=(torch.arange(n, device=dev) % 7 == 0)))),
        ("preview_items", lambda: digest(b.preview_items(k=3))),
        ("query_placements", lambda: digest(*b.query_placements(q, env_idx=list(range(0, 16, 2))))),
        ("query_placement", lambda: digest(b.query_placement(1, (sz(2), sz(2), sz(2)), sz(1), sz(1)))),
    ]
    if not cont:
        out.append(("height_maps", lambda: digest(b.height_maps(env_idx=[0, 5, 9]))))
        out.append(("random_policy_dev", lambda: digest(b.random_policy_dev(3, torch.tensor([4], dtype=torch.int64, device=dev)))))
    for name in heur:
        out.append(("heuristic_" + name, lambda name=name: digest(b.heuristic_actions(name, seed=2, t=1))))
    out += [
        ("snapshot_restore", snapshot_restore),
        ("captured_step", captured_step),
        ("state", lambda: digest(b.state(0), b.state(n - 1))),
        ("support_graph", lambda: digest(b.support_graph(0), b.support_graph(7))),
    ]
    return out


def run_config(cont, setting, ft, env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        if cont:
            b = pct_b200.PctBatch(N, setting, container_size=(1.0, 1.0, 1.0), item_set=C_ITEMS, continuous=True, obs_dtype=ft, seed=5)
        else:
            b = pct_b200.PctBatch(N, setting, item_set=D_ITEMS, obs_dtype=ft, seed=5)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    seq = calls(b, cont, setting)
    results = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for name, fn in seq:
            torch.cuda.synchronize()
            torch.cuda._sleep(1000)  # marker kernel: splits the trace into calls
            torch.cuda.synchronize()
            produced = fn()
            torch.cuda.synchronize()
            results.append({"call": name, "launches": b.kernel_launches, "digest": produced})
        torch.cuda._sleep(1000)
        torch.cuda.synchronize()
    b.close()
    path = "/tmp/launch_trace_%d.json" % os.getpid()
    prof.export_chrome_trace(path)
    with open(path) as f:
        ev = json.load(f)["traceEvents"]
    os.remove(path)
    kern = sorted((e for e in ev if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    groups, cur = [], None
    for e in kern:
        if "spin_kernel" in e["name"]:
            cur = []
            groups.append(cur)
        elif cur is not None:
            cur.append(e)
    assert len(groups) == len(results) + 1, (len(groups), len(results))
    for r, g in zip(results, groups):
        streams = {}
        for e in g:
            if "pct" not in e["name"]:
                continue  # torch's own kernels of the Python wrapper
            a = e["args"]
            streams.setdefault(a.get("stream"), []).append([e["name"], a.get("grid"), a.get("block"), a.get("shared memory"),
                                                            a.get("registers per thread")])
        r["kernels"] = sorted(streams.values())
    return results


def main():
    out = sys.argv[1]
    configs = []
    for cont in (False, True):
        for setting in (1, 2, 3):
            for ft in (torch.float32, torch.float64):
                configs.append((cont, setting, ft, {}))
            for vi, env in enumerate(VARIANTS[1:]):
                configs.append((cont, setting, torch.float64 if (vi + setting) % 2 else torch.float32, env))
    doc = []
    for cont, setting, ft, env in configs:
        tag = {"domain": "continuous" if cont else "discrete", "setting": setting, "obs": str(ft), "env": env}
        doc.append({"config": tag, "calls": run_config(cont, setting, ft, env)})
        print(json.dumps(tag), "calls:", len(doc[-1]["calls"]), "kernels:", sum(len(s) for c in doc[-1]["calls"] for s in c["kernels"]), flush=True)
    with open(out, "w") as f:
        json.dump({"lib": pct_b200.LIB_PATH, "configs": doc}, f, indent=0)


if __name__ == "__main__":
    main()
