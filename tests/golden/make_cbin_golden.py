"""Golden vectors of the continuous env on containers other than the unit cube (harness.CONT_BINS: a 1.2 x 0.8 x 1.0 pallet, the
reference constructor's 10 x 10 x 10 default, a 2400 x 1700 x 2300 bin in millimetres), recorded from the UNMODIFIED reference (needs
the reference checkout, oracle/ref_shim.py).  One file per bin and setting, tests/golden/cbin_<bin>_s<setting>.npz, holding

  t0_* / t1_*   two step trajectories under the shared policy (the format of make_golden_cases.record_cont_case, keys prefixed)
  h_stream, len_<name>, flat_<name>
                EPISODES episodes of heuristic.py's LASH / OnlineBPH / BR on one stream, the env's item_set being the 125 sizes
                scaled by the min side (BR counts the sizes that fit), in the format of make_heuristic_golden_continuous.py
  q, q_step, q_den, q_feas, q_h
                answers of Space.drop_box_virtual(dims, (lx, ly), False, density, setting, returnH=True) at the states before
                the steps q_step of trajectory t0: placements at W, L and H and 5e-7 / 2e-6 either side of them (each axis on
                its own), positions just below 0, zero sizes

    python tests/golden/make_cbin_golden.py [name ...]      -> tests/golden/cbin_*.npz (deterministic: a re-run writes equal arrays)
"""
import contextlib
import io
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), HERE):
    sys.path.insert(0, p)
import ref_shim  # noqa: E402
from harness import CONT_BINS, cont_case_stream, cont_item_set  # noqa: E402
from make_golden_cases import record_cont_case  # noqa: E402

TRAJ = ((601, 1), (602, 4))  # (items / policy seed, env id) of t0 and t1
EPISODES, H_SEED, H_ENV, H_LEN = 4, 9191, 3, 600
PROBE_STEPS = tuple(range(3, 70, 7))  # 10 states of t0
DELTAS = (0.0, 5e-7, -5e-7, 2e-6, -2e-6)


def make_env(Cm, c, stream, cls=None, item_set=None):
    """the reference env of record_cont_case, on an injected stream"""
    env = (cls or Cm.PackingContinuous)(setting=c["setting"], container_size=list(c["container"]), item_set=item_set or [(0.1, 0.1, 0.1)],
                                        internal_node_holder=c["nb"], leaf_node_holder=c["nl"], shuffle=False, sample_from_distribution=False)
    env.size_minimum = c["low"]
    env.space.low_bound = c["low"]  # = sample_left_bound of the sample_from_distribution configuration (C:bin3D.py:25-27)
    env.box_creator = ref_shim.make_stream_creator(Cm, [tuple(float(v) for v in (r if c["setting"] == 3 else r[:3])) for r in stream])
    env.test = True
    return env


def probe_set(env, c):
    """placements for the env's current item at its current state: at the three highest EMS corners, lx + sx / ly + sy / mh + sz at
    W / L / H and DELTAS away from them (one axis at a time), lx / ly just below 0, each size zero once, the corner itself (both yaws)"""
    W, L, H = c["container"]
    d = [float(v) for v in env.next_box]
    ems = [[float(v) for v in e] for e in env.space.EMS]
    q = []
    for i in sorted(range(len(ems)), key=lambda i: (-ems[i][2], i))[:3]:
        x0, y0 = ems[i][0], ems[i][1]
        q += [d + [x0, y0], [d[1], d[0], d[2], x0, y0]]
        for dl in DELTAS:
            q.append(d + [W - d[0] + dl, y0])
            q.append(d + [x0, L - d[1] + dl])
        _, mh = env.space.drop_box_virtual(d, (x0, y0), False, env.next_den, env.setting, returnH=True)
        for dl in DELTAS:
            q.append([d[0], d[1], H - mh + dl, x0, y0])
        for dl in (-5e-7, -2e-6):
            q.append(d + [dl, y0])
            q.append(d + [x0, dl])
        q += [[0.0, d[1], d[2], x0, y0], [d[0], 0.0, d[2], x0, y0], [d[0], d[1], 0.0, x0, y0]]
    return q


def record_probes(Cm, c, rec):
    """replays t0's rows on a fresh reference env and asks it the probe_set placements before each step of PROBE_STEPS"""
    env = make_env(Cm, c, rec["stream"])
    env.reset()
    out = dict(q=[], q_step=[], q_den=[], q_feas=[], q_h=[])
    for t, row in enumerate(rec["rows"]):
        if t in PROBE_STEPS:
            for x in probe_set(env, c):
                ok, mh = env.space.drop_box_virtual(list(x[:3]), (x[3], x[4]), False, env.next_den, env.setting, returnH=True)
                out["q"].append(x); out["q_step"].append(t); out["q_den"].append(float(env.next_den))
                out["q_feas"].append(bool(ok)); out["q_h"].append(float(mh))
        _, _, d, _ = env.step(row)
        if d:
            env.reset()
    return dict(q=np.array(out["q"], dtype=np.float64), q_step=np.array(out["q_step"]), q_den=np.array(out["q_den"]),
                q_feas=np.array(out["q_feas"]), q_h=np.array(out["q_h"]))


def record_heuristics(Cm, H, c):
    class Recording(Cm.PackingContinuous):
        def reset(self):
            if hasattr(self, "packed"):
                self.log.append([list(map(float, p)) for p in self.packed])
            return super().reset()

    stream = cont_case_stream(c, c.get("hseed", H_SEED + c["setting"]), H_ENV, H_LEN)
    rec = dict(h_stream=stream)
    for name, fn in (("LSAH", H.LASH), ("OnlineBPH", H.OnlineBPH), ("BR", H.BR)):
        env = make_env(Cm, c, stream, cls=Recording, item_set=cont_item_set(c))
        env.log = []
        with contextlib.redirect_stdout(io.StringIO()):
            fn(env, EPISODES)
        eps = env.log[:EPISODES]
        assert len(eps) == EPISODES and env.box_creator.pos < H_LEN
        rec["len_" + name] = np.array([len(e) for e in eps])
        rec["flat_" + name] = np.array([p for e in eps for p in e], dtype=np.float64).reshape(-1, 7)
    return rec


def main():
    _, Cm = ref_shim.load_reference()
    only = sys.argv[1:]
    sys.argv = [sys.argv[0]]
    import heuristic as H  # the reference module, unmodified
    for name, c in CONT_BINS.items():
        if only and name not in only:
            continue
        out = dict(name=name)
        for k, (seed, env_id) in enumerate(TRAJ):
            rec = record_cont_case(Cm, c, seed, env_id)
            if k == 0:
                out.update(record_probes(Cm, c, rec))
            out.update({"t%d_%s" % (k, f): v for f, v in rec.items()})
        out.update(record_heuristics(Cm, H, c))
        path = os.path.join(HERE, "cbin_%s.npz" % name)
        np.savez_compressed(path, **out)
        print(path, os.path.getsize(path) // 1024, "KiB", "episodes", int(out["t0_done"].sum()), int(out["t1_done"].sum()),
              "boxes", max(int(out["t0_counter"].max()), int(out["t1_counter"].max())),
              "heuristic lengths", [out["len_" + n].tolist() for n in ("LSAH", "OnlineBPH", "BR")],
              "probes", len(out["q"]), "feasible", int(out["q_feas"].sum()), flush=True)


if __name__ == "__main__":
    main()
