"""Golden vectors for ACTION ROWS THE LEAF LIST NEVER PROPOSES, recorded from the UNMODIFIED reference (needs the reference checkout,
oracle/ref_shim.py): each env is driven by the seeded placement rule of tests/rows_rule.py (valid leaves, box corners and arbitrary points
in every orientation LeafNode2Action can express, the zero row, and the odd encodings of each domain), on injected item streams with
shuffle=False, gym style (on done: the terminal observation, then reset).

Configurations: discrete 10 x 10 x 10 and the flat 12 x 7 x 9 container of harness.CASES, continuous the unit cube and the pallet bin of
harness.CONT_BINS, settings 1-3 each; plus the unit cube with the rows handed over as float32 (what a float32 policy tensor gives).

Per step: the row, the rule's kind, the observation, reward, done, counter and ratio; where the reference raises, the exception class
(err) instead (counter -1, no observation).  Each file also stores what the oracle's replay exercised (counts_*): failed real descents
that wrote loads, off-leaf successes on two or more supports, least-squares splits, raising steps.  tests/test_rows_cpu.py re-derives
them and asserts the totals (rows_rule.MIN_COUNTS).

    python tests/golden/make_golden_rows.py        -> tests/golden/rows_*.npz (deterministic: a re-run writes equal arrays)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]
import ref_shim  # noqa: E402
from harness import CONT_BINS, ITEM_SET, case_stream, cont_case_stream  # noqa: E402
from rows_rule import FLAT_ITEMS, MIN_COUNTS, make_oracle, oracle_counts_step, pick  # noqa: E402

STEPS = 250     # settings 1 and 3; setting 2 has no stability check, so its records are short (they pin the decode and the raising rows)
STEPS_S2 = 60
# rule and item seed per configuration, searched (8100-8115, 300 steps) for the most failed descents with loads and off-leaf multi-support
# successes; the env id of each configuration is its index in configs()
SEEDS = {"d_cube_s1": 8101, "d_flat_s1": 8110, "d_cube_s3": 8106, "d_flat_s3": 8100, "c_cube_s1": 8112, "c_pallet_s1": 8109,
         "c_cube_f32_s1": 8103, "c_cube_s3": 8115, "c_pallet_s3": 8100, "c_cube_f32_s3": 8108}
SEED = 8100


def configs():
    out = []
    for s in (1, 2, 3):
        out.append(("d_cube_s%d" % s, dict(domain="d", setting=s, container=(10, 10, 10), nb=80, nl=50, items=ITEM_SET)))
        out.append(("d_flat_s%d" % s, dict(domain="d", setting=s, container=(12, 7, 9), nb=70, nl=40, items=FLAT_ITEMS)))
    for s in (1, 2, 3):
        out.append(("c_cube_s%d" % s, dict(domain="c", setting=s, container=(1.0, 1.0, 1.0), nb=80, nl=50, lo=0.1, hi=0.5)))
        c = CONT_BINS["pallet_s%d" % s]
        out.append(("c_pallet_s%d" % s, dict(domain="c", setting=s, container=c["container"], nb=80, nl=50, lo=c["lo"], hi=c["hi"])))
        out.append(("c_cube_f32_s%d" % s, dict(domain="c", setting=s, container=(1.0, 1.0, 1.0), nb=80, nl=50, lo=0.1, hi=0.5, f32=True)))
    for name, c in out:
        c["seed"] = SEEDS.get(name, SEED)
        c["steps"] = STEPS_S2 if c["setting"] == 2 else STEPS
    return out


def make_ref_env(D, Cm, c, stream):
    if c["domain"] == "d":
        env = D.PackingDiscrete(setting=c["setting"], container_size=list(c["container"]), item_set=c["items"], internal_node_holder=c["nb"],
                                leaf_node_holder=c["nl"], shuffle=False)
        env.box_creator = ref_shim.make_stream_creator(D, [tuple(r) if c["setting"] == 3 else tuple(int(v) for v in r[:3]) for r in stream])
    else:
        env = Cm.PackingContinuous(setting=c["setting"], container_size=list(c["container"]), item_set=[(0.1, 0.1, 0.1)],
                                   internal_node_holder=c["nb"], leaf_node_holder=c["nl"], shuffle=False, sample_from_distribution=False)
        env.size_minimum = c["lo"]
        env.space.low_bound = c["lo"]  # = sample_left_bound of the sample_from_distribution configuration (C:bin3D.py:25-27)
        env.box_creator = ref_shim.make_stream_creator(Cm, [tuple(float(v) for v in (r if c["setting"] == 3 else r[:3])) for r in stream])
    env.test = True
    return env


def record(D, Cm, c, env_id):
    cont = c["domain"] == "c"
    n, seed = c["steps"] + 64, c["seed"]
    if cont:
        stream = cont_case_stream(dict(lo=c["lo"], hi=c["hi"], setting=c["setting"]), seed, env_id, n)
    else:
        stream = case_stream(dict(items=c["items"], setting=c["setting"]), seed, env_id, n)
    env = make_ref_env(D, Cm, c, stream)
    o = env.reset()
    rows, kinds, errs, obs, rew, done, counter, ratio = [], [], [], [o.copy()], [], [], [], []
    for t in range(c["steps"]):
        row, kind = pick(o, c["nb"], c["nl"], c["container"], cont, seed, env_id, t, f32=c.get("f32", False))
        if c.get("f32"):
            row = row.astype(np.float32)
        rows.append(row); kinds.append(kind)
        try:
            o, r, d, info = env.step(row.copy())
        except Exception as ex:  # the reference raises on this row: the episode ends there
            errs.append(type(ex).__name__); rew.append(0.0); done.append(True); counter.append(-1); ratio.append(-1.0)
            o = env.reset()
            obs.append(o.copy())
            continue
        errs.append(""); obs.append(o.copy()); rew.append(r); done.append(d)
        counter.append(info["counter"]); ratio.append(info.get("ratio", -1.0))
        if d:
            o = env.reset()
            obs.append(o.copy())
    return dict(domain=c["domain"], setting=c["setting"], container=np.array(c["container"], dtype=np.float64 if cont else np.int64), nb=c["nb"],
                nl=c["nl"], size_minimum=c["lo"] if cont else float(min(min(i) for i in c["items"])), stream=stream,
                rows=np.array(rows, dtype=np.float32 if c.get("f32") else np.float64), kind=np.array(kinds), err=np.array(errs), obs=np.array(obs),
                reward=np.array(rew, dtype=np.float64), done=np.array(done), counter=np.array(counter), ratio=np.array(ratio, dtype=np.float64))


def oracle_counts(g):
    """replay a record on the oracle (rows widened to float64) and count what it exercised"""
    orc = make_oracle(g)
    tot = dict(failed_with_loads=0, offleaf_multi=0, lstsq=0, raised=0)
    o = orc.reset()
    nb, nl = int(g["nb"]), int(g["nl"])
    for t in range(len(g["rows"])):
        row = g["rows"][t].astype(np.float64)
        lb = orc.n_lstsq
        res = orc.step(row)
        for k, v in oracle_counts_step(orc, row, o, res, nb, nl, lb).items():
            tot[k] += v
        tot["raised"] += int(res[3].get("error") == 2)
        o = orc.reset() if res[2] else res[0]
    return tot


def main():
    D, Cm = ref_shim.load_reference()
    only = sys.argv[1:]
    total = dict(failed_with_loads=0, offleaf_multi=0, lstsq=0, raised=0)
    for env_id, (name, c) in enumerate(configs()):
        path = os.path.join(HERE, "rows_%s.npz" % name)
        if only and name not in only:
            g = dict(np.load(path))
        else:
            g = record(D, Cm, c, env_id)
        cnt = oracle_counts(g)
        g.update({"counts_" + k: v for k, v in cnt.items()})
        if not only or name in only:
            np.savez_compressed(path, name=name, **{k: v for k, v in g.items() if k != "name"})
        for k, v in cnt.items():
            total[k] += v
        print(path, os.path.getsize(path) // 1024, "KiB", "episodes", int(np.sum(g["done"])), cnt, flush=True)
    print("total", total)
    for k, v in MIN_COUNTS.items():
        assert total[k] >= v, "the records exercise %s only %d times (want %d): change SEED / STEPS" % (k, total[k], v)


if __name__ == "__main__":
    main()
