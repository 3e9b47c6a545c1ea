"""Records item overrides on the UNMODIFIED reference -> tests/golden/items_s{1,2,3}.npz (PackingDiscrete) and citems_s{1,2,3}.npz
(PackingContinuous).  Needs /root/reference (run in the build container only).

    python tests/golden/make_item_golden.py

Each record drives the env on an injected item stream (oracle/ref_shim.py) with the deterministic test policy.  At about half the steps
it overrides the current item the way a lookahead / buffer caller of the reference does: `env.next_box = X; env.next_den = d`, then the
observation is rebuilt from the reference's own get_possible_position(), assembled as cur_observation assembles it (D:bin3D.py:70-93,
C:bin3D.py:79-99) but without gen_next_box.  The policy then picks a leaf of that observation and the env steps.

Stored per step t: `seen` (the observation the policy saw: the rebuilt one at an override), `override` / `item` (the override and its
[x, y, z, density]), `draw` (the stream position of the item that was current before the override), `rows`, `reward`, `done`, `counter`,
`ratio`, `after` (the next step's starting observation: what step returned, or the caller's reset observation after a done), and per done
`terminal` (the terminal observation step returned).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]
import ref_shim  # noqa: E402
from harness import make_stream, policy_pick  # noqa: E402
from pct_oracle import make_continuous_stream  # noqa: E402

STEPS = 200


def rebuild_observation(env):
    """cur_observation (D:bin3D.py:70-93 / C:bin3D.py:79-99) for the env's current next_box / next_den, without gen_next_box"""
    leaves = env.get_possible_position()
    env.next_box_vec[:, 3:6] = sorted(list(env.next_box))
    env.next_box_vec[:, 0] = env.next_den
    env.next_box_vec[:, -1] = 1
    return np.reshape(np.concatenate((env.space.box_vec, leaves, env.next_box_vec)), (-1))


def record(env, stream, other, setting, continuous, seed, env_id):
    rng = np.random.RandomState(seed + 17)
    o = env.reset()
    out = {k: [] for k in ("seen", "override", "item", "draw", "rows", "reward", "done", "counter", "ratio", "terminal", "after")}
    for t in range(STEPS):
        draw = env.box_creator.pos - 1  # the current item is the creator's last draw
        ov = rng.rand() < 0.5
        item = other[t] if ov else stream[draw]
        if ov:
            env.next_box = [float(v) for v in item[:3]] if continuous else [int(v) for v in item[:3]]
            env.next_den = float(item[3]) if setting == 3 else 1
            o = rebuild_observation(env)
        _, row = policy_pick(o, 80, 50, seed, env_id, t)
        seen = o.copy()
        o, r, d, info = env.step(row)
        terminal = o.copy()
        if d:
            o = env.reset()
        for k, v in (("seen", seen), ("override", ov), ("item", item), ("draw", draw), ("rows", row), ("reward", r), ("done", d),
                     ("counter", info["counter"]), ("ratio", info.get("ratio", -1.0)), ("terminal", terminal), ("after", o.copy())):
            out[k].append(v)
    out["terminal"] = [x for x, d in zip(out["terminal"], out["done"]) if d]
    return {k: np.array(v) for k, v in out.items()}


def main():
    D, Cm = ref_shim.load_reference()
    for setting in (1, 2, 3):
        seed, env_id = 3100 + setting, 4
        stream, other = make_stream(seed, env_id, STEPS + 64, setting), make_stream(seed + 1, env_id, STEPS, setting)
        env = D.PackingDiscrete(setting=setting, container_size=[10, 10, 10], item_set=[(i, j, k) for i in range(1, 6) for j in range(1, 6)
                                                                                         for k in range(1, 6)],
                                internal_node_holder=80, leaf_node_holder=50, shuffle=False)
        env.box_creator = ref_shim.make_stream_creator(D, [tuple(r) if setting == 3 else tuple(int(v) for v in r[:3]) for r in stream])
        env.test = True
        rec = record(env, stream, other, setting, False, seed, env_id)
        path = os.path.join(HERE, "items_s%d.npz" % setting)
        np.savez_compressed(path, setting=setting, stream=stream, **rec)
        print(path, os.path.getsize(path) // 1024, "KiB", "episodes", int(rec["done"].sum()), "overrides", int(rec["override"].sum()))
    for setting in (1, 2, 3):
        seed, env_id = 4100 + setting, 2
        stream, other = make_continuous_stream(seed, env_id, STEPS + 64, setting), make_continuous_stream(seed + 1, env_id, STEPS, setting)
        env = Cm.PackingContinuous(setting=setting, container_size=[1, 1, 1], item_set=[(0.1, 0.1, 0.1)], internal_node_holder=80,
                                   leaf_node_holder=50, shuffle=False, sample_from_distribution=False)
        env.size_minimum = 0.1
        env.space.low_bound = 0.1  # = sample_left_bound of the sample_from_distribution configuration (C:bin3D.py:25-27)
        env.box_creator = ref_shim.make_stream_creator(Cm, [tuple(float(v) for v in (r if setting == 3 else r[:3])) for r in stream])
        env.test = True
        rec = record(env, stream, other, setting, True, seed, env_id)
        path = os.path.join(HERE, "citems_s%d.npz" % setting)
        np.savez_compressed(path, setting=setting, stream=stream, **rec)
        print(path, os.path.getsize(path) // 1024, "KiB", "episodes", int(rec["done"].sum()), "overrides", int(rec["override"].sum()))


if __name__ == "__main__":
    main()
