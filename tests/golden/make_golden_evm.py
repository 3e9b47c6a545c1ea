"""Golden records of LNES='EVM' (EventPoint over the maintained EMS list and ZMAP), recorded from the UNMODIFIED reference (needs the
reference checkout): the env is built with LNES='EMS', so step() runs GENEMS (EMS + ZMAP upkeep), and Space.EMSPoint is rebound to
Space.EventPoint after each reset, so get_possible_position() calls EventPoint.

Per case: the item stream, the action rows (the shared test policy on the observation), and per observation a SHA-1 digest of its float64
bytes, its leaf rows (int16) and the reference's ZMAP (levels in key order, each with its four lists), flattened.  The CPU model
(tests/evm_oracle.py) runs beside the recording; `overflow_step` is the first observation on which it raises the candidate-overflow flag
(the reference has no capacity), and the record stops there.

    python tests/golden/make_golden_evm.py        -> tests/golden/evm_golden.npz
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]
import ref_shim  # noqa: E402
from evm_cases import EVM_CASES  # noqa: E402
from evm_oracle import EvmOracle  # noqa: E402
from harness import case_stream, policy_pick  # noqa: E402


def digest(obs):
    return np.frombuffer(hashlib.sha1(np.ascontiguousarray(obs, dtype=np.float64).tobytes()).digest(), dtype=np.uint8)


def flat_zmap(Z):
    """[n_levels, then per level: key, four lengths, the four lists]"""
    out = [len(Z)]
    for k, r in Z.items():
        out += [k] + [len(v) for v in r]
        for v in r:
            out += list(v)
    return np.array(out, dtype=np.int16)


def record(D, c):
    stream = case_stream(c, c["seed"], c["env"], c["steps"] + 64)
    env = D.PackingDiscrete(setting=c["setting"], container_size=list(c["container"]), item_set=c["items"], internal_node_holder=c["nb"],
                            leaf_node_holder=c["nl"], shuffle=False, LNES="EMS")
    env.box_creator = ref_shim.make_stream_creator(D, [tuple(r) if c["setting"] == 3 else tuple(int(v) for v in r[:3]) for r in stream])
    env.test = True
    model = EvmOracle(c["setting"], c["container"], c["nb"], c["nl"], stream=stream)

    def reset():
        env.reset()
        env.space.EMSPoint = env.space.EventPoint
        return np.asarray(env.cur_observation(), dtype=np.float64), model.reset()

    o, om = reset()
    rows, dig, leaves, zm = [], [], [], []
    overflow = -1
    for t in range(c["steps"] + 1):
        Z = {int(k): tuple([int(v) for v in r[q]] for q in ("x_up", "y_left", "x_bottom", "y_right")) for k, r in env.space.ZMAP.items()}
        dig.append(digest(o)); leaves.append(o.reshape(-1, 9)[c["nb"]:c["nb"] + c["nl"], :5].astype(np.int16)); zm.append(flat_zmap(Z))
        if model.flags:
            overflow = t
            break
        if t == c["steps"]:
            break
        _, row = policy_pick(o, c["nb"], c["nl"], c["seed"], c["env"], t)
        o, r, d, info = env.step(row)
        om, _, _, _ = model.step(row)
        o = np.asarray(o, dtype=np.float64)
        rows.append(row)
        if d:
            o, om = reset()
    zl = np.array([len(z) for z in zm])
    return dict(stream=stream, rows=np.array(rows), digest=np.stack(dig), leaves=np.stack(leaves), zmap=np.concatenate(zm),
                zmap_off=np.concatenate([[0], np.cumsum(zl)]), overflow_step=np.array(overflow))


def main():
    D, _ = ref_shim.load_reference()
    out = {}
    for name, c in EVM_CASES.items():
        rec = record(D, c)
        print(name, "steps", len(rec["rows"]), "overflow step", int(rec["overflow_step"]))
        for k, v in rec.items():
            out["%s/%s" % (name, k)] = v
    np.savez_compressed(os.path.join(HERE, "evm_golden.npz"), **out)


if __name__ == "__main__":
    main()
