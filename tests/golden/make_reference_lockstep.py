"""Records what tests/test_oracle_vs_reference.py compares the C oracle against, from the UNMODIFIED reference (needs a checkout of
alexfrom0815/Online-3D-BPP-PCT; ref_shim.REFERENCE_ROOT, set with PCT_REFERENCE_ROOT):

  * the default-configuration lock-step of settings 1-3 (260 steps, the reference's observations, rewards, done flags and infos),
  * the non-default configurations on fresh seeds (the recorders of make_golden_cases.py: observations, rewards, done flags, ...),
  * the geometric tie of the one known divergence (the reference's verdicts with LAPACK and with the oracle's solver),
  * the reference's convex hull / point-in-polygon results for tests/test_oracle_units.py.

Observations and hulls are stored as 64-bit digests (obs_digest below) so that the whole record stays small.  The actions are not stored:
the policy (policy_pick) is a function of the observation, so equal observations give the oracle the reference's actions.

    python tests/golden/make_reference_lockstep.py        -> tests/golden/reference_lockstep.npz
"""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), HERE]
PATH = os.path.join(HERE, "reference_lockstep.npz")

LOCKSTEP_STEPS, CASE_STEPS, CONT_CASE_STEPS, TIE_STEPS = 260, 60, 70, 47
TIE_SEED, TIE_ENV = 135409, 0
HULL_TRIALS = 600


def obs_digest(o):
    """first 8 bytes of the SHA-1 of the observation as float64, as an unsigned 64-bit integer"""
    return np.frombuffer(hashlib.sha1(np.ascontiguousarray(o, dtype=np.float64).tobytes()).digest()[:8], dtype=np.uint64)[0]


def info_text(info):
    return json.dumps({k: float(v) if isinstance(v, float) else v for k, v in info.items()}, sort_keys=True)


def hull_trials():
    """the random point sets and query points of test_hull_and_pip_match_reference_module, in its draw order"""
    rng = np.random.RandomState(3)
    for _ in range(HULL_TRIALS):
        k = rng.choice([1, 1, 2, 2, 3, 4, 6])
        pts = []
        for _ in range(k):
            x1, y1 = rng.randint(0, 8, 2); x2, y2 = x1 + rng.randint(1, 4), y1 + rng.randint(1, 4)
            pts += [[x1, y1], [x1, y2], [x2, y1], [x2, y2]]
        qs = []
        for _ in range(6):
            qs.append(np.array([rng.randint(0, 20) / 2.0, rng.randint(0, 20) / 2.0]) if rng.rand() < 0.5 else rng.uniform(0, 10, 2))
        yield pts, qs


def record_lockstep(D, setting):
    import ref_shim
    from harness import ITEM_SET, make_stream, policy_pick
    seed, env_id = 900 + setting, 3
    stream = make_stream(seed, env_id, LOCKSTEP_STEPS + 64, setting)
    ref = D.PackingDiscrete(setting=setting, container_size=[10, 10, 10], item_set=ITEM_SET, internal_node_holder=80,
                            leaf_node_holder=50, shuffle=False, LNES="EMS")
    ref.box_creator = ref_shim.make_stream_creator(D, [tuple(r) if setting == 3 else tuple(int(v) for v in r[:3]) for r in stream])
    ref.test = True
    o = ref.reset()
    obs, rew, done, info = [obs_digest(o)], [], [], []
    for t in range(LOCKSTEP_STEPS):
        _, row = policy_pick(o, 80, 50, seed, env_id, t)
        o, r, d, i = ref.step(row)
        obs.append(obs_digest(o)); rew.append(r); done.append(d); info.append(info_text(i))
        if d:
            o = ref.reset()
            obs.append(obs_digest(o))
    return {"obs": np.array(obs), "reward": np.array(rew, dtype=np.float64), "done": np.array(done), "info": np.array(info)}


def record_tie(D):
    """the lock-step prefix of the known divergence and the reference's verdicts on the tie, with LAPACK and with the oracle's solver"""
    import ref_shim
    from harness import CASES, case_stream, policy_pick
    from pct_oracle import _dp, lib
    import pct_envs.PctDiscrete0.space as SP
    c = CASES["holders_s1"]
    stream = case_stream(c, TIE_SEED, TIE_ENV, 200)
    ref = D.PackingDiscrete(setting=1, container_size=[10, 10, 10], item_set=c["items"], internal_node_holder=c["nb"], leaf_node_holder=c["nl"],
                            shuffle=False, LNES="EMS")
    ref.box_creator = ref_shim.make_stream_creator(D, [tuple(int(v) for v in r[:3]) for r in stream])
    ref.test = True
    o = ref.reset()
    pre = []
    for t in range(TIE_STEPS):
        pre.append(obs_digest(o))
        _, row = policy_pick(o, c["nb"], c["nl"], TIE_SEED, TIE_ENV, t)
        o, _, d, _ = ref.step(row)
        if d:
            o = ref.reset()
    final = obs_digest(o)
    lapack, L = np.linalg.lstsq, lib()
    seen = []

    def with_oracle_solver(A, b, rcond=None):
        r = lapack(A, b, rcond=rcond)
        x = np.zeros(A.shape[1])
        L.pcto_lstsq(_dp(np.ascontiguousarray(A, dtype=float)), A.shape[0], A.shape[1], _dp(np.ascontiguousarray(np.array(b, dtype=float).reshape(-1))), _dp(x))
        seen.append(np.abs(r[0].reshape(-1) - x).max())
        return (x.reshape(-1, 1),) + tuple(r[1:])

    args = ([4, 2, 1], (5, 0), False, ref.next_den, 1)
    with_lapack = ref.space.drop_box_virtual(*args)
    SP.np.linalg.lstsq = with_oracle_solver
    try:
        flipped = ref.space.drop_box_virtual(*args)
    finally:
        SP.np.linalg.lstsq = lapack
    return {"pre": np.array(pre), "final": np.array([final]), "with_lapack": np.array([bool(with_lapack)]),
            "with_oracle_solver": np.array([bool(flipped)]), "solver_gap": np.array(seen, dtype=np.float64)}


def record_hulls(D):
    from pct_envs.PctDiscrete0.convex_hull import ConvexHull, point_in_polygen
    from pct_envs.PctDiscrete0.space import Space
    sp = Space(10, 10, 10, 1, 80)
    counts, digests, pip = [], [], []
    for pts, qs in hull_trials():
        want = np.array(sp.scale_down(ConvexHull([list(p) for p in pts])), dtype=np.float64).reshape(-1, 2)
        counts.append(len(want)); digests.append(obs_digest(want))
        pip.append([bool(point_in_polygen(q, want.tolist())) for q in qs])
    return {"count": np.array(counts, dtype=np.int32), "digest": np.array(digests), "pip": np.array(pip)}


def main():
    import ref_shim
    import make_golden_cases as M
    from harness import CASES, CONT_CASES
    D, Cm = ref_shim.load_reference()
    out = {}
    for s in (1, 2, 3):
        for k, v in record_lockstep(D, s).items():
            out["lockstep_s%d_%s" % (s, k)] = v
    for name, c in sorted(CASES.items()):
        rec = M.record_case(D, dict(c, steps=CASE_STEPS), 8800, 4)
        for k in ("reward", "done", "counter", "ratio"):
            out["case_%s_%s" % (name, k)] = rec[k]
        out["case_%s_obs" % name] = np.array([obs_digest(o) for o in rec["obs"]])
    for name, c in sorted(CONT_CASES.items()):
        rec = M.record_cont_case(Cm, dict(c, steps=CONT_CASE_STEPS), 8801, 5)
        for k in ("reward", "done", "counter", "ratio"):
            out["ccase_%s_%s" % (name, k)] = rec[k]
        out["ccase_%s_obs" % name] = np.array([obs_digest(o) for o in rec["obs"]])
    for k, v in record_tie(D).items():
        out["tie_" + k] = v
    for k, v in record_hulls(D).items():
        out["hull_" + k] = v
    np.savez_compressed(PATH, **out)
    print(PATH, os.path.getsize(PATH) // 1024, "KiB")


if __name__ == "__main__":
    main()
