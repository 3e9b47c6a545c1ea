"""Records what two host-logic tests of tests/test_host_logic.py compare the drop-in vector surface against, from the UNMODIFIED reference
(needs a checkout of alexfrom0815/Online-3D-BPP-PCT; ref_shim.REFERENCE_ROOT, set with PCT_REFERENCE_ROOT):

  * test_vec_env_equals_reference_shmem_vecpytorch_monitor: 70 vector steps of the reference's VecPyTorch(ShmemVecEnv([Monitor(PackingDiscrete)]
    * 5)) stack (envs.py:75-116,159-182, wrapper/shmem_vec_env.py, wrapper/monitor.py) on the seeded item streams of the test — observation
    digests, reward / done arrays with their dtypes, and per env the info keys, counter and, on terminal steps, ratio / reward / Monitor's
    episode length and return;
  * test_make_vec_envs_takes_the_reference_args: the namespaces tools.get_args() builds from the test's command lines.

    python tests/golden/make_reference_surface.py        -> tests/golden/reference_surface.npz
"""
import importlib
import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), HERE]
PATH = os.path.join(HERE, "reference_surface.npz")

VEC_ENVS, VEC_STEPS = 5, 70
ARGVS = {"discrete": ["--setting", "1", "--num-processes", "6", "--seed", "9"],
         "continuous": ["--setting", "2", "--continuous", "--sample-from-distribution", "--num-processes", "4"]}


def vec_streams(setting):
    from harness import make_stream
    return np.stack([make_stream(50 + setting, e, 300, setting) for e in range(VEC_ENVS)])


def vec_rows(obs, setting, t):
    """the leaf rows both stacks are stepped with: float32 numpy, as train_tools.py:66-67 passes them"""
    from harness import policy_pick
    return np.stack([policy_pick(obs[e].astype(np.float64), 80, 50, 50 + setting, e, t)[1] for e in range(VEC_ENVS)]).astype(np.float32)


def info_record(info, done):
    rec = {"keys": sorted(info), "counter": int(info["counter"])}
    if done:
        rec.update(ratio=float(info["ratio"]), reward=float(info["reward"]), l=int(info["episode"]["l"]), r=float(info["episode"]["r"]))
    return rec


def record_vec_env(D, setting, log_dir):
    import ref_shim
    from harness import ITEM_SET
    renvs = importlib.import_module("envs")
    ShmemVecEnv = importlib.import_module("wrapper.shmem_vec_env").ShmemVecEnv
    Monitor = importlib.import_module("wrapper.monitor").Monitor
    from make_reference_lockstep import obs_digest
    streams = vec_streams(setting)

    def thunk(rank):
        def _t():
            env = D.PackingDiscrete(setting=setting, container_size=[10, 10, 10], item_set=ITEM_SET, internal_node_holder=80, leaf_node_holder=50,
                                    shuffle=False, LNES="EMS")
            env.box_creator = ref_shim.make_stream_creator(D, [tuple(int(v) for v in r[:3]) for r in streams[rank]])
            env.test = True
            return Monitor(env, os.path.join(log_dir, str(rank)), allow_early_resets=True)
        return _t

    probe = D.PackingDiscrete(setting=setting, container_size=[10, 10, 10], item_set=ITEM_SET)
    ref = renvs.VecPyTorch(ShmemVecEnv([thunk(r) for r in range(VEC_ENVS)], [probe.observation_space, probe.action_space], context="fork"), "cpu")
    try:
        o = ref.reset()
        dtypes = {"obs": str(o.dtype), "obs_shape": list(o.shape)}
        obs, rew, done, infos = [obs_digest(o.numpy())], [], [], []
        for t in range(VEC_STEPS):
            o, r, d, i = ref.step(vec_rows(o.numpy(), setting, t))
            dtypes.update(reward=str(r.dtype), reward_shape=list(r.shape), done=str(d.dtype))
            obs.append(obs_digest(o.numpy())); rew.append(r.numpy()[:, 0]); done.append(d)
            infos.append(json.dumps([info_record(i[e], d[e]) for e in range(VEC_ENVS)]))
    finally:
        ref.close()
    return {"obs": np.array(obs), "reward": np.array(rew), "done": np.array(done), "info": np.array(infos), "dtypes": np.array(json.dumps(dtypes))}


def record_args():
    import ref_shim
    compat = importlib.import_module("pct_b200.compat")
    out = {}
    for name, argv in ARGVS.items():
        out[name] = vars(compat.reference_args(ref_shim.REFERENCE_ROOT, argv))
    return json.dumps(out)


def main():
    import ref_shim
    D, _ = ref_shim.load_reference()
    out = {"args": np.array(record_args())}
    with tempfile.TemporaryDirectory() as log_dir:
        for setting in (1, 2):
            for k, v in record_vec_env(D, setting, log_dir).items():
                out["vec_s%d_%s" % (setting, k)] = v
    np.savez_compressed(PATH, **out)
    print(PATH, os.path.getsize(PATH) // 1024, "KiB")


if __name__ == "__main__":
    main()
