"""Batched evaluation over a trajectory dataset (SURVEY.md §8(f)-3).

The reference evaluates ONE environment at a time (evaluation.py:27-40, evaluation_tools.py:7-52): `LoadBoxCreator`
(pct_envs/PctDiscrete0/binCreator.py:41-72) walks the `.pt` dataset (a list of trajectories, each a list of
[x, y, z] or [x, y, z, density] items), episode k playing trajectory k+1 (reset() pre-increments the index, so
trajectory 0 is never used) followed by the [100, 100, 100] sentinel that ends the episode; the loop records
`infos['ratio']`, `infos['counter']` and the episode's `env.packed`, then writes `trajs.npy` and `result.txt`.

Here the same episodes are spread over N environments of one GPU batch: environment e plays episodes e, e+N, e+2N, ...
back to back (the kernels' auto-reset jumps to the next trajectory boundary exactly like LoadBoxCreator.reset), the
policy sees every live environment at once, and the per-episode records come out in the reference's episode order.
"""
import os

import numpy as np
import torch

from .batch import PctBatch

SENTINEL = 100.0  # binCreator.py:62


def load_trajectories(data):
    """`data`: path of a torch-saved dataset (binCreator.py:48-49) or an in-memory list of (len, 3|4) arrays."""
    if isinstance(data, (str, os.PathLike)):
        data = torch.load(data, weights_only=False)
    return [np.asarray(t, dtype=np.float64).reshape(len(t), -1) for t in data]


def round3(trajs):
    """PackingContinuous in test mode rounds every item size to 3 decimals with Python's round (C:bin3D.py:84-87); the density
    column is left alone.  Applied on the host when the streams are built, so the kernels see what the reference env sees."""
    out = []
    for t in trajs:
        t = np.array(t, dtype=np.float64)
        for r in t:
            for i in range(3):
                r[i] = round(float(r[i]), 3)
        out.append(t)
    return out


def first_leaf_policy(obs, batch):
    """Deterministic stand-in policy: the first leaf row (index 0), i.e. the first feasible candidate in reference order."""
    return torch.zeros((obs.shape[0],), dtype=torch.int32, device=obs.device)


def _streams(trajs, episodes, n_envs, pad=1):
    """(n_envs, (quota+1)*traj_len, 4) item streams: env e gets trajectories e+1, e+1+N, ... each padded with at least `pad` sentinels.
    A buffered env (buffer=B) holds B draws at a time, so it needs pad = B: its last refills then draw sentinels and never reach into the next
    trajectory (B = 1 is the plain env's padding)."""
    traj_len = max(len(t) for t in trajs) + int(pad)
    quota = [(episodes - e + n_envs - 1) // n_envs for e in range(n_envs)]
    slots = max(quota) + 1  # one all-sentinel trajectory after the last real one: finished envs idle in 1-step episodes
    s = np.full((n_envs, slots, traj_len, 4), SENTINEL)
    s[..., 3] = 1.0
    for e in range(n_envs):
        for j in range(quota[e]):
            t = trajs[e + j * n_envs + 1]
            s[e, j, :len(t), :t.shape[1]] = t
    return s.reshape(n_envs, slots * traj_len, 4), traj_len, np.array(quota)


def evaluate_batched(data, setting, policy=None, container_size=(10, 10, 10), item_set=None, episodes=None, n_envs=1024,
                     continuous=False, LNES="EMS", internal_node_holder=80, leaf_node_holder=50, device=0, out_dir=None,
                     sample_left_bound=None, max_steps=None, buffer=None):
    """Runs `episodes` evaluation episodes (default: every trajectory but the first, like evaluation_episodes = len-1).

    policy(obs (N, obs_len) float32 CUDA tensor, batch) -> (N,) integer CUDA tensor of leaf indices.
    buffer=B: buffered envs (PctBatch(..., buffer=B)) that hold B items of the trajectory at a time; the policy then returns flat leaf indices
    j * NL + l into the leaves of all B items, as buffered_drl_gat does.
    Returns {'ratio': (episodes,) f64, 'length': (episodes,) int, 'packed': list of per-episode [[x,y,z,lx,ly,lz,0], ...],
             'result': the text of result.txt}; with `out_dir`, also writes trajs.npy and result.txt there
    (evaluation_tools.py:44-52).
    """
    trajs = load_trajectories(data)
    if len(trajs) < 2:
        raise ValueError("the dataset needs at least two trajectories (trajectory 0 is never played, binCreator.py:54-55)")
    episodes = len(trajs) - 1 if episodes is None else int(episodes)
    if not 0 < episodes <= len(trajs) - 1:
        raise ValueError("episodes must be in 1..len(dataset)-1 (the reference raises IndexError past the end)")
    n = max(1, min(int(n_envs), episodes))
    if continuous:
        trajs = round3(trajs)
    stream, traj_len, quota = _streams(trajs, episodes, n, pad=buffer or 1)
    policy = first_leaf_policy if policy is None else policy
    size_minimum = None
    if item_set is None:  # D:bin3D.py:23 takes min(item_set); a dataset run without one uses the smallest item of the data
        size_minimum = float(min(t[:, :3].min() for t in trajs[1:episodes + 1])) if sample_left_bound is None else float(sample_left_bound)
    odt = torch.float64 if continuous else torch.float32  # float32 holds the discrete coordinates exactly
    batch = PctBatch(n, setting, container_size=container_size, item_set=item_set, internal_node_holder=internal_node_holder,
                     leaf_node_holder=leaf_node_holder, continuous=continuous, obs_dtype=odt, device=device, item_stream=stream,
                     size_minimum=size_minimum, LNES=LNES, **({} if buffer is None else dict(buffer=buffer)))
    batch.set_trajectory_length(traj_len)
    nb = batch.nb
    binvol = float(container_size[0]) * float(container_size[1]) * float(container_size[2])
    ratio = np.zeros(episodes)
    length = np.zeros(episodes, dtype=np.int64)
    packed = [None] * episodes
    played = np.zeros(n, dtype=np.int64)
    obs = batch.reset()
    prev = torch.empty((n, nb * 9), dtype=odt, device=obs.device)
    limit = int(max_steps) if max_steps else (int(quota.max()) + 1) * (traj_len + 1)
    conv = float if continuous else int
    for _ in range(limit):
        if (played >= quota).all():
            break
        prev.copy_(obs[:, :nb * 9])  # internal-node rows = every box placed so far, in placement order (D:space.py:385-386)
        idx = policy(obs if odt == torch.float32 else obs.float(), batch)
        obs, _, done, info = batch.step(leaf_idx=idx.to(torch.int32))
        done_h = done.cpu().numpy().astype(bool)
        if not done_h.any():
            continue
        who = np.nonzero(done_h & (played < quota))[0]
        if len(who) == 0:
            continue
        info_h = info.cpu().numpy()
        counter = info_h[:, 0]
        PctBatch.check_flags(info_h[who, 1], what="evaluate_batched")  # a flagged episode would not be the reference's: never silent
        rows = prev[torch.from_numpy(who).to(prev.device)].cpu().numpy().reshape(len(who), nb, 9)
        for k, e in enumerate(who):
            ep = int(e + played[e] * n)
            c = int(counter[e])
            items, vol = [], 0.0
            for r in rows[k, :c]:
                if continuous:  # rows hold lo / hi corners; the sizes carry 3 decimals, so rounding the differences returns them exactly
                    x, y, z = float(np.round(r[3] - r[0], 6)), float(np.round(r[4] - r[1], 6)), float(np.round(r[5] - r[2], 6))
                else:
                    x, y, z = conv(r[3] - r[0]), conv(r[4] - r[1]), conv(r[5] - r[2])
                items.append([x, y, z, conv(r[0]), conv(r[1]), conv(r[2]), 0])  # D:bin3D.py:177-178
                vol += x * y * z  # Space.get_ratio (D:space.py:334-339)
            packed[ep], ratio[ep], length[ep] = items, vol / binvol, c
            played[e] += 1
    batch.close()
    if not (played >= quota).all():
        raise RuntimeError("evaluation did not finish within %d steps" % limit)
    result = "Evaluation using {} episodes\nMean ratio {:.5f}, mean length{:.5f}\n".format(episodes, np.mean(ratio), np.mean(length))
    if out_dir is not None:
        os.makedirs(out_dir, exist_ok=True)
        arr = np.empty(episodes, dtype=object)  # ragged list of lists (what np.save made of it on the reference's numpy)
        for i, p in enumerate(packed):
            arr[i] = p
        np.save(os.path.join(out_dir, "trajs.npy"), arr, allow_pickle=True)
        with open(os.path.join(out_dir, "result.txt"), "w") as f:
            f.write(result)
    return dict(ratio=ratio, length=length, packed=packed, result=result)


def main(argv=None):
    """`python -m pct_b200.evaluation --dataset-path set.pt --setting 1 ...` (mirrors the evaluation.py flags that matter here)"""
    import argparse
    ap = argparse.ArgumentParser(description=main.__doc__)
    ap.add_argument("--dataset-path", required=True)
    ap.add_argument("--setting", type=int, default=1)
    ap.add_argument("--continuous", action="store_true")
    ap.add_argument("--container-size", type=float, nargs=3, default=[10, 10, 10])
    ap.add_argument("--lnes", default="EMS")
    ap.add_argument("--internal-node-holder", type=int, default=80)
    ap.add_argument("--leaf-node-holder", type=int, default=50)
    ap.add_argument("--evaluation-episodes", type=int, default=None)
    ap.add_argument("--num-envs", type=int, default=1024)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--out-dir", default=None)
    ap.add_argument("--buffer", type=int, default=None, help="buffered envs holding B items (the policy picks among the leaves of all of them)")
    a = ap.parse_args(argv)
    cs = a.container_size if a.continuous else [int(c) for c in a.container_size]
    out = evaluate_batched(a.dataset_path, a.setting, container_size=cs, episodes=a.evaluation_episodes, n_envs=a.num_envs,
                           continuous=a.continuous, LNES=a.lnes, internal_node_holder=a.internal_node_holder,
                           leaf_node_holder=a.leaf_node_holder, device=a.device, out_dir=a.out_dir, buffer=a.buffer)
    print(out["result"])


if __name__ == "__main__":
    main()
