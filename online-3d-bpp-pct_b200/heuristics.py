"""Heuristic baselines, batched (SURVEY.md §8(f)-4).

The reference runs each baseline as a Python loop over ONE env (heuristic.py:11-577: per item, enumerate placements, call
`env.space.drop_box_virtual` for each, score, `env.step` with the best).  Here thousands of envs advance together: one
selection kernel (`pct_heuristic_actions`, csrc/pct_heuristics.cuh) picks every env's placement with the same enumeration
order, scores and tie rules, and the ordinary step kernels apply them.  The summary matches what every function of
heuristic.py returns: (mean utilisation, variance of utilisation, mean number of packed items).

    python -m pct_b200.heuristics --heuristic LSAH --setting 2 --evaluation-episodes 1000        (heuristic.py:579-610)
    python -m pct_b200.heuristics --heuristic LSAH --setting 2 --evaluation-episodes 1000 --buffer 3   (online packing with a buffer of 3)
"""
import numpy as np
import torch

from . import _lib
from .batch import PctBatch
from .evaluation import _streams, load_trajectories, round3

HEURISTICS = tuple(_lib.HEURISTIC_CODES)  # LSAH, OnlineBPH, BR, MACS, DBL, HM, RANDOM (tools.py:209)
CONTINUOUS_HEURISTICS = ("LSAH", "OnlineBPH", "BR")  # tools.py:217-218


def run_heuristic(name, setting, episodes, container_size=(10, 10, 10), item_set=None, data=None, n_envs=1024, seed=0, device=0,
                  internal_node_holder=80, leaf_node_holder=50, max_steps=None, return_episodes=False, continuous=False,
                  sample_from_distribution=False, sample_left_bound=None, sample_right_bound=None, item_stream=None, buffer=None):
    """Plays `episodes` episodes of baseline `name` spread over min(n_envs, episodes) envs of one GPU batch.

    data=None: items are drawn on the fly from `item_set` (RandomBoxCreator) — or, continuous + sample_from_distribution, from
    U(a, b) rounded to 3 decimals (C:bin3D.py:103-115); env e plays episodes e, e+N, ...
    data=path|list: the trajectory dataset of `--load-dataset` (LoadBoxCreator: episode k plays trajectory k+1).
    item_stream: (n, len, 3|4) per-env draw sequences instead (tests).
    continuous=True: PackingContinuous; only LSAH, OnlineBPH and BR (tools.py:217-218).
    buffer=B: buffered envs holding B items; the baseline picks the item and its placement (buffer_heuristic_actions, DESIGN.md section 22).
    With B = 1 the results are those without a buffer.
    -> (mean ratio, var ratio, mean length) like heuristic.py; with return_episodes also the per-episode arrays / packed lists.
    """
    if name not in _lib.HEURISTIC_CODES:
        raise ValueError("unknown heuristic %r (options: %s)" % (name, " ".join(HEURISTICS)))
    if continuous and name not in CONTINUOUS_HEURISTICS:
        raise ValueError("only LSAH, OnlineBPH, and BR allowed for continuous environment")  # tools.py:218
    episodes = int(episodes)
    n = max(1, min(int(n_envs), episodes))
    stream = traj_len = None
    if data is not None:
        trajs = load_trajectories(data)
        if continuous:  # PackingContinuous in test mode rounds the item sizes to 3 decimals (C:bin3D.py:84-87), like evaluate_batched and the facade
            trajs = round3(trajs)
        if not 0 < episodes <= len(trajs) - 1:
            raise ValueError("episodes must be in 1..len(dataset)-1")
        stream, traj_len, quota = _streams(trajs, episodes, n, pad=buffer or 1)
    else:
        quota = np.array([(episodes - e + n - 1) // n for e in range(n)])
        if item_stream is not None:
            stream = np.asarray(item_stream, dtype=np.float64)[:n]
    # continuous: float64 observations, so that the placed boxes read back below are the env's own float64 coordinates
    odt = torch.float64 if continuous else torch.float32
    batch = PctBatch(n, setting, container_size=container_size, item_set=item_set, internal_node_holder=internal_node_holder,
                     leaf_node_holder=leaf_node_holder, obs_dtype=odt, seed=seed, device=device, item_stream=stream, continuous=continuous,
                     sample_from_distribution=sample_from_distribution, sample_left_bound=sample_left_bound,
                     sample_right_bound=sample_right_bound, **({} if buffer is None else dict(buffer=buffer)))
    if traj_len:
        batch.set_trajectory_length(traj_len)
    nb = batch.nb
    binvol = float(container_size[0]) * float(container_size[1]) * float(container_size[2])
    ratio, length, packed = np.zeros(episodes), np.zeros(episodes, dtype=np.int64), [None] * episodes
    played = np.zeros(n, dtype=np.int64)
    obs = batch.reset()
    prev = torch.empty((n, nb * 9), dtype=odt, device=obs.device) if return_episodes else None
    limit = int(max_steps) if max_steps else (int(quota.max()) + 1) * (internal_node_holder + 2)
    t = 0
    while not (played >= quota).all() and t < limit:
        if prev is not None:
            prev.copy_(obs[:, :nb * 9])
        if buffer is None:
            rows = batch.heuristic_actions(name, seed=seed, t=t)
            obs, _, done, info = batch.step(actions=rows)
        else:
            slots, rows = batch.buffer_heuristic_actions(name, seed=seed, t=t)
            obs, _, done, info = batch.buffer_step_rows(slots, rows)
        t += 1
        done_h = done.cpu().numpy().astype(bool)
        who = np.nonzero(done_h & (played < quota))[0]
        if len(who) == 0:
            continue
        rec = PctBatch.decode_info(info)
        # "no feasible placement" is delivered as a row no item matches (PCT_FLAG_BAD_ACTION, include/pct_b200.h) and ends the episode like the
        # reference's `done = True` without stepping: expected here; every other flag means the episode is not the reference's
        PctBatch.check_flags(rec["flags"][who], ignore=2, what="run_heuristic")
        boxes = prev[torch.from_numpy(who).to(prev.device)].cpu().numpy().reshape(len(who), nb, 9) if prev is not None else None
        for k, e in enumerate(who):
            ep = int(e + played[e] * n)
            c = int(rec["counter"][e])
            length[ep] = c
            if boxes is None:
                ratio[ep] = float(rec["ratio"][e])
            else:  # Space.get_ratio in float64 from the placed boxes (D:space.py:334-339 / C:space.py:316-321)
                items, vol = [], 0.0
                for r in boxes[k, :c]:
                    if continuous:  # rows are [lx, ly, lz, lx+x, ly+y, lz+z]; sizes carry <= 6 decimals, so rounding returns them exactly
                        x, y, z = (float(np.round(r[3] - r[0], 6)), float(np.round(r[4] - r[1], 6)), float(np.round(r[5] - r[2], 6)))
                        items.append([x, y, z, float(r[0]), float(r[1]), float(r[2]), 0])
                    else:
                        x, y, z = int(r[3] - r[0]), int(r[4] - r[1]), int(r[5] - r[2])
                        items.append([x, y, z, int(r[0]), int(r[1]), int(r[2]), 0])
                    vol += x * y * z
                packed[ep], ratio[ep] = items, vol / binvol
            played[e] += 1
    batch.close()
    if not (played >= quota).all():
        raise RuntimeError("heuristic run did not finish within %d steps" % limit)
    summary = (float(np.mean(ratio)), float(np.var(ratio)), float(np.mean(length)))
    if return_episodes:
        return summary, dict(ratio=ratio, length=length, packed=packed, steps=t)
    return summary


def main(argv=None):
    import argparse
    ap = argparse.ArgumentParser(description="Heuristic baseline arguments (tools.get_args_heuristic, tools.py:200-230)")
    ap.add_argument("--continuous", action="store_true", help="Use continuous enviroment, otherwise the enviroment is discrete")
    ap.add_argument("--setting", type=int, default=2)
    ap.add_argument("--evaluation-episodes", type=int, default=10)
    ap.add_argument("--load-dataset", action="store_true")
    ap.add_argument("--dataset-path", type=str)
    ap.add_argument("--heuristic", type=str, default="LSAH", help="Options: LSAH DBL MACS OnlineBPH HM BR RANDOM")
    ap.add_argument("--container-size", type=float, nargs=3, default=None, help="givenData.container_size: [10,10,10]; continuous: [1,1,1]")
    ap.add_argument("--num-envs", type=int, default=1024)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--buffer", type=int, default=None, help="online packing with a buffer: every env holds B items, the baseline picks one")
    a = ap.parse_args(argv)
    item_set = [(i, j, k) for i in range(1, 6) for j in range(1, 6) for k in range(1, 6)]  # givenData.py:7-14
    cs = a.container_size or ([1.0, 1.0, 1.0] if a.continuous else [10, 10, 10])  # givenData.py:4-5
    if not a.continuous:
        cs = [int(c) for c in cs]
    # heuristic.py:585-591 builds PackingContinuous with its class defaults — sample_from_distribution=True, U(0.1, 0.5) (C:bin3D.py:14-16) —
    # also under --load-dataset: the dataset then supplies the items, but Space.low_bound stays sample_left_bound = 0.1 (C:bin3D.py:25-27)
    mean, var, length = run_heuristic(a.heuristic, a.setting, a.evaluation_episodes, container_size=cs, item_set=item_set,
                                      data=a.dataset_path if a.load_dataset else None, n_envs=a.num_envs, device=a.device,
                                      continuous=a.continuous, sample_from_distribution=a.continuous,
                                      sample_left_bound=0.1 if a.continuous else None, sample_right_bound=0.5 if a.continuous else None,
                                      buffer=a.buffer)
    print("The average space utilization:", mean)
    print("The variance of space utilization:", var)
    print("The average number of packed items:", length)


if __name__ == "__main__":
    main()
