"""PctVecEnv — the reference's vectorised-environment surface on top of the CUDA batch.

Replaces `VecPyTorch(ShmemVecEnv([make_env(...)] * N))` (reference: envs.py:75-116,159-182,
wrapper/shmem_vec_env.py:20-156, wrapper/vec_env.py:29-139): same methods, same return types, same
auto-reset semantics, but observations never leave the GPU and there are no worker processes.

    obs                      torch.float32 (N, 1179) on the device      (VecPyTorch.reset/step_wait, envs.py:166-182)
    reward                   torch.float32 (N, 1) on the CPU             (envs.py:181)
    done                     numpy bool (N,)                             (shmem_vec_env.py:81)
    infos                    tuple of N dicts; finished envs carry {'counter','ratio','reward','episode':{'r','l','t'}}
                             (D:bin3D.py:163-164, wrapper/monitor.py:58-77; consumed at train_tools.py:72-79)
"""
import time
from collections.abc import Sequence

import numpy as np
import torch

from .batch import PctBatch


class LazyInfos(Sequence):
    """The `infos` of one vector step: behaves like the reference's tuple of N dicts (len, indexing, iteration, ==), but a dict is only
    built when its env is looked at — the reference's consumer reads `infos[i]` for the finished envs only (train_tools.py:72-79), and
    building 4096 dicts per step costs ~10x the kernels' time.  Finished envs carry {'counter','ratio','reward','episode':{'r','l','t'}}
    (D:bin3D.py:163-164, wrapper/monitor.py:58-77); every env carries 'counter' (D:bin3D.py:186) and 'flags' when a capacity flag is set."""

    __slots__ = ("_rec", "_done", "_now", "_cache")

    def __init__(self, rec, done, now):
        self._rec, self._done, self._now, self._cache = rec, done, now, {}

    def __len__(self):
        return len(self._done)

    def __getitem__(self, e):
        if isinstance(e, slice):
            return tuple(self[i] for i in range(*e.indices(len(self))))
        if e < 0:
            e += len(self)
        if not 0 <= e < len(self):
            raise IndexError(e)
        d = self._cache.get(e)
        if d is None:
            rec = self._rec
            d = {"counter": int(rec["counter"][e])}
            if self._done[e]:
                ratio = float(rec["ratio"][e])
                d.update(ratio=ratio, reward=ratio * 10,
                         episode={"r": round(float(rec["ep_reward"][e]), 6), "l": int(rec["ep_len"][e]), "t": self._now})
            if rec["flags"][e]:
                d["flags"] = int(rec["flags"][e])
            self._cache[e] = d
        return d

    def __eq__(self, other):
        return len(self) == len(other) and all(a == b for a, b in zip(self, other))

    def __repr__(self):
        return "LazyInfos(%d envs, %d finished)" % (len(self), int(np.count_nonzero(self._done)))


class _BoxSpace(object):
    """Stand-in for gym.spaces.Box (D:bin3D.py:41-42) when gym is not installed."""

    def __init__(self, low, high, shape, dtype=np.float32):
        self.low, self.high, self.shape, self.dtype = low, high, tuple(shape), np.dtype(dtype)


def _make_box(low, high, shape):
    try:
        import gym  # noqa
        return gym.spaces.Box(low=low, high=high, shape=shape)
    except Exception:
        return _BoxSpace(low, high, shape)


class PctVecEnv(object):
    """N PCT environments stepped together on one GPU; duck-types wrapper.vec_env.VecEnv."""

    closed = False
    viewer = None
    metadata = {"render.modes": []}

    def __init__(self, num_envs, setting, container_size=(10, 10, 10), item_set=None, internal_node_holder=80,
                 leaf_node_holder=50, continuous=False, device=0, seed=0, env_id_base=0, sample_from_distribution=False,
                 sample_left_bound=None, sample_right_bound=None, item_stream=None, LNES="EMS", shuffle=False, copy_obs=True,
                 raise_on_flags=True, **_ignored):
        """copy_obs: return a fresh observation tensor every step like VecPyTorch does (a 19 MB device-to-device copy at 4096 envs); False hands
        out the library-owned buffer that the next step rewrites in place (zero-copy; the caller must not modify it: delta observation rows).
        shuffle: the reference's kwarg (np.random.shuffle of the candidate list, D:bin3D.py:114-115) as a keyed device-side permutation (PctBatch).
        raise_on_flags: a capacity / hand-over flag in any env's step record (pct_step_info.flags: overflowed EMS / candidate / edge / support
        capacity, bad action, sync timeout) raises PctError instead of only appearing in that env's info dict."""
        self.copy_obs, self.raise_on_flags = bool(copy_obs), bool(raise_on_flags)
        self.batch = PctBatch(num_envs, setting, container_size=container_size, item_set=item_set,
                              internal_node_holder=internal_node_holder, leaf_node_holder=leaf_node_holder, continuous=continuous,
                              obs_dtype=torch.float32, seed=seed, env_id_base=env_id_base, device=device,
                              sample_from_distribution=sample_from_distribution, sample_left_bound=sample_left_bound,
                              sample_right_bound=sample_right_bound, item_stream=item_stream, LNES=LNES, shuffle=shuffle)
        self.num_envs = int(num_envs)
        self.device = self.batch.device
        self.observation_space = _make_box(0.0, float(container_size[2]), (self.batch.obs_len,))
        self.action_space = None  # the reference env never defines one (read at envs.py:107)
        self._tstart = time.time()
        self._pending = None
        n = self.num_envs
        # one pinned block for everything step_wait hands back on the host: reward (N f32) | info (N x 8 i32) | done (N u8) -> ONE sync per step
        self._cuda = self.device.type == "cuda"  # (the CPU tests drive this class over an oracle-backed stand-in for PctBatch)
        self._host = torch.empty((n * 4 + n * 32 + n,), dtype=torch.uint8, pin_memory=self._cuda)
        self._dev_pack = torch.empty((n * 4 + n * 32 + n,), dtype=torch.uint8, device=self.device)

    # ---- VecEnv API (wrapper/vec_env.py:48-108) ----
    def reset(self):
        obs = self.batch.reset()
        return obs.clone() if self.copy_obs else obs

    def step_async(self, actions):
        """actions: (N, 9) leaf rows (torch tensor or numpy, any float dtype) — what train_tools.py:66-67 passes —
        or a (N,) / (N,1) integer tensor of leaf indices (fast path, no row decode)."""
        if isinstance(actions, np.ndarray):
            actions = torch.from_numpy(np.ascontiguousarray(actions))
        if actions.dtype in (torch.int32, torch.int64) and actions.numel() == self.num_envs:
            self._pending = ("idx", actions.reshape(-1).to(self.device, non_blocking=True))
        else:
            self._pending = ("rows", actions.reshape(self.num_envs, -1)[:, :9].to(self.device, non_blocking=True))

    def step_wait(self):
        kind, a = self._pending
        self._pending = None
        if kind == "idx":
            obs, rew, done, info = self.batch.step(leaf_idx=a)
        else:
            if a.shape[1] < 9:  # 6-float rows (evaluation_tools.py:24)
                a = torch.cat([a, torch.zeros((a.shape[0], 9 - a.shape[1]), dtype=a.dtype, device=a.device)], dim=1)
            obs, rew, done, info = self.batch.step(actions=a)
        n = self.num_envs
        pk = getattr(self.batch, "_pack", None)  # PctBatch keeps reward | info | done in one allocation: one device -> host copy
        if pk is None:
            pk = self._dev_pack
            pk[:4 * n].view(torch.float32).copy_(rew)
            pk[4 * n:36 * n].view(torch.int32).copy_(info.reshape(-1))
            pk[36 * n:].copy_(done)
        self._host.copy_(pk, non_blocking=True)
        if self.copy_obs:
            obs = obs.clone()
        if self._cuda:
            torch.cuda.current_stream(self.device).synchronize()  # the one host sync of the step
        hb = self._host.numpy()
        reward = torch.from_numpy(hb[:4 * n].view(np.float32).copy()).unsqueeze(1)
        rec_raw = hb[4 * n:36 * n].view(np.int32).reshape(n, 8).copy()
        done_h = hb[36 * n:].astype(bool)
        rec = PctBatch.decode_info(rec_raw)
        if self.raise_on_flags:
            PctBatch.check_flags(rec["flags"], what="PctVecEnv.step")
        infos = LazyInfos(rec, done_h, round(time.time() - self._tstart, 6))
        return obs, reward, done_h, infos

    def step(self, actions):
        self.step_async(actions)
        return self.step_wait()

    def close(self):
        if not self.closed:
            self.batch.close()
            self.closed = True

    @property
    def unwrapped(self):
        return self

    def get_images(self):
        raise NotImplementedError

    def render(self, mode="human"):
        raise NotImplementedError
