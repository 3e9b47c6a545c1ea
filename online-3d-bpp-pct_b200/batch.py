"""PctBatch — N PCT environments living on one H100, stepped by the CUDA kernels behind the C ABI.

PyTorch is used for device buffers and streams only (observation / action / reward tensors); every
environment computation happens inside libpct_b200.so.  Mirrors the constructor kwargs of the reference's
PackingDiscrete / PackingContinuous (pct_envs/PctDiscrete0/bin3D.py:9-15, pct_envs/PctContinuous0/bin3D.py:9-17).
"""
import ctypes as C

import numpy as np
import torch

from . import _lib


class PctError(RuntimeError):
    pass


class PctBatch(object):
    def __init__(self, n_envs, setting, container_size=(10, 10, 10), item_set=None, internal_node_holder=80,
                 leaf_node_holder=50, continuous=False, obs_dtype=torch.float32, seed=0, env_id_base=0, device=0,
                 sample_from_distribution=False, sample_left_bound=None, sample_right_bound=None, item_stream=None,
                 size_minimum=None, auto_reset=True, LNES="EMS", shuffle=False):
        """shuffle: the reference's `shuffle` kwarg (D:bin3D.py:114-115; tools.py:136 defaults --shuffle to True for training): the ordered candidate list
        is permuted before the feasibility tests and the leaf cap, by a keyed counter-based permutation (include/pct_b200.h, pct_config::shuffle)."""
        if not torch.cuda.is_available():
            raise PctError("pct_b200 needs a CUDA device (sm_90a kernels; there is no CPU fallback)")
        self.L = _lib.lib()
        self.n_envs = int(n_envs)
        self.device = torch.device("cuda", device)
        self.nb, self.nl = int(internal_node_holder), int(leaf_node_holder)
        self.obs_dtype = obs_dtype
        self.container_size = tuple(container_size)
        self.setting = int(setting)
        self.continuous = bool(continuous)
        cfg = _lib.Config()
        cfg.domain = _lib.PCT_CONTINUOUS if continuous else _lib.PCT_DISCRETE
        cfg.setting = self.setting
        for i in range(3):
            cfg.container_size[i] = float(container_size[i])
        cfg.internal_node_holder, cfg.leaf_node_holder = self.nb, self.nl
        cfg.obs_dtype = _lib.PCT_F64 if obs_dtype == torch.float64 else _lib.PCT_F32
        cfg.item_mode = _lib.PCT_ITEMS_RANDOM
        cfg.sample_from_distribution = int(bool(sample_from_distribution))
        if sample_from_distribution:
            # tools.get_args :178-181
            if sample_left_bound is None:
                sample_left_bound = 0.1 * min(container_size)
            if sample_right_bound is None:
                sample_right_bound = 0.5 * min(container_size)
            cfg.sample_left_bound, cfg.sample_right_bound = float(sample_left_bound), float(sample_right_bound)
        if size_minimum is None:
            # D:bin3D.py:23 / C:bin3D.py:25-29
            if continuous and sample_from_distribution:
                size_minimum = sample_left_bound
            else:
                size_minimum = float(np.min(np.array(item_set))) if item_set is not None else 1.0
        cfg.size_minimum = float(size_minimum)
        cfg.seed = int(seed) & ((1 << 64) - 1)
        cfg.env_id_base = int(env_id_base)
        cfg.no_auto_reset = 0 if auto_reset else 1
        cfg.lnes = _lib.LNES_CODES[LNES]
        cfg.shuffle = int(bool(shuffle))
        self.cfg = cfg
        self.did_reset = False
        h = C.c_void_p()
        rc = self.L.pct_create(C.byref(cfg), self.n_envs, int(device), C.byref(h))
        if rc != 0:
            raise PctError("pct_create failed (%d): %s" % (rc, self.L.pct_last_error(None).decode()))
        self.h = h
        self.obs_len = self.L.pct_obs_len(self.h)
        if item_set is not None:
            self.set_item_set(item_set)
        if item_stream is not None:
            self.set_item_stream(item_stream)
        with torch.cuda.device(self.device):
            self._obs = torch.empty((self.n_envs, self.obs_len), dtype=obs_dtype, device=self.device)
            # reward (N f32) | info (N x 8 i32) | done (N u8) live in ONE allocation, so that a host-facing caller fetches all three with one copy
            n = self.n_envs
            self._pack = torch.zeros((n * 4 + n * 32 + n,), dtype=torch.uint8, device=self.device)
            self._rew = self._pack[:4 * n].view(torch.float32)
            self._info = self._pack[4 * n:36 * n].view(torch.int32).view(n, 8)
            self._done = self._pack[36 * n:]
            self._idx = torch.zeros((self.n_envs,), dtype=torch.int32, device=self.device)

    # -- plumbing ------------------------------------------------------------------------------------------
    def _check(self, rc, what):
        if rc != 0:
            raise PctError("%s failed (%d): %s" % (what, rc, self.L.pct_last_error(self.h).decode()))

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def set_item_set(self, item_set):
        a = np.ascontiguousarray(np.array(item_set, dtype=np.float64).reshape(-1, 3))
        self._check(self.L.pct_set_item_set(self.h, a.ctypes.data_as(C.POINTER(C.c_double)), len(a)), "pct_set_item_set")

    def set_item_stream(self, stream):
        """stream: array (n_envs, len, 3|4) of per-env draws (x, y, z[, density])."""
        a = np.array(stream, dtype=np.float64)
        if a.ndim != 3 or a.shape[0] != self.n_envs:
            raise PctError("item stream must have shape (n_envs, len, 3|4)")
        if a.shape[2] == 3:
            a = np.concatenate([a, np.ones(a.shape[:2] + (1,))], axis=2)
        a = np.ascontiguousarray(a)
        self._check(self.L.pct_set_item_stream(self.h, a.ctypes.data_as(C.POINTER(C.c_double)), a.shape[1]), "pct_set_item_stream")

    def set_trajectory_length(self, traj_len):
        self._check(self.L.pct_set_trajectory_length(self.h, int(traj_len)), "pct_set_trajectory_length")

    # -- device-resident API -------------------------------------------------------------------------------
    def reset(self, out=None, env_idx=None, mask=None, info=None):
        """Without env_idx / mask: reset every env (VecEnv.reset()).  With one of them: env.reset() for the chosen envs only
        (pct_reset_envs, include/pct_b200.h), enqueued on the current stream (graph-capturable) after a first full reset.  env_idx: distinct
        env indices (indices outside [0, n_envs) are skipped); mask: an (n_envs,) bool / uint8 tensor, e.g. the `done` of the last step,
        so `reset(mask=done)` gives gym semantics to a batch built with auto_reset=False.  Every env of the batch is re-expanded (envs not
        chosen come out unchanged) and the complete observation goes to `out` (default: the batch's own observation buffer, under the
        delta-row contract of step), which is returned: clone() a terminal observation before resetting over it.  info: optional
        (n_envs, 8) int32 tensor for the pct_step_info records of the new expansions.  An empty env_idx enqueues nothing."""
        if env_idx is None and mask is None:
            if info is not None:
                raise PctError("reset: info is written by a reset of chosen envs (env_idx or mask) only")
            obs = self._obs if out is None else out
            self._check(self.L.pct_reset(self.h, C.c_void_p(obs.data_ptr()), self._stream()), "pct_reset")
            self.did_reset = True
            return obs
        if env_idx is not None and mask is not None:
            raise PctError("reset: pass env_idx or mask, not both")
        if not self.did_reset:
            raise PctError("reset(env_idx / mask) before the first reset() of the batch")
        obs = self._obs if out is None else self._out(out, (self.n_envs, self.obs_len), self.obs_dtype, "reset out")
        if info is not None:
            info = self._out(info, (self.n_envs, 8), torch.int32, "reset info")
        idx = m = None
        if mask is not None:
            if not torch.is_tensor(mask):
                mask = torch.as_tensor(np.asarray(mask))
            if mask.dtype not in (torch.bool, torch.uint8) or tuple(mask.shape) != (self.n_envs,):
                raise PctError("reset mask must be an (n_envs,) = (%d,) bool or uint8 tensor" % self.n_envs)
            m = mask.to(self.device).contiguous()
            if m.dtype == torch.bool:
                m = m.view(torch.uint8)  # same bytes (0 / 1): no copy, so a captured graph reads the caller's tensor
            n = self.n_envs
        else:
            idx = self._index(env_idx, "env_idx")
            n = int(idx.numel())
            if n == 0:
                return obs
        ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
        self._check(self.L.pct_reset_envs(self.h, ptr(idx), n, ptr(m), C.c_void_p(obs.data_ptr()), ptr(info), self._stream()),
                    "pct_reset_envs")
        return obs

    def step(self, actions=None, leaf_idx=None, out=None):
        """actions: (N,9) float32/float64 CUDA tensor of leaf rows, or leaf_idx: (N,) int32 CUDA tensor.
        Returns (obs, reward(N,), done(N,) uint8, info(N,8) int32 raw pct_step_info records) — all on the GPU.
        NOTE: without `out`, the four tensors are the library-owned buffers, rewritten IN PLACE by the next reset / step (zero-copy; and with the
        delta observation rows, include/pct_b200.h, the observation buffer must not be modified by the caller).  Keep a result across steps with
        .clone(), or pass your own `out` buffers (e.g. a rollout storage, GraphedRollout); PctVecEnv hands out fresh observation tensors."""
        obs = self._obs if out is None else out
        a_ptr, i_ptr, f64 = None, None, 0
        if actions is not None:
            if actions.dtype not in (torch.float32, torch.float64):
                actions = actions.float()
            actions = actions.contiguous()
            if actions.shape != (self.n_envs, 9):
                raise PctError("actions must have shape (n_envs, 9)")
            a_ptr, f64 = C.c_void_p(actions.data_ptr()), int(actions.dtype == torch.float64)
        else:
            leaf_idx = leaf_idx.to(torch.int32).contiguous()
            i_ptr = C.c_void_p(leaf_idx.data_ptr())
        self._check(self.L.pct_step(self.h, a_ptr, f64, i_ptr, C.c_void_p(obs.data_ptr()), C.c_void_p(self._rew.data_ptr()),
                                    C.c_void_p(self._done.data_ptr()), C.c_void_p(self._info.data_ptr()), self._stream()), "pct_step")
        return obs, self._rew, self._done, self._info

    def random_policy(self, seed, t, out=None):
        idx = self._idx if out is None else out
        self._check(self.L.pct_policy_random(self.h, C.c_void_p(idx.data_ptr()), int(seed) & ((1 << 64) - 1), int(t), self._stream()),
                    "pct_policy_random")
        return idx

    def random_policy_dev(self, seed, t_dev, out=None):
        """random_policy with the step counter read from a device int64 tensor at execution time (graph-capturable)"""
        idx = self._idx if out is None else out
        self._check(self.L.pct_policy_random_dev(self.h, C.c_void_p(idx.data_ptr()), int(seed) & ((1 << 64) - 1), C.c_void_p(t_dev.data_ptr()),
                                                 self._stream()), "pct_policy_random_dev")
        return idx

    # -- snapshot / restore (include/pct_b200.h) --------------------------------------------------------------
    @property
    def snapshot_bytes(self):
        """bytes of one env record (fixed per domain)"""
        return int(self.L.pct_snapshot_bytes(self.h))

    def _index(self, idx, what):
        if idx is None:
            return None
        if not torch.is_tensor(idx):
            idx = torch.as_tensor(np.asarray(idx, dtype=np.int32))
        if idx.dim() != 1:
            raise PctError("%s must be one-dimensional" % what)
        return idx.to(device=self.device, dtype=torch.int32).contiguous()

    def snapshot(self, env_idx=None, out=None):
        """State records of envs `env_idx` (default: every env) -> (n, snapshot_bytes) uint8 CUDA tensor, filled on the current stream.
        The records hold no pointers: they can be moved to another GPU, saved and restored into any slot of a batch with the same
        configuration (restore)."""
        idx = self._index(env_idx, "env_idx")
        n = self.n_envs if idx is None else int(idx.numel())
        B = self.snapshot_bytes
        if out is None:
            out = torch.empty((n, B), dtype=torch.uint8, device=self.device)
        elif out.dtype != torch.uint8 or out.device != self.device or not out.is_contiguous() or tuple(out.shape) != (n, B):
            raise PctError("snapshot out must be a contiguous (%d, %d) uint8 tensor on %s" % (n, B, self.device))
        self._check(self.L.pct_snapshot(self.h, C.c_void_p(idx.data_ptr()) if idx is not None else None, n, C.c_void_p(out.data_ptr()),
                                        self._stream()), "pct_snapshot")
        return out

    def restore(self, snap, env_idx=None, rec_idx=None, out=None, write_obs=True):
        """Env env_idx[i] <- record rec_idx[i] of `snap` (defaults: env i, record i; one record may feed many envs).  Destinations must be
        distinct.  Record indices outside `snap` are skipped (on the device, without a synchronisation).  Writes the complete observation
        rows of the restored envs into `out` (default: the batch's own observation buffer) and returns it; write_obs=False writes no rows
        (the next step then rewrites every row of the restored envs) and returns None.  A record of another configuration leaves its env
        unchanged and flags it (bad_snapshot, reported by the next step)."""
        if snap.dtype != torch.uint8 or snap.dim() != 2 or snap.shape[1] != self.snapshot_bytes:
            raise PctError("snapshot must be an (n, %d) uint8 tensor" % self.snapshot_bytes)
        snap = snap.to(self.device).contiguous()
        env = self._index(env_idx, "env_idx")
        rec = self._index(rec_idx, "rec_idx")
        n = int(env.numel()) if env is not None else (int(rec.numel()) if rec is not None else int(snap.shape[0]))
        if rec is not None:
            if int(rec.numel()) != n:
                raise PctError("env_idx and rec_idx must have the same length")
            rec = torch.where((rec >= 0) & (rec < snap.shape[0]), rec, torch.full_like(rec, -1))
        elif n > snap.shape[0]:
            raise PctError("restore of %d envs from %d records without rec_idx" % (n, snap.shape[0]))
        obs = None
        if write_obs:
            obs = self._obs if out is None else out
            if obs.dtype != self.obs_dtype or not obs.is_contiguous() or tuple(obs.shape) != (self.n_envs, self.obs_len):
                raise PctError("restore out must be a contiguous (n_envs, obs_len) tensor of the batch's observation dtype")
        self._check(self.L.pct_restore(self.h, C.c_void_p(env.data_ptr()) if env is not None else None,
                                       C.c_void_p(rec.data_ptr()) if rec is not None else None, n, C.c_void_p(snap.data_ptr()),
                                       C.c_void_p(obs.data_ptr()) if obs is not None else None, self._stream()), "pct_restore")
        return obs

    # -- heuristic baselines (heuristic.py) ------------------------------------------------------------------
    def heuristic_actions(self, name, seed=0, t=0, out=None):
        """(N, 9) float32 CUDA tensor of action rows: the placement the baseline `name` (LSAH, OnlineBPH, BR, MACS, DBL, HM,
        RANDOM) selects for every env's current item; feed to step(actions=...).
        Continuous domain: LSAH / OnlineBPH / BR (tools.py:217-218), float64 rows."""
        if name not in _lib.HEURISTIC_CODES:
            raise PctError("unknown heuristic %r" % (name,))
        if self.continuous:
            if out is None:
                if getattr(self, "_hrows", None) is None:
                    self._hrows = torch.zeros((self.n_envs, 9), dtype=torch.float64, device=self.device)
                out = self._hrows
            if out.dtype != torch.float64 or not out.is_contiguous() or out.shape != (self.n_envs, 9):
                raise PctError("continuous heuristic rows must be a contiguous (n_envs, 9) float64 tensor")
            self._check(self.L.pct_heuristic_actions_f64(self.h, _lib.HEURISTIC_CODES[name], C.c_void_p(out.data_ptr()), self._stream()),
                        "pct_heuristic_actions_f64")
            return out
        if out is None:
            if getattr(self, "_hrows", None) is None:
                self._hrows = torch.zeros((self.n_envs, 9), dtype=torch.float32, device=self.device)
            out = self._hrows
        self._check(self.L.pct_heuristic_actions(self.h, _lib.HEURISTIC_CODES[name], C.c_void_p(out.data_ptr()), int(seed) & ((1 << 64) - 1),
                                                 int(t), self._stream()), "pct_heuristic_actions")
        return out

    def query_placement(self, env, dims, lx, ly, density=1.0, want_map=False):
        """Space.drop_box_virtual for one env (D:space.py:393-433): -> (feasible, rest_height[, height map after])"""
        if self.continuous:  # C:space.py:380-425 has no returnMap
            d, feas, mh = (C.c_double * 3)(float(dims[0]), float(dims[1]), float(dims[2])), C.c_int32(), C.c_double()
            self._check(self.L.pct_query_placement_f64(self.h, int(env), d, float(lx), float(ly), float(density), C.byref(feas), C.byref(mh)),
                        "pct_query_placement_f64")
            return (bool(feas.value), mh.value, None) if want_map else (bool(feas.value), mh.value)
        d = (C.c_int32 * 3)(int(dims[0]), int(dims[1]), int(dims[2]))
        feas, mh = C.c_int32(), C.c_int32()
        W, L = int(self.container_size[0]), int(self.container_size[1])
        hm = np.zeros((W, L), dtype=np.int32) if want_map else None
        self._check(self.L.pct_query_placement(self.h, int(env), d, int(lx), int(ly), float(density), C.byref(feas), C.byref(mh),
                                               hm.ctypes.data_as(C.POINTER(C.c_int32)) if want_map else None), "pct_query_placement")
        return (bool(feas.value), mh.value, hm) if want_map else (bool(feas.value), mh.value)

    # -- batched placement queries and height maps (include/pct_b200.h) --------------------------------------------
    def _out(self, t, shape, dtype, what):
        if not torch.is_tensor(t) or t.dtype != dtype or t.device != self.device or not t.is_contiguous() or tuple(t.shape) != shape:
            raise PctError("%s must be a contiguous %s %s tensor on %s" % (what, shape, dtype, self.device))
        return t

    def query_placements(self, queries, env_idx=None, density=None, out=None):
        """Space.drop_box_virtual(dims, (lx, ly), False, density, setting, returnH=True) (D:space.py:393-433, C:space.py:380-425) for k
        placements of each of n envs, enqueued on the current stream (graph-capturable, read-only: a step after a query behaves as without it).
        queries: (n, k, 5) tensor of [x, y, z, lx, ly] (oriented sizes, then the position), converted to int32 (discrete) / float64
        (continuous) on the batch's device.  Row r asks env env_idx[r] (default: env r); the envs of one call must be distinct, and rows of
        an index outside [0, n_envs) answer infeasible / 0.  density: (n, k) densities (default: each env's current item density).
        out: optional preallocated (feasible, rest_height) pair.  -> (feasible (n, k) bool, rest_height (n, k) int32 | float64)."""
        qd = torch.float64 if self.continuous else torch.int32
        if not torch.is_tensor(queries):
            queries = torch.as_tensor(np.asarray(queries))
        if queries.dim() != 3 or queries.shape[2] != 5:
            raise PctError("queries must have shape (n, k, 5): [x, y, z, lx, ly] per placement")
        n, k = int(queries.shape[0]), int(queries.shape[1])
        q = queries.to(device=self.device, dtype=qd).contiguous()
        idx = self._index(env_idx, "env_idx")
        if idx is not None and int(idx.numel()) != n:
            raise PctError("env_idx must have one entry per query row (%d)" % n)
        if idx is None and n > self.n_envs:
            raise PctError("%d query rows without env_idx for %d envs" % (n, self.n_envs))
        den = None
        if density is not None:
            if not torch.is_tensor(density):
                density = torch.as_tensor(np.asarray(density, dtype=np.float64))
            if tuple(density.shape) != (n, k):
                raise PctError("density must have shape (n, k) = (%d, %d)" % (n, k))
            den = density.to(device=self.device, dtype=torch.float64).contiguous()
        if out is None:
            feas = torch.empty((n, k), dtype=torch.bool, device=self.device)
            rest = torch.empty((n, k), dtype=qd, device=self.device)
        else:
            if len(out) != 2:
                raise PctError("out must be a (feasible, rest_height) pair")
            feas = self._out(out[0], (n, k), torch.bool, "out[0] (feasible)")
            rest = self._out(out[1], (n, k), qd, "out[1] (rest_height)")
        ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None and t.numel() else None
        fn, what = (self.L.pct_query_placements_f64, "pct_query_placements_f64") if self.continuous else (self.L.pct_query_placements, "pct_query_placements")
        self._check(fn(self.h, ptr(idx), n, k, ptr(q), ptr(den), ptr(feas), ptr(rest), self._stream()), what)
        return feas, rest

    def height_maps(self, env_idx=None, out=None):
        """Space.plain[:W, :L] (D:space.py:278, 317-326), the height map, of envs env_idx (default: every env) -> (n, W, L) int32 CUDA
        tensor, filled on the current stream (graph-capturable, read-only).  Indices outside [0, n_envs) give a zero map.  Discrete only."""
        if self.continuous:
            raise PctError("height_maps: the continuous Space has no height map (discrete domain only)")
        idx = self._index(env_idx, "env_idx")
        n = self.n_envs if idx is None else int(idx.numel())
        shape = (n, int(self.container_size[0]), int(self.container_size[1]))
        out = torch.empty(shape, dtype=torch.int32, device=self.device) if out is None else self._out(out, shape, torch.int32, "height_maps out")
        self._check(self.L.pct_height_maps(self.h, C.c_void_p(idx.data_ptr()) if idx is not None and n else None, n,
                                           C.c_void_p(out.data_ptr()) if out.numel() else None, self._stream()), "pct_height_maps")
        return out

    # -- item preview and item override (include/pct_b200.h): lookahead and buffer packing ---------------------------------
    def preview_items(self, k=1, env_idx=None, out=None):
        """BoxCreator.preview(k) (binCreator.py) of envs env_idx (default: every env) -> (n, k, 4) float64 CUDA tensor of [x, y, z, density],
        filled on the current stream (graph-capturable, read-only).  [:, 0] is each env's current item (preview_items()[:, 0, :3] is the
        batched current-item accessor), [:, j] the item its source delivers j - 1 draws later.  A reset in between (trajectory jumps)
        makes the entries past it stale.  Rows of an index outside [0, n_envs) are zeros."""
        k = int(k)
        if k < 1:
            raise PctError("preview_items: k must be >= 1")
        idx = self._index(env_idx, "env_idx")
        n = self.n_envs if idx is None else int(idx.numel())
        shape = (n, k, 4)
        out = torch.empty(shape, dtype=torch.float64, device=self.device) if out is None else self._out(out, shape, torch.float64, "preview_items out")
        self._check(self.L.pct_preview_items(self.h, C.c_void_p(idx.data_ptr()) if idx is not None and n else None, n, k,
                                             C.c_void_p(out.data_ptr()) if out.numel() else None, self._stream()), "pct_preview_items")
        return out

    def set_items(self, items, env_idx=None, density=None, out=None, info=None):
        """Env env_idx[i] (default: env i) <- items[i] as its current item, without consuming a draw, then the leaf expansion of
        cur_observation for it (the reference's `env.next_box = item` + get_possible_position()).  items: (n, 3) sizes, converted to int32
        (discrete) / float64 (continuous); density: (n,) densities (default: keep each env's current density).  EVERY env of the batch is
        re-expanded (envs not listed come out unchanged), and the complete observation goes to `out` (default: the batch's own observation
        buffer, under the delta-row contract of step), which is returned.  info: optional (n_envs, 8) int32 tensor for the pct_step_info
        records (capacity flags of the new expansions, n_leaf, ...).  The envs of one call must be distinct.  No items (n == 0): nothing is
        enqueued and nothing is written."""
        qd = torch.float64 if self.continuous else torch.int32
        if not torch.is_tensor(items):
            items = torch.as_tensor(np.asarray(items))
        if items.dim() != 2 or items.shape[1] != 3:
            raise PctError("items must have shape (n, 3): [x, y, z] per item")
        n = int(items.shape[0])
        it = items.to(device=self.device, dtype=qd).contiguous()
        idx = self._index(env_idx, "env_idx")
        if idx is not None and int(idx.numel()) != n:
            raise PctError("env_idx must have one entry per item (%d)" % n)
        if idx is None and n > self.n_envs:
            raise PctError("%d items without env_idx for %d envs" % (n, self.n_envs))
        den = None
        if density is not None:
            if not torch.is_tensor(density):
                density = torch.as_tensor(np.asarray(density, dtype=np.float64))
            if tuple(density.shape) != (n,):
                raise PctError("density must have shape (n,) = (%d,)" % n)
            den = density.to(device=self.device, dtype=torch.float64).contiguous()
        obs = self._obs if out is None else self._out(out, (self.n_envs, self.obs_len), self.obs_dtype, "set_items out")
        if info is not None:
            info = self._out(info, (self.n_envs, 8), torch.int32, "set_items info")
        ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None and t.numel() else None
        self._check(self.L.pct_set_items(self.h, ptr(idx), n, ptr(it), ptr(den), C.c_void_p(obs.data_ptr()), ptr(info), self._stream()),
                    "pct_set_items")
        return obs

    # -- host-buffer API (what the reference's VecEnv exchanges over its pipes) --------------------------------
    def reset_host(self, obs_out):
        self._check(self.L.pct_reset_host(self.h, C.c_void_p(obs_out.ctypes.data)), "pct_reset_host")
        self.did_reset = True
        return obs_out

    def step_host(self, obs_out, rew_out, done_out, info_out=None, actions=None, leaf_idx=None):
        a_ptr, i_ptr, f64 = None, None, 0
        if actions is not None:
            a_ptr, f64 = C.c_void_p(actions.ctypes.data), int(actions.dtype == np.float64)
        else:
            i_ptr = C.c_void_p(leaf_idx.ctypes.data)
        self._check(self.L.pct_step_host(self.h, a_ptr, f64, i_ptr, C.c_void_p(obs_out.ctypes.data), C.c_void_p(rew_out.ctypes.data),
                                         C.c_void_p(done_out.ctypes.data), C.c_void_p(info_out.ctypes.data) if info_out is not None else None),
                    "pct_step_host")

    # -- introspection -------------------------------------------------------------------------------------
    @staticmethod
    def check_flags(flags, ignore=0, what="pct_step"):
        """Raise PctError when any env's step record carries a capacity / hand-over flag (pct_step_info.flags) outside `ignore`: a flagged env's
        results are not the reference's (which would have raised IndexError / ValueError, or has no such limit).  Used by PctVecEnv,
        evaluate_batched and run_heuristic; low-level PctBatch.step callers check `decode_info(info)['flags']` themselves."""
        f = np.asarray(flags).astype(np.int64) & ~int(ignore)
        if f.any():
            bad = np.nonzero(f)[0]
            names = sorted({nm for v in f[bad] for bit, nm in _lib.FLAG_NAMES.items() if v & bit})
            raise PctError("%s flagged %d env(s) (first: env %d, flags %d = %s) — results of flagged envs are not the reference's"
                           % (what, len(bad), int(bad[0]), int(f[bad[0]]), "|".join(names)))

    @staticmethod
    def decode_info(info_cpu):
        """(N,8) int32 tensor/array of pct_step_info records -> dict of numpy arrays."""
        a = info_cpu.cpu().numpy() if hasattr(info_cpu, "cpu") else np.asarray(info_cpu)
        f = a.view(np.float32)
        return dict(counter=a[:, 0], flags=a[:, 1], ratio=f[:, 2], ep_reward=f[:, 3], ep_len=a[:, 4], n_leaf=a[:, 5], n_cand=a[:, 6],
                    n_ems=a[:, 7])

    def state(self, env):
        d = _lib.StateDump()
        self._check(self.L.pct_get_state(self.h, int(env), C.byref(d)), "pct_get_state")
        boxes = np.array([list(d.boxes[i]) for i in range(d.n_boxes)]).reshape(-1, 7)
        ems = np.array([list(d.ems[i]) for i in range(min(d.n_ems, 256))]).reshape(-1, 6)
        return dict(n_boxes=d.n_boxes, n_ems=d.n_ems, n_leaf=d.n_leaf, flags=d.flags, draw_pos=d.draw_pos,
                    next_box=list(d.next_box), next_den=d.next_den, boxes=boxes, ems=ems)

    def profile(self, on=True):
        self._check(self.L.pct_profile_enable(self.h, int(on)), "pct_profile_enable")

    def profile_read(self):
        """-> ({'apply': ms, 'candidates': ms, 'feas_emit': ms} summed over the recorded steps, n_steps)"""
        ms = (C.c_double * 3)()
        n = C.c_int32()
        self._check(self.L.pct_profile_read(self.h, ms, C.byref(n)), "pct_profile_read")
        return dict(apply=ms[0], candidates=ms[1], feas_emit=ms[2]), n.value

    @property
    def kernel_launches(self):
        return int(self.L.pct_kernel_launches(self.h))

    @property
    def state_bytes_per_env(self):
        return int(self.L.pct_state_bytes_per_env(self.h))

    def close(self):
        if getattr(self, "h", None):
            self.L.pct_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
