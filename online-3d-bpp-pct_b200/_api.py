"""Public surface of pct_b200."""
from . import _lib
from ._lib import build, LIB_PATH
from .batch import PctBatch, PctError

__all__ = ["PctBatch", "PctError", "build", "LIB_PATH"]
try:  # host-side mirror of the reference's gym.Env / VecEnv surface
    from .vec_env import PctVecEnv
    from .envs import PackingDiscrete, PackingContinuous, make_vec_envs, registration_envs
    from .distributed import shard_range, make_sharded_vec_env, gather_observations
    from .rollout import GraphedRollout, drl_gat_policy, buffered_drl_gat
    from .evaluation import evaluate_batched, load_trajectories
    from .heuristics import run_heuristic, HEURISTICS
    __all__ += ["PctVecEnv", "PackingDiscrete", "PackingContinuous", "make_vec_envs", "registration_envs", "shard_range",
                "make_sharded_vec_env", "gather_observations", "GraphedRollout", "drl_gat_policy", "buffered_drl_gat", "evaluate_batched", "load_trajectories",
                "run_heuristic", "HEURISTICS"]
except ImportError:  # pragma: no cover - during bring-up
    pass
