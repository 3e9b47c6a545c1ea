"""One-ply lookahead over a buffered batch (INTEGRATION.md, "Lookahead over a buffered batch"): branch every root env into K children in a
search batch of the same configuration, step each child with a different flat leaf index, and commit the best child's state over its root.

The search batch must draw what its root would draw: its item stream repeats each root's stream row K times (child i * K + k has root i's row),
and the batch is built without `shuffle` (the keyed shuffle uses the env index).  The test runs exactly this code
(tests/test_gpu_buffer_envs.py)."""
import torch


def candidate_flats(obs, nb, nl, B, K, gen):
    """(n, K) flat leaf indices j * NL + l: K distinct valid leaves of each env's buffered observation, drawn at random (invalid ones,
    the zero action, fill the rest when an env has fewer than K leaves)"""
    n = obs.shape[0]
    valid = obs[:, nb * 9:(nb + B * nl) * 9].reshape(n, B * nl, 9)[:, :, 8] == 1
    key = torch.rand((n, B * nl), generator=gen, device=obs.device) + valid.to(torch.float32)
    return key.topk(K, dim=1).indices.to(torch.int32)


def one_ply(root, search, flats):
    """root: buffered PctBatch of n envs; search: one of n * K envs, same configuration.  flats: (n, K) flat leaf indices.
    Commits, on every root, the child with the highest reward (the first on a tie); -> (n,) the flat index each root took."""
    n, K = flats.shape
    dev = root.device
    snaps = root.buffer_snapshot()
    rec = torch.arange(n, device=dev, dtype=torch.int32).repeat_interleave(K)
    search.buffer_restore(snaps, rec_idx=rec, write_obs=False)
    every = torch.ones(n * K, dtype=torch.bool, device=dev)
    _, reward, _, _ = search.buffer_step_envs(flats.reshape(-1), mask=every)
    best = reward.view(n, K).argmax(dim=1)
    child = torch.arange(n, device=dev) * K + best
    root.buffer_restore(search.buffer_snapshot(env_idx=child))
    return flats[torch.arange(n, device=dev), best]
