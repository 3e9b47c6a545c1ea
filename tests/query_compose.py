"""DBL and HM (heuristic.py:431-493, :232-293) written in torch on two primitives only: a batch's height_maps() and query_placements().

This is what a user writes to try a placement rule of their own on thousands of envs.  The GPU tests check that it picks exactly the
row of the built-in heuristic_actions("DBL" / "HM"); the CPU tests run it on an oracle-backed stand-in of the two calls.
"""
import torch

# `x, y, z = next_box`, `y, x, z = ...`, `z, x, y = ...`, `z, y, x = ...`, `x, z, y = ...`, `y, z, x = ...` (heuristic.py:176-187)
ROT = ((0, 1, 2), (1, 0, 2), (1, 2, 0), (2, 1, 0), (0, 2, 1), (2, 0, 1))
NO_ROW = (1.0, 0, 0, 1.0, 0, 0, 0, 0, 1.0)  # matches no item: the step ends the episode, like the reference's "no placement"


def grid_queries(next_box, W, L, setting):
    """(n, 3) int next items -> queries (n, W*L*R, 5) in the enumeration order of heuristic.py:253-254 (lx, then ly, then the
    rotation), and the mask of the grid points inside the loop bounds of the UNROTATED item"""
    R = 6 if setting == 2 else 2
    n, dev = next_box.shape[0], next_box.device
    nb = next_box.to(torch.int64)
    dims = nb[:, torch.tensor(ROT[:R], device=dev)]                                  # (n, R, 3)
    lx = torch.arange(W, device=dev).view(1, W, 1, 1).expand(n, W, L, R)
    ly = torch.arange(L, device=dev).view(1, 1, L, 1).expand(n, W, L, R)
    q = torch.cat([dims.view(n, 1, 1, R, 3).expand(n, W, L, R, 3), lx[..., None], ly[..., None]], dim=-1)
    inside = (lx < (W - nb[:, 0] + 1).view(n, 1, 1, 1)) & (ly < (L - nb[:, 1] + 1).view(n, 1, 1, 1))
    return q.reshape(n, W * L * R, 5), inside.reshape(n, W * L * R)


def composed_rows(batch, name, next_box):
    """(n, 9) float32 action rows of DBL / HM for every env of `batch`, whose current items are `next_box` (n, 3)"""
    W, L = int(batch.container_size[0]), int(batch.container_size[1])
    q, inside = grid_queries(next_box, W, L, batch.setting)
    feas, h = batch.query_placements(q)
    q, h = q.to(torch.int64), h.to(torch.int64)
    sx, sy, sz, lx, ly = q.unbind(-1)
    if name == "DBL":  # heuristic.py:482
        score = lx + ly + 100 * h
    elif name == "HM":  # heuristic.py:281: 100 * np.sum(height map after the placement)
        hm = batch.height_maps().to(torch.int64)
        n = hm.shape[0]
        S = torch.zeros((n, W + 1, L + 1), dtype=torch.int64, device=hm.device)
        S[:, 1:, 1:] = hm.cumsum(1).cumsum(2)
        x2, y2 = (lx + sx).clamp(max=W), (ly + sy).clamp(max=L)
        at = lambda i, j: S.view(n, -1).gather(1, i * (L + 1) + j)
        foot = at(x2, y2) - at(lx, y2) - at(x2, ly) + at(lx, ly)
        score = lx + ly + 100 * (hm.sum((1, 2))[:, None] - foot + sx * sy * (h + sz))
    else:
        raise ValueError(name)
    ok = feas & inside
    K = q.shape[1]
    key = torch.where(ok, score * K + torch.arange(K, device=q.device), torch.iinfo(torch.int64).max)  # first minimum in enumeration order
    best = key.argmin(1)
    c = q[torch.arange(q.shape[0], device=q.device), best]
    sx, sy, lx, ly = c[:, 0], c[:, 1], c[:, 3], c[:, 4]
    z = torch.zeros_like(lx)
    rows = torch.stack([lx, ly, z, lx + sx, ly + sy, z, z, z, torch.ones_like(lx)], 1).to(torch.float32)
    return torch.where(ok.any(1)[:, None], rows, torch.tensor(NO_ROW, dtype=torch.float32, device=q.device))
