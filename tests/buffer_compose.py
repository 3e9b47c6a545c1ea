"""Buffer packing ("online packing with buffer": the agent picks one of B buffered items, then places it) written in torch on public
PctBatch calls only: snapshot / restore, set_items, heuristic_actions and query_placements.

Each env keeps B items drawn from its own item sequence.  One decision:
  1. fans every env out into B children on a second batch (snapshot -> restore with rec_idx);
  2. sets buffered item j on child j (set_items);
  3. scores child j by the placement the built-in heuristic picks for it (DBL; continuous: LSAH): its rest height from
     query_placements, infeasible (no placement) = +inf.  Rule: the lowest rest height, ties to the lower buffer index;
  4. sets the chosen item on the env (set_items) and steps it with the child's action row;
  5. refills the buffer slot from the env's sequence.
A test helper (like query_compose.py), not a public API.
"""
import torch


def oriented_sizes(rows, items):
    """(m, 9) action rows and (m, 3) items -> (m, 3) oriented sizes [x, y, z]: LeafNode2Action (D:bin3D.py:139-149, C:bin3D.py:151-167),
    x and y are the row's extents and z is the item entry left after removing one entry equal to x, then one equal to y"""
    x, y = rows[:, 3] - rows[:, 0], rows[:, 4] - rows[:, 1]
    left = torch.ones_like(items, dtype=torch.bool)
    for ext in (x, y):
        hit = left & ((items - ext[:, None]).abs() < 1e-6)
        first = hit & (hit.cumsum(1) == 1)
        left = left & ~first
    z = torch.where(left, items, torch.zeros_like(items)).max(1).values  # the remaining entry (sizes are positive)
    return torch.stack([x, y, z], 1)


class BufferDriver(object):
    """parent: the PctBatch being packed; child: a PctBatch of the same configuration with parent.n_envs * B envs.
    source: (n, L, 4) float64 tensor of [x, y, z, density] per env, read cyclically to fill the buffers."""

    def __init__(self, parent, child, source, B):
        self.p, self.c, self.B = parent, child, B
        n = parent.n_envs
        assert child.n_envs == n * B
        self.src = source.to(parent.device)
        self.pos = B  # next position of every env's sequence
        self.buf = self.src[:, :B].clone()  # (n, B, 4)
        self.rec = torch.arange(n, device=parent.device).repeat_interleave(B)
        self.envs = torch.arange(n, device=parent.device)

    def decide(self):
        """one decision for every env -> (chosen items (n, 4), action rows (n, 9), buffer index (n,))"""
        n, B = self.p.n_envs, self.B
        self.c.restore(self.p.snapshot(), rec_idx=self.rec, write_obs=False)
        items = self.buf.reshape(n * B, 4)
        self.c.set_items(items[:, :3], density=items[:, 3])
        rows = self.c.heuristic_actions("LSAH" if self.c.continuous else "DBL").clone()
        dims = oriented_sizes(rows.to(torch.float64), items[:, :3])
        q = torch.cat([dims, rows[:, :2].to(torch.float64)], 1).view(n * B, 1, 5)
        feas, rest = self.c.query_placements(q)
        score = torch.where(feas[:, 0], rest[:, 0].to(torch.float64), torch.full_like(rest[:, 0], float("inf"), dtype=torch.float64))
        j = score.view(n, B).argmin(1)  # first minimum: ties go to the lower buffer index
        chosen = self.buf[self.envs, j].clone()
        return chosen, rows.view(n, B, 9)[self.envs, j].contiguous(), j

    def step(self):
        """decide, set the chosen items, step, refill -> (chosen items, action rows, (obs after set_items), step outputs)"""
        chosen, act, j = self.decide()
        obs_set = self.p.set_items(chosen[:, :3], density=chosen[:, 3]).clone()
        out = self.p.step(actions=act)
        L = self.src.shape[1]
        self.buf[self.envs, j] = self.src[:, self.pos % L]
        self.pos += 1
        return chosen, act, obs_set, out
