"""Item preview and item override of buffered envs (pct_buffer_preview_items / pct_buffer_set_items; DESIGN.md section 21), test
infrastructure:

- ItemsOracle: the buffered env on the oracle (tests/buffer_oracle.py: BufferedOracle) with the two calls, set_items(buf) and preview(k).
- one_ply_any_source: the one-ply lookahead of tests/buffer_search.py for a search batch whose item source is unrelated to the roots'
  (INTEGRATION.md, "Search without mirrored streams").  The test runs exactly this code (tests/test_gpu_buffer_items.py).
"""
import numpy as np

from buffer_oracle import BufferedOracle


class ItemsOracle(BufferedOracle):
    """BufferedOracle with pct_buffer_set_items / pct_buffer_preview_items"""

    def set_items(self, buf):
        """pct_buffer_set_items: the B slots <- buf ((B, 4) [x, y, z, density]; discrete sizes truncated and clamped to [0, 255]), no draw
        consumed, every slot re-observed; the new slots' flags join the sticky ones -> (obs, record) with record = dict(counter, flags,
        n_leaf, n_cand, n_ems, slot_flags), the fields pct_set_items writes"""
        buf = np.array(buf, dtype=np.float64).reshape(self.B, 4)
        if self.c["domain"] == "discrete":
            buf[:, :3] = np.clip(np.trunc(buf[:, :3]), 0, 255)
        self.buf[:] = buf
        self._observe()
        self.sticky |= self.slot_flags
        rec = dict(counter=len(self.orc.packed), flags=self.sticky, n_leaf=int(self.n_leaf.sum()), n_cand=int(self.n_cand.sum()),
                   n_ems=len(self.orc.ems()), slot_flags=self.slot_fl.copy())
        return self.obs, rec

    def preview(self, k):
        """pct_buffer_preview_items: the next k draws, (k, 4): the items the next placing steps put into the slots they empty"""
        L = len(self.stream)
        return self.stream[[(self.pos + i) % L for i in range(k)]].copy()


def one_ply_any_source(root, search, flats):
    """buffer_search.one_ply for a search batch with an item source of its own, unrelated to the roots'.  After the children step, each
    child's buffer is set to what its root would hold.  A placing step refilled the slot it emptied from the search batch's source: that
    slot takes the root's buffer_preview_items(1), the draw at the root's position.  A child whose episode ended refilled all B slots from
    the draw position the root holds (the reset draws B items from there when no trajectory length is set): they take the root's next B
    draws.  Under set_trajectory_length the reset jumps to the next trajectory first, so such roots would need the preview at the jump;
    this example is for batches without one.  Still without `shuffle` (the keyed shuffle uses the env index).  Then commit as one_ply
    does; -> (n,) the flat index each root took."""
    import torch
    n, K = flats.shape
    dev = root.device
    B, nl = root.buffer, root.nl
    rec = torch.arange(n, device=dev, dtype=torch.int32).repeat_interleave(K)
    search.buffer_restore(root.buffer_snapshot(), rec_idx=rec, write_obs=False)
    every = torch.ones(n * K, dtype=torch.bool, device=dev)
    _, reward, done, _ = search.buffer_step_envs(flats.reshape(-1), mask=every)
    nxt = root.buffer_preview_items(B)[rec.long()]  # (n * K, B, 4): each child's root's next B draws
    buf = search.buffer_items()
    f = flats.reshape(-1).long()
    j = torch.where((f >= 0) & (f < B * nl), f // nl, torch.zeros_like(f))  # the slot a placing step emptied
    buf[torch.arange(n * K, device=dev), j] = nxt[:, 0]
    ended = done.bool()
    buf[ended] = nxt[ended]
    search.buffer_set_items(buf)
    best = reward.view(n, K).argmax(dim=1)
    child = torch.arange(n, device=dev) * K + best
    root.buffer_restore(search.buffer_snapshot(env_idx=child))
    return flats[torch.arange(n, device=dev), best]
