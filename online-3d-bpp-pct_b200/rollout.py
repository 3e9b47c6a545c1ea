"""Device-resident n-step rollout (SURVEY.md §8(f)-1): policy -> env.step, T times, with no host round trip.

The reference collects rollouts as
    logp, idx, ... = policy(all_nodes); leaf = leaf_nodes[batchX, idx]; obs, r, d, infos = envs.step(leaf.cpu().numpy())
    pct_rollout.insert(...)                                             (train_tools.py:63-70, storage.py:33-39)
i.e. one device->host->device trip per step.  Here the selected leaf INDEX goes straight into pct_step, every observation is
written by the kernel directly into a (T+1, N, obs_len) storage tensor (the layout of PCTRolloutStorage.obs), and the whole
T-step sequence is captured once in a CUDA graph and replayed with a single launch.
"""
import torch


def drl_gat_policy(net, tools, internal_node_holder=80, leaf_node_holder=50, norm_factor=1.0, deterministic=False):
    """Adapter for the reference's UNMODIFIED policy network (model.DRL_GAT, loaded e.g. by compat.load_policy_modules): the calls of the
    collection loop train_tools.py:63-66 — tools.get_leaf_nodes on the observation, PCT_policy(all_nodes, normFactor=factor) -> (log-prob,
    index, entropy, value) — as a GraphedRollout policy.  The selected leaf INDEX goes straight into pct_step (the reference looks the leaf row
    up and ships it through numpy: `leaf_nodes[batchX, selectedIdx.squeeze()].cpu().numpy()`, :65-66; the kernel reads the same leaf by index).
    torch.distributions' argument validation synchronises with the host (simplex check), which a CUDA graph cannot capture: it is switched
    off globally here, as any graph-captured use of torch.distributions requires.  deterministic=True (evaluation's argmax) contains a
    host-side branch in the reference (`if torch.sum(masked_outs) == 0`, attention_model.py:140) and therefore only runs with use_graph=False."""
    import torch.distributions
    torch.distributions.Distribution.set_default_validate_args(False)

    def policy(obs, t_dev):
        all_nodes, _ = tools.get_leaf_nodes(obs, internal_node_holder, leaf_node_holder)
        logp, idx, _, value = net(all_nodes, deterministic, normFactor=norm_factor)
        return idx.reshape(-1), logp, value
    return policy


def buffered_drl_gat(net, B, internal_node_holder=80, leaf_node_holder=50):
    """The reference's DRL_GAT on a buffered batch (PctBatch(..., buffer=B)): `net` is built with leaf_node_holder = B * NL (the leaf
    blocks of the B items are one leaf list to its pointer), and its encoder's graph_size, fixed at construction, becomes the node count of
    a buffered observation, NB + B * NL + B (graph_encoder.py: `graph_size`).  The item rows after the leaf blocks are read as next-item rows
    by observation_decode_leaf_node (tools.py) and embedded by AttentionModel.forward as they are.  Drive it with
    drl_gat_policy(net, tools, internal_node_holder, B * leaf_node_holder); its leaf index is the batch's flat index j * NL + l."""
    net.actor.embedder.graph_size = int(internal_node_holder) + int(B) * int(leaf_node_holder) + int(B)
    return net


class GraphedRollout(object):
    """policy: callable(obs (N, obs_len) float32 CUDA tensor, t_dev int64 CUDA scalar tensor) -> int32 CUDA tensor (N,) of leaf indices,
    made of capturable torch ops (e.g. a DRL_GAT forward + argmax / multinomial); None = the built-in uniform-valid-leaf kernel.
    A policy may also return (indices, action_log_probs (N,1), values (N,1)) — see drl_gat_policy —: they are stored per step in
    `action_log_probs` / `value_preds`, and `masks` = 1 - done, i.e. every tensor PCTRolloutStorage.insert receives (storage.py:33-39)."""

    def __init__(self, batch, num_steps, policy=None, policy_seed=0, use_graph=True):
        self.batch, self.T, self.policy, self.seed = batch, int(num_steps), policy, int(policy_seed)
        n, dev = batch.n_envs, batch.device
        self.obs = torch.zeros((self.T + 1, n, batch.obs_len), dtype=batch.obs_dtype, device=dev)
        self.rewards = torch.zeros((self.T, n), dtype=torch.float32, device=dev)
        self.dones = torch.zeros((self.T, n), dtype=torch.uint8, device=dev)
        self.actions = torch.zeros((self.T, n), dtype=torch.int32, device=dev)
        self.action_log_probs = torch.zeros((self.T, n, 1), dtype=torch.float32, device=dev)
        self.value_preds = torch.zeros((self.T, n, 1), dtype=torch.float32, device=dev)
        self.masks = torch.ones((self.T + 1, n, 1), dtype=torch.float32, device=dev)
        self.t_dev = torch.zeros((), dtype=torch.int64, device=dev)
        self.graph = None
        self.use_graph = use_graph
        self._started = False

    def start(self):
        self.batch.reset(out=self.obs[0])
        self.t_dev.zero_()
        self._started = True

    def _steps(self):
        b = self.batch
        for t in range(self.T):
            if self.policy is None:
                idx = b.random_policy_dev(self.seed, self.t_dev, out=self.actions[t])
            else:
                out = self.policy(self.obs[t], self.t_dev)
                if isinstance(out, tuple):
                    idx, logp, value = out
                    self.action_log_probs[t].copy_(logp.reshape(-1, 1))
                    self.value_preds[t].copy_(value.reshape(-1, 1))
                else:
                    idx = out
                self.actions[t].copy_(idx.reshape(-1).to(torch.int32))
                idx = self.actions[t]
            _, r, d, _ = b.step(leaf_idx=idx, out=self.obs[t + 1])
            self.rewards[t].copy_(r)
            self.dones[t].copy_(d)
            self.masks[t + 1].copy_((1 - d.to(torch.float32)).reshape(-1, 1))  # train_tools.py:70 torch.tensor(1 - done)
            self.t_dev += 1

    def run(self):
        """One T-step rollout continuing from the last observation; returns (obs, rewards, dones, actions) storages."""
        if not self._started:
            self.start()
        else:
            self.obs[0].copy_(self.obs[self.T])  # storage.after_update (storage.py:41-43)
            self.masks[0].copy_(self.masks[self.T])
        if not self.use_graph:
            self._steps()
        else:
            if self.graph is None:
                # start() already launched every env kernel once (first launches set kernel attributes, which cannot be captured); a torch policy gets
                # one eager call on a side stream for the same reason (lazy cuBLAS / cuDNN handle creation and autotuning are not capturable)
                if self.policy is not None:
                    side = torch.cuda.Stream(device=self.batch.device)
                    side.wait_stream(torch.cuda.current_stream(self.batch.device))
                    with torch.cuda.stream(side):
                        for _ in range(2):
                            self.policy(self.obs[0], self.t_dev)
                    torch.cuda.current_stream(self.batch.device).wait_stream(side)
                    torch.cuda.synchronize(self.batch.device)
                self.graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self.graph):
                    self._steps()
            self.graph.replay()
        return self.obs, self.rewards, self.dones, self.actions
