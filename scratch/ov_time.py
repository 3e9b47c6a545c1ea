import sys, time, torch
sys.path.insert(0, __import__('os').path.dirname(__import__('os').path.dirname(__import__('os').path.abspath(__file__))))
import pct_b200
n = int(sys.argv[1]); setting = int(sys.argv[2])
items = [(i, j, k) for i in range(1, 6) for j in range(1, 6) for k in range(1, 6)]
b = pct_b200.PctBatch(n, setting, item_set=items, seed=1234)
b.reset()
flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
for t in range(200):
    b.step(leaf_idx=b.random_policy(99, t))
torch.cuda.synchronize()
K = 600
ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(K)]
for t in range(K):
    flush.zero_()
    ev[t][0].record()
    idx = b.random_policy(99, 200 + t)
    b.step(leaf_idx=idx)
    ev[t][1].record()
torch.cuda.synchronize()
ms = sorted(e0.elapsed_time(e1) for e0, e1 in ev)
info = b._info.cpu()
print("n=%d s=%d: %.4f ms/step (p50 %.4f p99 %.4f) -> %.2fM env-steps/s   flags_or=%d" % (n, setting, sum(ms) / K, ms[K // 2], ms[int(K * .99)], n * K / sum(ms) / 1e3, int(info[:, 1].max())), flush=True)
