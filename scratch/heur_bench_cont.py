import sys, time, torch
sys.path.insert(0, __import__('os').path.dirname(__import__('os').path.dirname(__import__('os').path.abspath(__file__))))
import pct_b200
items = [(round(0.1 * i, 1), round(0.1 * j, 1), round(0.1 * k, 1)) for i in range(1, 6) for j in range(1, 6) for k in range(1, 6)]
for name, setting, n in (("LSAH", 2, 4096), ("OnlineBPH", 2, 4096), ("BR", 2, 4096), ("LSAH", 1, 4096), ("OnlineBPH", 1, 4096), ("BR", 1, 4096)):
    b = pct_b200.PctBatch(n, setting, container_size=(1.0, 1.0, 1.0), item_set=items, continuous=True, sample_from_distribution=True, seed=3)
    b.reset()
    for t in range(30):
        b.step(actions=b.heuristic_actions(name))
    torch.cuda.synchronize()
    e0, e1, e2 = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    K, sel = 100, 0.0
    t0 = time.perf_counter()
    for t in range(K):
        e0.record(); rows = b.heuristic_actions(name); e1.record()
        b.step(actions=rows)
        e1.synchronize(); sel += e0.elapsed_time(e1)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    print("%-9s continuous setting %d  %5d envs: %.3f ms/step (selection kernel %.3f ms)  %.2fM placements/s" % (name, setting, n, dt / K * 1e3, sel / K, n * K / dt / 1e6), flush=True)
    b.close()
