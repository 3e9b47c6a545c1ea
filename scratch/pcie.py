import sys, time, torch
sys.path.insert(0, __import__('os').path.dirname(__import__('os').path.dirname(__import__('os').path.abspath(__file__))))
for mb in (4.83, 19.3, 38.6, 256):
    nb = int(mb * 1e6)
    d = torch.empty(nb, dtype=torch.uint8, device='cuda'); h = torch.empty(nb, dtype=torch.uint8, pin_memory=True)
    for _ in range(3): h.copy_(d, non_blocking=True)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20): h.copy_(d, non_blocking=True)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 20
    e0.record()
    for _ in range(20): d.copy_(h, non_blocking=True)
    e1.record(); torch.cuda.synchronize()
    ms2 = e0.elapsed_time(e1) / 20
    print("%.1f MB: D2H %.3f ms = %.1f GB/s   H2D %.3f ms = %.1f GB/s" % (mb, ms, nb / ms / 1e6, ms2, nb / ms2 / 1e6), flush=True)
