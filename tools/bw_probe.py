import torch, time
x = torch.empty(8*1024*1024*16, dtype=torch.float16, device="cuda")
y = torch.empty_like(x)
def t(f, n=20):
    for _ in range(3): f()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): f()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3
nb = x.numel() * 2
us = t(lambda: x.fill_(1.0)); print(f"fill 268MB: {us:.1f} us  {nb/us/1e6:.2f} TB/s write")
us = t(lambda: y.copy_(x)); print(f"copy 268MB: {us:.1f} us  {2*nb/us/1e6:.2f} TB/s r+w")
us = t(lambda: x.sum()); print(f"read 268MB: {us:.1f} us  {nb/us/1e6:.2f} TB/s read")
big = torch.empty(1<<30, dtype=torch.float16, device="cuda")
us = t(lambda: big.fill_(1.0), 5); print(f"fill 2GB: {us:.1f} us  {big.numel()*2/us/1e6:.2f} TB/s write")
# L2-resident read rate: ONE reduction kernel reads a 20 MB buffer (inside the 50 MB L2) 64 times over -- the buffer is
# viewed as 64 rows of stride 0, so every row is the same memory and nothing is copied; after the first pass every read
# hits L2 (each row is far larger than an SM's L1), and the kernel runs long enough (~1 GB read) that launch gaps do not count
l2 = torch.ones(10 * 1024 * 1024, dtype=torch.float16, device="cuda")
rows = l2.expand(64, l2.numel())
us = t(lambda: rows.sum(dim=1), 10); print(f"read 20MB x 64 (L2-resident): {us:.1f} us  {rows.numel()*2/us/1e6:.2f} TB/s read")
