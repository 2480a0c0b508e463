"""Runs a few LSIGF forward+backward steps on the headline workload (for a profiler's launch list of the backward pass)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import gnn_b200
from gnn_b200 import graphs
N, K, G, F, B = 1_000_000, 5, 64, 64, 1
gso = graphs.er_gso(N, 32, seed=1)
g = torch.Generator().manual_seed(0)
bound = 1 / np.sqrt(G * K)
h = ((torch.rand(F, 1, K, G, generator=g) * 2 - 1) * bound).cuda().requires_grad_(True)
b = ((torch.rand(F, 1, generator=g) * 2 - 1) * bound).cuda().requires_grad_(True)
x = torch.randn(B, G, N, generator=g).cuda().requires_grad_(True)
dy = torch.randn(B, F, N, generator=g).cuda()
torch.cuda.synchronize()
steps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
for i in range(steps):
    x.grad = h.grad = b.grad = None
    torch.cuda.nvtx.range_push("step")
    y = gnn_b200.LSIGF(h, gso, x, b)
    y.backward(dy)
    torch.cuda.nvtx.range_pop()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for i in range(5):
    x.grad = h.grad = b.grad = None
    gnn_b200.LSIGF(h, gso, x, b).backward(dy)
e1.record(); torch.cuda.synchronize()
print("fwd+bwd ms/step", e0.elapsed_time(e1) / 5)
