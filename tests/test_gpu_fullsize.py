"""Oracle parity at BASELINE.json's FULL sizes (`pytest -m gpu`, H100): the CUDA path vs the fp64 CPU oracle on
random inputs with all feature columns distinct — forward and every gradient.  VERDICT r1 "weak #1": the earlier
full-size test only compared the CUDA path with itself (fixed point / linearity / adjoints).

The checker is oracle/lsigf_oracle.py:lsigf_sparse_stream / lsigf_grads_sparse_stream (restatement of graphML.py:83-176
and of its autograd, pinned to the reference-generated fixtures in tests/test_oracle_golden.py), with the sparse products
threaded over the host cores.  Tolerance: max|a - ref| / max|ref| <= 1e-4 (north_star), fp32 arithmetic on the GPU.
"""
import time

import numpy as np
import pytest
import torch

import lsigf_oracle as orc

pytestmark = pytest.mark.gpu

TOL32 = 1e-4

# the workloads of bench.py (same generators and seeds): headline, cfg2 (C = 2048), cfg4 (tensor GSO, E = 4)
CASES = {
    "er1m": dict(graph="er", N=1_000_000, deg=32, E=1, K=5, G=64, F=64, B=1, seed=1),
    "cfg2": dict(graph="er", N=100_000, deg=16, E=1, K=5, G=64, F=64, B=32, seed=2),
    "cfg4": dict(graph="er", N=200_000, deg=16, E=4, K=3, G=32, F=32, B=32, seed=4),
}


def rel(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


@pytest.mark.parametrize("name", ["er1m", "cfg2", "cfg4"])
def test_full_size_vs_oracle(name):
    import scipy.sparse as sp
    import gnn_b200
    from gnn_b200 import graphs
    gnn_b200._cabi.load()
    w = CASES[name]
    N, E, K, G, F, B = w["N"], w["E"], w["K"], w["G"], w["F"], w["B"]
    gso = graphs.er_gso(N, w["deg"], seed=w["seed"], E=E)
    g = torch.Generator().manual_seed(1234)
    bound = 1.0 / np.sqrt(G * K)
    h = (torch.rand(F, E, K, G, generator=g) * 2 - 1) * bound
    b = (torch.rand(F, 1, generator=g) * 2 - 1) * bound
    x = torch.randn(B, G, N, generator=g)                     # every (b, g) column different
    dy = torch.randn(B, F, N, generator=g)
    hd, bd, xd = (t.cuda().requires_grad_(True) for t in (h, b, x))
    y = gnn_b200.LSIGF(hd, gso, xd, bd)
    y.backward(dy.cuda())
    torch.cuda.synchronize()
    got = dict(y=y.detach().cpu().numpy(), dh=hd.grad.cpu().numpy(), dx=xd.grad.cpu().numpy(), db=bd.grad.cpu().numpy())
    del y, hd, xd, bd
    torch.cuda.empty_cache()

    t0 = time.time()
    S = [sp.csr_matrix((v.astype(np.float64), c, r), shape=(N, N)) for (r, c, v) in gso.csr]
    h64, b64, x64, dy64 = (t.double().numpy() for t in (h, b, x, dy))
    want_y = orc.lsigf_sparse_stream(h64, S, x64, b64, spmm=orc.threaded_spmm)
    want_dh, want_dx, want_db = orc.lsigf_grads_sparse_stream(h64, S, x64, dy64, (F, 1), spmm=orc.threaded_spmm)
    errs = dict(y=rel(got["y"], want_y), dh=rel(got["dh"], want_dh), dx=rel(got["dx"], want_dx), db=rel(got["db"], want_db))
    print("full-size parity %s: %s  (oracle %.1f s)" % (name, {k: "%.2e" % v for k, v in errs.items()}, time.time() - t0))
    assert max(errs.values()) < TOL32, errs
