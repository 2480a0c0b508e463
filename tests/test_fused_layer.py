"""SURVEY.md §8 f-1: the fused `GraphFilter -> ReLU -> MaxPoolLocal` layer (reference: alegnn/modules/architectures.py:274-296,
alegnn/utils/graphML.py:1968-2019) against fixtures produced by the UNMODIFIED reference (tests/golden/layer_cases.npz,
oracle/make_golden.py:gen_layer).

CPU leg: the host logic (fuse_layers rewiring, bias / activation plumbing, neighbourhood matrix) with the oracle standing
in for the two CUDA dispatch hooks.  GPU leg: ReLU in the contraction epilogue (tensor-core and FMA kernels), its
backward from the saved output, the CUDA max-pool gather and its arg-max scatter — forward and every gradient.
"""
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

import lsigf_oracle as orc


def rel(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def _cases(golden_dir):
    z = np.load(os.path.join(golden_dir, "layer_cases.npz"))
    return z, sorted({k.split("_")[0] for k in z.files})


def _build(z, c, dtype, device):
    import gnn_b200
    N, Nout, B, G, F, K, E, hops = (int(v) for v in z[c + "_meta"])
    S = torch.tensor(z[c + "_S"], dtype=dtype, device=device)
    gf = gnn_b200.GraphFilter(G, F, K, E, True)
    gf.load_state_dict({"weight": torch.tensor(z[c + "_weight"]), "bias": torch.tensor(z[c + "_bias"])})
    gf = gf.to(dtype=dtype, device=device)
    gf.addGSO(S)
    pool = gnn_b200.MaxPoolLocal(N, Nout, hops)
    pool.addGSO(S)
    net = nn.Sequential(gf, nn.ReLU(), pool)
    return net, gf, pool


def test_fuse_layers_host_logic(golden_dir, monkeypatch):
    import gnn_b200
    from gnn_b200 import graphML, pooling
    z, cases = _cases(golden_dir)

    def dispatch(h, S, x, b, act=0):                 # oracle stand-in for the CUDA dispatch (activation included)
        y = orc.lsigf_dense_torch(h, S, x, b)
        return torch.relu(y) if act else y

    def gather_max(x, nb32, n_out, max_nb):          # torch stand-in for the CUDA gather
        B, F, _ = x.shape
        return x.index_select(2, nb32.reshape(-1).long()).reshape(B, F, n_out, max_nb).max(dim=3)[0]

    monkeypatch.setattr(graphML, "_dispatch", dispatch)
    monkeypatch.setattr(pooling, "_gather_max", gather_max)
    for c in cases:
        net, gf, pool = _build(z, c, torch.float64, "cpu")
        # same neighbourhoods as the reference layer (the reference lists them in python-set order, here sorted)
        assert np.array_equal(np.sort(pool.neighborhood.numpy(), axis=1), np.sort(z[c + "_neighborhood"], axis=1))
        keys_before = sorted(net.state_dict().keys())
        assert gnn_b200.fuse_layers(net) == 1
        assert gf.fused_activation == "relu" and isinstance(net[1], nn.Identity)
        assert sorted(net.state_dict().keys()) == keys_before                         # checkpoint keys unchanged
        x = torch.tensor(z[c + "_x"], requires_grad=True)
        y = net(x)
        y.backward(torch.tensor(z[c + "_dy"]))
        assert rel(y.detach().numpy(), z[c + "_y"]) < 1e-12
        assert rel(x.grad.numpy(), z[c + "_dx"]) < 1e-11
        assert rel(gf.weight.grad.numpy(), z[c + "_dweight"]) < 1e-11
        assert rel(gf.bias.grad.numpy(), z[c + "_dbias"]) < 1e-11
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        pooling._gather_max_cuda(torch.zeros(1, 1, 3), torch.zeros(3, 1, dtype=torch.int32), 3, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-11), (torch.float32, 1e-4)])
@pytest.mark.parametrize("fuse", [True, False])
def test_fused_layer_golden_gpu(golden_dir, dtype, tol, fuse):
    import gnn_b200
    gnn_b200._cabi.load()
    z, cases = _cases(golden_dir)
    for c in cases:
        net, gf, pool = _build(z, c, dtype, "cuda")
        if fuse:
            assert gnn_b200.fuse_layers(net) == 1
        x = torch.tensor(z[c + "_x"], dtype=dtype, device="cuda", requires_grad=True)
        y = net(x)
        y.backward(torch.tensor(z[c + "_dy"], dtype=dtype, device="cuda"))
        torch.cuda.synchronize()
        assert tuple(y.shape) == z[c + "_y"].shape
        errs = dict(y=rel(y.detach().cpu().numpy(), z[c + "_y"]), dx=rel(x.grad.cpu().numpy(), z[c + "_dx"]),
                    dw=rel(gf.weight.grad.cpu().numpy(), z[c + "_dweight"]), db=rel(gf.bias.grad.cpu().numpy(), z[c + "_dbias"]))
        assert max(errs.values()) < tol, (c, fuse, errs)


@pytest.mark.gpu
def test_fused_relu_on_the_tensor_core_contraction():
    """G = F = 64 takes the wgmma contraction: its epilogue applies the ReLU; backward masks with the saved output."""
    import gnn_b200
    from gnn_b200 import graphs
    N, K, G, F, B = 30000, 4, 64, 64, 2
    gso = graphs.er_gso(N, 10, seed=3)
    gen = torch.Generator().manual_seed(2)
    h = ((torch.rand(F, 1, K, G, generator=gen) - 0.5) * 0.3).cuda().requires_grad_(True)
    b = ((torch.rand(F, 1, generator=gen) - 0.5) * 0.3).cuda().requires_grad_(True)
    x = torch.randn(B, G, N, generator=gen).cuda().requires_grad_(True)
    dy = torch.randn(B, F, N, generator=gen).cuda()
    y_f = gnn_b200.LSIGF(h, gso, x, b, activation="relu")
    y_f.backward(dy)
    g_f = [t.grad.clone() for t in (h, x, b)]
    for t in (h, x, b):
        t.grad = None
    y_u = torch.relu(gnn_b200.LSIGF(h, gso, x, b))
    y_u.backward(dy)
    assert torch.equal(y_f, y_u)                                  # same kernel arithmetic, max(., 0) in the epilogue
    for a, r in zip(g_f, (h.grad, x.grad, b.grad)):
        assert rel(a.cpu().numpy(), r.cpu().numpy()) < 1e-6
    assert float((y_f == 0).float().mean()) > 0.2                # the mask really is active


@pytest.mark.gpu
def test_maxpool_cuda_on_a_large_sparse_graph():
    """CUDA gather-max + arg-max scatter vs a torch gather on a 200k-node graph (node-major in, node-major out)."""
    import gnn_b200
    from gnn_b200 import graphs
    N, Nout, B, F = 200_000, 50_000, 2, 32
    gso = graphs.er_gso(N, 8, seed=5)
    pool = gnn_b200.MaxPoolLocal(N, Nout, 1)
    pool.addGSO(gso)
    x = torch.randn(B, F, N, device="cuda", requires_grad=True)
    y = pool(x)
    g = torch.randn_like(y)
    (gx,) = torch.autograd.grad(y, x, g)
    nb = pool.neighborhood.cuda()
    xr = x.detach().clone().requires_grad_(True)
    yr = xr.index_select(2, nb.reshape(-1)).reshape(B, F, Nout, pool.maxNeighborhoodSize).max(dim=3)[0]
    (gr,) = torch.autograd.grad(yr, xr, g)
    assert torch.equal(y, yr)
    assert rel(gx.cpu().numpy(), gr.cpu().numpy()) < 1e-6
