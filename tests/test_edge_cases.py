"""Host-logic properties (CPU, hypothesis) and GPU edge cases of the LSIGF path: empty graphs, single node, isolated
nodes and self-loops, partial gradient requests, non-contiguous inputs, large batches."""
import numpy as np
import pytest
import torch
from hypothesis import given, settings, strategies as st

import lsigf_oracle as orc


def _rel(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


# ------------------------------------------------------------------------------------------------ CPU host logic
@settings(max_examples=60, deadline=None, derandomize=True)
@given(B=st.integers(1, 4), C=st.integers(1, 9), N=st.integers(2, 12), pad=st.integers(0, 5))
def test_node_major_view_detection(B, C, N, pad):
    import gnn_b200
    ld = B * C + pad
    buf = torch.arange(N * ld, dtype=torch.float32).reshape(N, ld)
    view = buf[:, :B * C].view(N, B, C).permute(1, 2, 0)          # what LSIGF returns
    assert gnn_b200.node_major_ld(view) == ld
    # element-wise ops keep the dimension order (node axis slowest): exact strides when the buffer has no padding,
    # compacted rows otherwise — either way the next layer consumes the result without a transpose
    assert gnn_b200.node_major_ld(torch.relu(view)) == (ld if pad == 0 else B * C)
    plain = torch.zeros(B, C, N)
    if B * C > 1:
        assert gnn_b200.node_major_ld(plain) is None               # the reference's [B, C, N] layout needs a transpose
    assert gnn_b200.padded_ld(B * C, torch.float32) % 8 == 0 and gnn_b200.padded_ld(B * C, torch.float64) % 4 == 0


@settings(max_examples=30, deadline=None, derandomize=True)
@given(N=st.integers(1, 25), E=st.integers(1, 3), seed=st.integers(0, 10 ** 6))
def test_dense_csr_roundtrip(N, E, seed):
    import scipy.sparse as sp
    import gnn_b200
    from gnn_b200.gso import dense_to_csr
    rng = np.random.default_rng(seed)
    S = rng.standard_normal((E, N, N)) * (rng.random((E, N, N)) < 0.3)
    g = gnn_b200.SparseGSO.from_dense(torch.tensor(S))
    assert g.shape == (E, N, N) and g.nnz() == int((S != 0).sum())
    assert np.array_equal(g.to_dense().numpy(), S)
    for e in range(E):
        r, c, v = dense_to_csr(torch.tensor(S[e]))
        m = sp.csr_matrix(S[e])
        m.sort_indices()
        assert np.array_equal(r.numpy(), m.indptr) and np.array_equal(c.numpy(), m.indices)
        assert np.array_equal(v.numpy(), m.data)


@pytest.mark.filterwarnings("ignore:Sparse")
def test_torch_sparse_gso_inputs():
    """The GSO may arrive as a torch sparse tensor (SURVEY.md §8b extension): [E, N, N] COO or batched CSR, or a list of
    2-D COO / CSR / CSC tensors — same host CSR as the dense route, duplicates summed, never densified."""
    import gnn_b200
    rng = np.random.default_rng(0)
    E, N = 2, 9
    pattern = rng.random((N, N)) < 0.3
    D = torch.tensor(rng.standard_normal((E, N, N)) * pattern)           # same pattern for every e: batched CSR exists
    ref = gnn_b200.SparseGSO.from_dense(D)

    def same(g):
        return g.shape == ref.shape and g.dtype == ref.dtype and \
            all(np.array_equal(a, b) for x, y in zip(g.csr, ref.csr) for a, b in zip(x, y))

    assert same(gnn_b200.SparseGSO.from_torch_sparse(D.to_sparse()))
    assert same(gnn_b200.SparseGSO.from_torch_sparse(D.to_sparse_csr()))
    assert same(gnn_b200.SparseGSO.from_torch_sparse([D[e].to_sparse_csr() for e in range(E)]))
    assert same(gnn_b200.SparseGSO.from_torch_sparse([D[e].to_sparse_csc() for e in range(E)]))
    dup = torch.sparse_coo_tensor(torch.tensor([[0, 0, 2], [1, 1, 0]]), torch.tensor([1.0, 2.0, 5.0]), (3, 3))
    assert torch.equal(gnn_b200.SparseGSO.from_torch_sparse([dup]).to_dense()[0],
                       torch.tensor([[0.0, 3.0, 0.0], [0.0, 0.0, 0.0], [5.0, 0.0, 0.0]]))
    f32 = gnn_b200.SparseGSO.from_torch_sparse(D.to_sparse(), dtype=torch.float32)
    assert f32.dtype == torch.float32 and np.array_equal(f32.csr[0][2], ref.csr[0][2].astype(np.float32))


@settings(max_examples=30, deadline=None, derandomize=True)
@given(N=st.integers(1, 30), P=st.integers(1, 5), seed=st.integers(0, 10 ** 6))
def test_row_partition_covers_everything(N, P, seed):
    """The equal row blocks of the node-sharded path tile [0, P*R) exactly; slices of CSR rows re-assemble the matrix."""
    import scipy.sparse as sp
    from gnn_b200.distributed import row_slice, transpose_csr
    m = sp.random(N, N, density=0.3, format="csr", random_state=np.random.RandomState(seed % 2 ** 31))
    m.sort_indices()
    csr = (m.indptr.astype(np.int64), m.indices.astype(np.int32), m.data)
    R = (N + P - 1) // P
    rows = []
    for p in range(P):
        rp, c, v = row_slice(csr, p * R, (p + 1) * R)
        assert len(rp) == R + 1 and rp[0] == 0 and rp[-1] == len(c) == len(v)
        rows.append(sp.csr_matrix((v, c, rp), shape=(R, N)))
    full = sp.vstack(rows)[:N]
    assert (abs(full - m)).sum() == 0
    tr = transpose_csr(csr, N)
    assert (abs(sp.csr_matrix((tr[2], tr[1], tr[0]), shape=(N, N)) - m.T)).sum() == 0


# ------------------------------------------------------------------------------------------------ GPU edge cases
@pytest.mark.gpu
@pytest.mark.parametrize("dtype,tol", [(torch.float32, 1e-5), (torch.float64, 1e-12)])
def test_empty_graph_and_single_node(dtype, tol):
    import gnn_b200
    # no edges at all: only the k = 0 taps act (x S^k = 0 for k >= 1)
    F, E, K, G, N, B = 3, 2, 4, 5, 37, 2
    rng = np.random.default_rng(1)
    h, x, b = rng.standard_normal((F, E, K, G)), rng.standard_normal((B, G, N)), rng.standard_normal((F, 1))
    S = np.zeros((E, N, N))
    t = lambda a: torch.tensor(a, dtype=dtype, device="cuda")  # noqa: E731
    y = gnn_b200.LSIGF(t(h), t(S), t(x), t(b))
    rnd = lambda a: torch.tensor(a, dtype=dtype).double().numpy()  # noqa: E731
    assert _rel(y.cpu().numpy(), np.einsum("feg,bgn->bfn", rnd(h)[:, :, 0, :], rnd(x)) + rnd(b)[None]) < tol
    # one node with a self-loop
    S1 = np.full((1, 1, 1), 0.5)
    h1, x1 = rng.standard_normal((2, 1, 3, 2)), rng.standard_normal((3, 2, 1))
    y1 = gnn_b200.LSIGF(t(h1), t(S1), t(x1), None)
    assert _rel(y1.cpu().numpy(), orc.lsigf_dense(rnd(h1), rnd(S1), rnd(x1), None)) < tol


@pytest.mark.gpu
def test_isolated_nodes_self_loops_and_partial_grads():
    import gnn_b200
    dtype = torch.float64
    c = orc.random_case(9, N=60, B=2, G=4, F=3, K=4, E=1, avg_deg=3, bias="F1")
    S = c["S"].copy()
    S[0, 5, :] = 0; S[0, :, 5] = 0            # isolated node
    S[0, 7, 7] = 0.25                         # self-loop
    t = lambda a, g=False: torch.tensor(a, dtype=dtype, device="cuda").requires_grad_(g)  # noqa: E731
    # only the taps ask for a gradient; no bias
    h = t(c["h"], True)
    x = t(c["x"])
    y = gnn_b200.LSIGF(h, t(S), x, None)
    y.backward(t(c["dy"]))
    assert x.grad is None
    dh, dx, _ = orc.lsigf_grads_dense(c["h"], S, c["x"], c["dy"])
    assert _rel(y.detach().cpu().numpy(), orc.lsigf_dense(c["h"], S, c["x"], None)) < 1e-12
    assert _rel(h.grad.cpu().numpy(), dh) < 1e-12
    # only the input asks for a gradient
    x2 = t(c["x"], True)
    gnn_b200.LSIGF(t(c["h"]), t(S), x2, t(c["b"])).backward(t(c["dy"]))
    assert _rel(x2.grad.cpu().numpy(), dx) < 1e-12 and x2.grad.is_contiguous()


@pytest.mark.gpu
def test_non_contiguous_input_and_large_batch():
    import gnn_b200
    c = orc.random_case(12, N=90, B=64, G=3, F=5, K=3, E=2, avg_deg=4, bias="FN")
    t = lambda a: torch.tensor(a, dtype=torch.float32, device="cuda")  # noqa: E731
    xw = torch.zeros(64, 3, 180, device="cuda")
    xw[:, :, ::2] = t(c["x"])
    x_strided = xw[:, :, ::2]                                  # neither contiguous nor node-major
    y = gnn_b200.LSIGF(t(c["h"]), t(c["S"]), x_strided, t(c["b"]))
    rnd = lambda a: torch.tensor(a, dtype=torch.float32).double().numpy()  # noqa: E731
    assert _rel(y.cpu().numpy(), orc.lsigf_dense(rnd(c["h"]), rnd(c["S"]), rnd(c["x"]), rnd(c["b"]))) < 1e-4
    yc = gnn_b200.to_feature_major(y)
    assert yc.is_contiguous() and torch.equal(yc, y)


@pytest.mark.gpu
def test_plan_cache_follows_in_place_gso_updates():
    """GraphFilter keeps the dense S by reference (graphML.py:2123); changing it in place must invalidate the plan."""
    import gnn_b200
    torch.manual_seed(0)
    N = 40
    S = (torch.rand(1, N, N, device="cuda") < 0.1).float() * 0.2
    layer = gnn_b200.GraphFilter(2, 3, 3).cuda()
    layer.addGSO(S)
    x = torch.randn(2, 2, N, device="cuda")
    y0 = layer(x).clone()
    S.mul_(0.5)                                                # same storage, new version counter
    y1 = layer(x)
    ref = orc.lsigf_dense(layer.weight.detach().cpu().double().numpy(), S.cpu().double().numpy(),
                          x.cpu().double().numpy(), layer.bias.detach().cpu().double().numpy())
    assert _rel(y1.detach().cpu().numpy(), ref) < 1e-5
    assert not torch.allclose(y0, y1)


@pytest.mark.gpu
def test_host_taps_or_bias_are_rejected():
    """The kernels read h and b on the device: host tensors must raise before any launch, not reach a kernel as host
    pointers.  A node-gated layer moved to the GPU before addGSO builds its gate filters on the GPU as well."""
    import gnn_b200
    from gnn_b200 import recurrent as rec
    c = orc.random_case(13, N=30, B=2, G=3, F=4, K=3, E=1, avg_deg=4, bias="F1")
    gpu = lambda a: torch.tensor(a, dtype=torch.float32, device="cuda")  # noqa: E731
    cpu = lambda a: torch.tensor(a, dtype=torch.float32)  # noqa: E731
    with pytest.raises(RuntimeError, match="on one device"):
        gnn_b200.LSIGF(cpu(c["h"]), gpu(c["S"]), gpu(c["x"]), gpu(c["b"]))
    with pytest.raises(RuntimeError, match="on one device"):
        gnn_b200.LSIGF(gpu(c["h"]), gpu(c["S"]), gpu(c["x"]), cpu(c["b"]))
    layer = rec.NodeGatedHiddenState(2, 4, 3).cuda()
    layer.addGSO(gpu(c["S"]))
    assert all(p.is_cuda for p in layer.parameters())
    z, _ = layer(torch.randn(2, 3, 2, 30, device="cuda"), torch.randn(2, 4, 30, device="cuda"))
    torch.cuda.synchronize()
    assert z.shape == (2, 3, 4, 30) and bool(torch.isfinite(z).all())
