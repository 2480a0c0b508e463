"""Hidden-state recursion on a batch- and time-varying GSO (gnn_b200.delayed: GRNN_DB, HiddenState_DB) against fixtures
produced by the unmodified reference (tests/golden/grnn_db_cases.npz <- oracle/make_golden.py gen_grnn_db;
graphML.py:1096-1290, :3395-3538).

The CUDA path keeps the K-1 delayed copies of the hidden state node-major and advances them with one CSR hop per time step
and edge feature (operator (t, e) of ONE device plan built from the GSO batch).  CPU tests check the operator construction
and the recursion / autograd wiring with torch.sparse standing in for the hop kernel and the dense CPU oracle for the
input-to-hidden filter; GPU tests run the same fixtures through the CUDA kernels."""
import os

import numpy as np
import pytest
import torch

import lsigf_oracle as orc
from host_filters import SparseSlabOps as _SparseSlabOps
from host_filters import dense_from_csr as _dense_from_csr

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "grnn_db_cases.npz"))
TAGS = ["ga", "gb", "gc", "gd", "ge", "gf"]
SIGMA = {0: torch.tanh, 1: torch.relu}


def _rel(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


@pytest.fixture
def cpu_hooks(monkeypatch):
    from gnn_b200 import delayed
    made = []

    def apply(h, S, x_big, b_big):
        csr, M = delayed.block_delay_csr(S)
        return orc.lsigf_dense_torch(h, _dense_from_csr(csr, M, S.dtype), x_big, b_big)

    def slab_ops(S):
        made.append(_SparseSlabOps(S))
        return made[-1]

    monkeypatch.setattr(delayed, "_apply", apply)
    monkeypatch.setattr(delayed, "_slab_ops", slab_ops)
    return made


def _check_case(tag, dtype, device, tol):
    from gnn_b200 import delayed
    B, T, N, F, H, K, E, bias, sg = (int(v) for v in GOLD[tag + "_meta"])
    t = lambda a, g=True: torch.tensor(GOLD[tag + "_" + a], dtype=dtype, device=device).requires_grad_(g)  # noqa: E731
    a, b, x, z0 = t("a"), t("b"), t("x"), t("z0")
    xb, zb = (t("xb"), t("zb")) if bias else (None, None)
    z = delayed.GRNN_DB(a, b, t("S", False), x, z0, SIGMA[sg], xb, zb)
    assert tuple(z.shape) == (B, T, H, N)
    z.backward(t("dz", False))
    got = [("z", z.detach()), ("da", a.grad), ("db", b.grad), ("dx", x.grad), ("dz0", z0.grad)]
    if bias:
        got += [("dxb", xb.grad), ("dzb", zb.grad)]
    for name, val in got:
        assert _rel(val.cpu().numpy(), GOLD[tag + "_" + name]) < tol, (tag, name)
    return B, T, N, F, H, K, E


def _check_layer(dtype, device, tol):
    from gnn_b200 import delayed
    B, T, N, F, H, K, E = (int(v) for v in GOLD["layer_meta"])
    layer = delayed.HiddenState_DB(F, H, K, torch.tanh, E, True)
    assert sorted(layer.state_dict()) == ["aWeights", "bWeights", "xBias", "zBias"]      # the reference's checkpoint keys
    layer = layer.to(device=device, dtype=dtype)               # before loading: fp64 fixtures must not pass through fp32
    layer.load_state_dict({k: torch.tensor(GOLD["layer_p_" + k]) for k in layer.state_dict()})
    layer.addGSO(torch.tensor(GOLD["layer_S"], dtype=dtype, device=device))
    x = torch.tensor(GOLD["layer_x"], dtype=dtype, device=device, requires_grad=True)
    z0 = torch.tensor(GOLD["layer_z0"], dtype=dtype, device=device, requires_grad=True)
    z, zT = layer(x, z0)
    assert tuple(z.shape) == (B, T, H, N) and tuple(zT.shape) == (B, 1, 1, H, N)          # graphML.py:3512-3514
    ((z * torch.tensor(GOLD["layer_dz"], dtype=dtype, device=device)).sum() +
     (zT * torch.tensor(GOLD["layer_dzT"], dtype=dtype, device=device)).sum()).backward()
    assert _rel(z.detach().cpu().numpy(), GOLD["layer_z"]) < tol
    assert _rel(zT.detach().cpu().numpy(), GOLD["layer_zT"]) < tol
    assert _rel(x.grad.cpu().numpy(), GOLD["layer_dx"]) < tol
    assert _rel(z0.grad.cpu().numpy(), GOLD["layer_dz0"]) < tol
    for name, prm in layer.named_parameters():
        assert _rel(prm.grad.cpu().numpy(), GOLD["layer_g_" + name]) < tol, name
    return layer, x, z0


# ------------------------------------------------------------------------------------------------ CPU host logic
def test_slab_operators_layout():
    """Operator o = (t-1)*E + e is the block-diagonal (over b) S[b, t, e] on rows (b, n); `bwd` holds it, `fwd` its
    transpose, both with ascending columns; S[:, 0] is never used (nothing is shifted into t = 0)."""
    from gnn_b200 import delayed
    rng = np.random.default_rng(2)
    B, T, E, N = 3, 4, 2, 5
    S = torch.tensor(rng.standard_normal((B, T, E, N, N)) * (rng.random((B, T, E, N, N)) < 0.4))
    fwd, bwd, R = delayed.slab_csr(S)
    assert R == B * N and len(fwd) == len(bwd) == (T - 1) * E
    for t in range(1, T):
        for e in range(E):
            o = (t - 1) * E + e
            A = torch.block_diag(*[S[b, t, e] for b in range(B)])
            assert torch.equal(_dense_from_csr([bwd[o]], R, S.dtype)[0], A)
            assert torch.equal(_dense_from_csr([fwd[o]], R, S.dtype)[0], A.t())
            for (rowptr, col, val) in (fwd[o], bwd[o]):
                assert rowptr.dtype == torch.int64 and col.dtype == torch.int32 and rowptr[0] == 0 and rowptr[-1] == col.numel()
                for r in range(R):
                    c = col[rowptr[r]:rowptr[r + 1]]
                    assert torch.all(c[1:] > c[:-1])
    assert delayed.slab_csr(S[:, :1]) == ([], [], R)           # a single time step: no operator at all
    empty = torch.zeros(2, 3, 1, 4, 4, dtype=torch.float64)   # no edges anywhere: operators exist and are empty
    f0, b0, _ = delayed.slab_csr(empty)
    assert len(f0) == 2 and all(c.numel() == 0 and int(r[-1]) == 0 for (r, c, v) in f0 + b0)


@pytest.mark.parametrize("tag", TAGS)
def test_recursion_matches_reference_fixtures(tag, cpu_hooks):
    B, T, N, F, H, K, E = _check_case(tag, torch.float64, "cpu", 1e-12)
    # one hop per time step (from t = 1) and edge feature advances all K-1 delays at once; none when K = 1 or T = 1
    want = (T - 1) * E if K > 1 else 0
    assert sum(o.hops for o in cpu_hooks) == want


def test_layer_host_logic(cpu_hooks):
    layer, x, z0 = _check_layer(torch.float64, "cpu", 1e-12)
    with pytest.raises(AssertionError):
        layer.addGSO(torch.zeros(2, 3, 3))                     # the reference's 5-D check (graphML.py:3517)
    with pytest.raises(AssertionError):
        layer(x[:, :2], z0)                                    # T must match the stored GSO (graphML.py:3499)
    with pytest.raises(AssertionError):
        layer(x, z0[:, :1])                                    # hidden features (graphML.py:3505)
    assert "hidden_features=4" in layer.extra_repr() and "GSO stored" in layer.extra_repr()


def test_nonlinearity_sees_the_reference_layout(cpu_hooks):
    """sigma is applied to a [B, H, N] tensor like in the reference (graphML.py:1212), so a nonlinearity that is not
    element-wise (here: a softmax over the node axis) gives the reference's result too."""
    from gnn_b200 import delayed
    rng = np.random.default_rng(5)
    B, T, N, F, H, K, E = 2, 4, 5, 2, 3, 3, 1
    S = torch.tensor(np.stack([np.stack([orc.random_sparse_gso(rng, N, 3, E) for _ in range(T)]) for _ in range(B)]))
    a, b = torch.tensor(rng.uniform(-0.5, 0.5, (H, E, K, F))), torch.tensor(rng.uniform(-0.5, 0.5, (H, E, K, H)))
    x, z0 = torch.tensor(rng.standard_normal((B, T, F, N))), torch.tensor(rng.standard_normal((B, H, N)))
    sigma = lambda v: torch.softmax(v, dim=2)                  # noqa: E731
    z = delayed.GRNN_DB(a, b, S, x, z0, sigma)
    # dense restatement of the recursion, reference layout
    zs, hist = [], [z0]
    for t in range(T):
        acc = 0.0
        for k in range(K):
            if t - k < 0:
                continue
            xs, zz = x[:, t - k], hist[t - k]                  # x_{t-k}, z_{t-1-k}
            for s in range(t - k + 1, t + 1):
                xs, zz = torch.matmul(xs, S[:, s, 0]), torch.matmul(zz, S[:, s, 0])
            acc = acc + torch.einsum("hf,bfn->bhn", a[:, 0, k], xs) + torch.einsum("hg,bgn->bhn", b[:, 0, k], zz)
        zs.append(sigma(acc))
        hist.append(zs[-1])
    assert _rel(z.numpy(), torch.stack(zs, 1).numpy()) < 1e-12


def test_product_path_is_loud_on_cpu():
    from gnn_b200 import delayed
    t = lambda n: torch.tensor(GOLD["ga_" + n])                # noqa: E731
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        delayed.GRNN_DB(t("a"), t("b"), t("S"), t("x"), t("z0"), torch.tanh)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        delayed._SlabOps(t("S"))


def test_install_retargets_the_reference():
    """install() points the reference's GRNN_DB / HiddenState_DB at this package and uninstall() restores them."""
    import types
    import gnn_b200
    from gnn_b200 import delayed
    names = ("LSIGF", "GraphFilter", "EVGF", "EdgeVariantGF", "MaxPoolLocal", "MaxLocalActivation", "MedianLocalActivation",
             "HiddenState", "TimeGatedHiddenState", "NodeGatedHiddenState", "LSIGF_DB", "GraphFilter_DB", "GRNN_DB",
             "HiddenState_DB")
    fake = types.SimpleNamespace(**{n: object() for n in names})
    before = {n: getattr(fake, n) for n in names}
    gnn_b200.install(fake)
    assert fake.GRNN_DB is delayed.GRNN_DB and fake.HiddenState_DB is delayed.HiddenState_DB
    gnn_b200.uninstall(fake)
    assert all(getattr(fake, n) is before[n] for n in names)


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("tag", TAGS)
@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-11), (torch.float32, 1e-4)])
def test_gpu_grnn_db_matches_reference_fixtures(tag, dtype, tol):
    _check_case(tag, dtype, "cuda", tol)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-11), (torch.float32, 1e-4)])
def test_gpu_hiddenstate_db_layer(dtype, tol):
    _check_layer(dtype, "cuda", tol)
