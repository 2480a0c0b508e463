"""Edge-gated graph recurrent layer (gnn_b200.edgegated, csrc/egate.cu) against fixtures produced by the unmodified
reference (tests/golden/grnn_edge_cases.npz <- oracle/make_golden_edge.py: EdgeGatedHiddenState,
alegnn/utils/graphML.py:4033-4209, GatedGRNN's edge path :1410-1451 / :1474-1514, learnAttentionGSO :640-737).

CPU tests check the host logic (pattern, gate layouts, recursion, autograd wiring) with torch restatements standing in
for the two kernels (`_attention`, `_gated_hop`) and the dense CPU oracle for the gate GRNNs' filter; GPU tests run
the real kernels against the fixtures, against the fp64 restatement in oracle/egate_oracle.py, at scale, and on one-,
two- and three-node graphs.  Each launch branch of egate.cu's kernels has a componentwise-bounded row in
tests/test_egate_dispatch.py."""
import os

import numpy as np
import pytest
import torch

import egate_oracle as ego
import lsigf_oracle as orc

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "grnn_edge_cases.npz"))
TAGS = ["base", "nobias", "k1", "kgt", "relu", "diag", "neg"]
SIGMA = {0: torch.tanh, 1: torch.relu}


def _rel(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def _meta(tag):
    seed, N, B, T, F, H, K, bias, sg = (int(v) for v in GOLD[tag + "_meta"])
    return seed, N, B, T, F, H, K, bool(bias), SIGMA[sg]


def _fixture_params(tag):
    return {k[len(tag) + 3:]: torch.tensor(GOLD[k]) for k in GOLD.files if k.startswith(tag + "_p_")}


def _layer_for(tag, dtype, device, S=None):
    import gnn_b200
    seed, N, B, T, F, H, K, bias, sigma = _meta(tag)
    layer = gnn_b200.EdgeGatedHiddenState(F, H, K, sigma, 1, bias)
    layer.addGSO(torch.tensor(GOLD[tag + "_S"], dtype=dtype, device=device) if S is None else S)
    sd = _fixture_params(tag)
    assert list(sd) == list(layer.state_dict())              # the reference's names, in the reference's order
    layer.load_state_dict(sd)
    return layer.to(device=device, dtype=dtype)


def _run_and_compare(tag, dtype, device, tol, S=None):
    seed, N, B, T, F, H, K, bias, sigma = _meta(tag)
    layer = _layer_for(tag, dtype, device, S)
    x = torch.tensor(GOLD[tag + "_x"], dtype=dtype, device=device, requires_grad=True)
    z0 = torch.tensor(GOLD[tag + "_z0"], dtype=dtype, device=device, requires_grad=True)
    z, zT = layer(x, z0)
    assert tuple(z.shape) == (B, T, H, N) and tuple(zT.shape) == (B, 1, 1, H, N)
    z.backward(torch.tensor(GOLD[tag + "_dz"], dtype=dtype, device=device))
    assert _rel(z.detach().cpu().numpy(), GOLD[tag + "_z"]) < tol
    assert _rel(zT.detach().cpu().numpy(), GOLD[tag + "_zT"]) < tol
    assert _rel(x.grad.cpu().numpy(), GOLD[tag + "_dx"]) < tol
    assert _rel(z0.grad.cpu().numpy(), GOLD[tag + "_dz0"]) < tol
    names = [n for n, _ in layer.named_parameters()]
    assert len(names) == (16 if bias else 10)
    for name, p in layer.named_parameters():
        ref = GOLD["%s_g_%s" % (tag, name)]
        got = np.zeros(ref.shape) if p.grad is None else p.grad.cpu().numpy()
        if not np.any(ref):                                   # K = 1: the gates reach nothing
            assert not np.any(got), name
        else:
            assert _rel(got, ref) < tol, name
    return layer


# ------------------------------------------------------------------------------------ torch restatements of the kernels
def _attention_torch(s, mixer, pat):
    """s [N, Bs] -> alpha [nnz, Bs], through the fp64 restatement's per-non-zero index arithmetic."""
    return ego.egate_attention_coo(s.t(), mixer, pat.m_row, pat.m_col.long(), pat.N).t()


def _gated_hop_torch(u, gate, pat):
    """u [N, Bs, C], gate [Bs, nnz] -> u S~ per sample, over the pattern's CSR of S^T and its mask positions."""
    j = torch.repeat_interleave(torch.arange(pat.N, device=u.device), pat.t_rowptr.diff())
    i = pat.t_col.long()
    pos = pat.t_pos.long()
    w = torch.where(pos >= 0, gate[:, pos.clamp(min=0)] * pat.t_val.to(u.dtype), torch.zeros((), dtype=u.dtype))
    return ego.egate_hop_coo(u.permute(1, 2, 0), w, i, j).permute(2, 0, 1)


@pytest.fixture
def torch_kernels(monkeypatch):
    import gnn_b200
    from gnn_b200 import edgegated as eg
    from gnn_b200 import recurrent as rec
    monkeypatch.setattr(eg, "_attention", _attention_torch)
    monkeypatch.setattr(eg, "_gated_hop", _gated_hop_torch)

    def lsigf(h, S, x, b=None):
        if isinstance(S, gnn_b200.SparseGSO):                 # the gate GRNNs' filter: dense oracle on small N
            rowptr, col, val = S.csr[0]
            D = torch.zeros(1, S.N, S.N, dtype=x.dtype)
            D[0, torch.from_numpy(np.repeat(np.arange(S.N), np.diff(rowptr))), torch.from_numpy(col.astype(np.int64))] = \
                torch.from_numpy(val).to(x.dtype)
            S = D
        return orc.lsigf_dense_torch(h, S, x, b)
    monkeypatch.setattr(rec, "_lsigf", lsigf)
    monkeypatch.setattr(gnn_b200.graphML, "LSIGF", lsigf)


# ------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("tag", TAGS)
def test_host_logic_matches_reference_fixtures(tag, torch_kernels):
    _run_and_compare(tag, torch.float64, "cpu", 1e-11)


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_matches_reference_fixtures(tag):
    """The fp64 restatement the at-scale GPU test trusts (egate_oracle.edge_gated_hidden_state_coo) equals the reference."""
    seed, N, B, T, F, H, K, bias, sigma = _meta(tag)
    S = GOLD[tag + "_S"][0]
    rows, cols = np.nonzero(S)
    p = {k: v.clone().requires_grad_(True) for k, v in _fixture_params(tag).items()}
    x = torch.tensor(GOLD[tag + "_x"], requires_grad=True)
    z0 = torch.tensor(GOLD[tag + "_z0"], requires_grad=True)
    z, qHat, qCheck, _ = ego.edge_gated_hidden_state_coo(p, N, rows, cols, S[rows, cols], x, z0, sigma)
    z.backward(torch.tensor(GOLD[tag + "_dz"]))
    assert _rel(z.detach().numpy(), GOLD[tag + "_z"]) < 1e-11
    assert _rel(x.grad.numpy(), GOLD[tag + "_dx"]) < 1e-11
    assert _rel(z0.grad.numpy(), GOLD[tag + "_dz0"]) < 1e-11
    for name, t in p.items():
        ref = GOLD["%s_g_%s" % (tag, name)]
        got = np.zeros(ref.shape) if t.grad is None else t.grad.numpy()
        assert (not np.any(got)) if not np.any(ref) else _rel(got, ref) < 1e-11, name


def test_sparse_attention_reproduces_the_reference_dense_gates():
    """alpha on the mask equals the reference's dense learnAttentionGSO (graphML.py:640-737); off the mask it is 0."""
    tag = "base"
    seed, N, B, T, F, H, K, bias, sigma = _meta(tag)
    S = GOLD[tag + "_S"][0]
    rows, cols = np.nonzero(S)
    p = _fixture_params(tag)
    with torch.no_grad():
        _, qHat, qCheck, (mr, mc) = ego.edge_gated_hidden_state_coo(p, N, rows, cols, S[rows, cols],
                                                                    torch.tensor(GOLD[tag + "_x"]),
                                                                    torch.tensor(GOLD[tag + "_z0"]), sigma)
    for name, q in (("qHat", qHat), ("qCheck", qCheck)):
        dense = np.zeros((B, T, N, N))
        dense[:, :, mr, mc] = q.numpy()
        ref = GOLD[tag + "_" + name][:, :, 0]
        assert np.abs(dense - ref).max() < 1e-13
        off = np.ones((N, N), bool)
        off[mr, mc] = False
        assert not np.any(ref[:, :, off])                     # the reference's gates vanish off the mask too
    # the mask is |S + I| > 1e-9 (graphML.py:692) and each gate row sums to 1 over it
    assert sorted(zip(mr, mc)) == sorted(zip(*np.nonzero(np.abs(S + np.eye(N)) > 1e-9)))
    np.testing.assert_allclose(GOLD[tag + "_qHat"].sum(-1), 1.0, rtol=0, atol=1e-13)


def _pattern_dense(pat):
    N = pat.N
    M = np.zeros((N, N), bool)
    M[pat.m_row.numpy(), pat.m_col.numpy()] = True
    return M


def test_pattern_edge_cases():
    """S_ii = -1 (diagonal outside the mask), a node whose only entry is S_ii = -1 (empty mask row), a node without
    entries (mask row = the diagonal alone), explicit S entries below the tolerance, and SparseGSO input."""
    import gnn_b200
    from gnn_b200 import edgegated as eg
    N = 7
    S = np.zeros((N, N))
    S[0, 1], S[0, 3], S[1, 0], S[3, 5], S[5, 3], S[6, 6] = 0.5, -0.25, 0.75, 0.125, 2.0, 0.3
    S[2, 2] = -1.0                       # only entry of row 2, diagonal drops out: empty mask row
    S[3, 3] = -1.0                       # diagonal outside the mask, row keeps (3, 5)
    S[5, 0] = 1e-12                      # an S entry below the tolerance: outside the mask
    pat = eg.EdgeGatePattern(torch.tensor(S).reshape(1, N, N))
    mask = np.abs(S + np.eye(N)) > 1e-9
    assert (_pattern_dense(pat) == mask).all()
    assert pat.nnz == mask.sum()
    m_rowptr = pat.m_rowptr.numpy()
    assert m_rowptr[3] - m_rowptr[2] == 0                     # row 2: empty
    assert list(pat.m_col.numpy()[m_rowptr[4]:m_rowptr[5]]) == [4]   # row 4 (no entries): the diagonal alone
    # positions: every S entry points at its own mask slot or at -1
    mr, mc = pat.m_row.numpy(), pat.m_col.numpy()
    j = np.repeat(np.arange(N), np.diff(pat.t_rowptr.numpy()))
    i = pat.t_col.numpy()
    for ii, jj, p, v in zip(i, j, pat.t_pos.numpy(), pat.t_val.numpy()):
        assert v == S[ii, jj]
        if mask[ii, jj]:
            assert (mr[p], mc[p]) == (ii, jj)
        else:
            assert p == -1
    assert sorted(zip(i, j)) == sorted(zip(*np.nonzero(S)))
    i2 = np.repeat(np.arange(N), np.diff(pat.s_rowptr.numpy()))
    assert sorted(zip(i2, pat.s_col.numpy(), pat.s_pos.numpy())) == sorted(zip(i, j, pat.t_pos.numpy()))
    np.testing.assert_array_equal(pat.m_sval.numpy(), S[mr, mc])
    # the transposed mask lists column j's entries
    jT = np.repeat(np.arange(N), np.diff(pat.mT_rowptr.numpy()))
    assert (mc[pat.mT_perm.numpy()] == jT).all()
    # SparseGSO: built from the CSR, never densified, same pattern
    spat = eg.EdgeGatePattern(gnn_b200.SparseGSO.from_dense(torch.tensor(S).reshape(1, N, N)))
    for name in eg.EdgeGatePattern._TENSORS:
        assert torch.equal(getattr(spat, name), getattr(pat, name)), name


def test_sparse_gso_layer_matches_fixture(torch_kernels):
    import gnn_b200
    S = gnn_b200.SparseGSO.from_dense(torch.tensor(GOLD["neg_S"]))
    _run_and_compare("neg", torch.float64, "cpu", 1e-11, S=S)


def test_state_dict_keys_and_seeded_parameters_match_the_reference():
    """Same keys in the same order, and a seeded build (construction, then addGSO, then .double(), as the fixture
    generator does) reproduces the reference's parameters bit for bit: same RNG consumption order."""
    import gnn_b200
    for tag in TAGS:
        seed, N, B, T, F, H, K, bias, sigma = _meta(tag)
        torch.manual_seed(seed)
        layer = gnn_b200.EdgeGatedHiddenState(F, H, K, sigma, 1, bias)
        layer.addGSO(torch.tensor(GOLD[tag + "_S"]))
        layer.double()
        sd = layer.state_dict()
        ref = _fixture_params(tag)
        assert list(sd) == list(ref)
        for k in ref:
            assert torch.equal(sd[k], ref[k]), (tag, k)
    assert tuple(layer.inputGateGAT.mixer.shape) == (1, 1, 2) and tuple(layer.inputGateGAT.weight.shape) == (1, 1, 1, H)


def test_addgso_creates_fresh_gate_attentions():
    import gnn_b200
    layer = gnn_b200.EdgeGatedHiddenState(1, 3, 2)
    S = torch.tensor(GOLD["base_S"], dtype=torch.float32)
    layer.addGSO(S)
    first = layer.inputGateGAT
    layer.addGSO(S)
    assert layer.inputGateGAT is not first                    # graphML.py:4190-4191
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        layer(torch.zeros(1, 2, 1, S.shape[1]), torch.zeros(1, 3, S.shape[1]))


def test_install_edge_gating_is_opt_in():
    import types
    import gnn_b200
    names = ("LSIGF", "GraphFilter", "EVGF", "EdgeVariantGF", "MaxPoolLocal", "MaxLocalActivation",
             "MedianLocalActivation", "HiddenState", "TimeGatedHiddenState", "NodeGatedHiddenState", "LSIGF_DB",
             "GraphFilter_DB", "GRNN_DB", "HiddenState_DB", "GatedGRNN", "EdgeGatedHiddenState")
    gml = types.ModuleType("graphML_standin")
    for n in names:
        setattr(gml, n, type(n, (), {}))
    orig = {n: getattr(gml, n) for n in names}
    try:
        gnn_b200.install(gml)
        assert gml.EdgeGatedHiddenState is orig["EdgeGatedHiddenState"] and gml.GatedGRNN is orig["GatedGRNN"]
        gnn_b200.install(gml, edge_gating=True)
        assert gml.EdgeGatedHiddenState is gnn_b200.EdgeGatedHiddenState
        assert gml.GatedGRNN is orig["GatedGRNN"]
    finally:
        gnn_b200.uninstall(gml)
    assert {n: getattr(gml, n) for n in names} == orig
    try:
        gnn_b200.install(gml, edge_gating=True)
        assert gml.EdgeGatedHiddenState is gnn_b200.EdgeGatedHiddenState
    finally:
        gnn_b200.uninstall(gml)
    assert {n: getattr(gml, n) for n in names} == orig


def test_gated_grnn_points_edge_gates_to_the_new_entry_point():
    from gnn_b200 import recurrent as rec
    B, T, N, H = 2, 3, 5, 2
    q = torch.ones(B, T, 1, N, N)
    with pytest.raises(NotImplementedError, match="edge gating.*EdgeGatedGRNN"):
        rec.GatedGRNN(torch.ones(H, 1, 2, 1), torch.ones(H, 1, 2, H), torch.eye(N).reshape(1, N, N),
                      torch.ones(B, T, 1, N), torch.ones(B, H, N), torch.tanh, q, q)


# ------------------------------------------------------------------------------------------------------------ GPU
def _random_graph(rng, N, neg_diag=True):
    """Varied degrees: empty rows, degree-1 rows, a hub row and a hub column, S_ii = -1 nodes, explicit diagonals."""
    deg = rng.integers(0, 9, N)
    deg[::11] = 0
    deg[1] = min(N, 300)
    rows = np.repeat(np.arange(N), deg)
    cols = np.concatenate([rng.choice(N, d, replace=False) for d in deg])
    hub = rng.choice(N, min(N, 200), replace=False)
    rows, cols = np.concatenate((rows, hub)), np.concatenate((cols, np.full(hub.size, 3)))
    key = np.unique(rows * N + cols)
    rows, cols = key // N, key % N
    vals = rng.standard_normal(rows.size) / 4
    if neg_diag:
        vals[(rows == cols) & (rows % 5 == 0)] = -1.0
    return rows, cols, vals


def _pattern_from_coo(N, rows, cols, vals, device):
    import gnn_b200
    import scipy.sparse as sp
    m = sp.csr_matrix((vals, (rows, cols)), shape=(N, N))
    m.sort_indices()
    return gnn_b200.EdgeGatePattern(gnn_b200.SparseGSO([(m.indptr, m.indices, m.data)], N)).on(device)


def _tol(dtype):
    return 1e-12 if dtype == torch.float64 else 2e-5


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("Bs", [1, 6, 13])
def test_attention_kernels_vs_fp64_restatement(dtype, Bs):
    from gnn_b200 import edgegated as eg
    rng = np.random.default_rng(1000 + Bs)
    N = 700
    rows, cols, vals = _random_graph(rng, N)
    pat = _pattern_from_coo(N, rows, cols, vals, "cuda")
    s = torch.tensor(rng.standard_normal((N, Bs)) * 2, device="cuda", requires_grad=True)
    mixer = torch.tensor([0.7, -1.3], dtype=torch.float64, device="cuda", requires_grad=True)
    da = torch.tensor(rng.standard_normal((pat.nnz, Bs)), device="cuda")
    ref = _attention_torch(s, mixer, pat)
    gs, gm = torch.autograd.grad((ref * da).sum(), (s, mixer))
    s2 = s.detach().to(dtype).requires_grad_(True)
    m2 = mixer.detach().to(dtype).requires_grad_(True)
    out = eg._run_attention(s2, m2, pat)
    gs2, gm2 = torch.autograd.grad((out * da.to(dtype)).sum(), (s2, m2))
    for got, want in ((out, ref), (gs2, gs), (gm2, gm)):
        assert _rel(got.detach().double().cpu().numpy(), want.detach().cpu().numpy()) < _tol(dtype) * 10
    # rows sum to one wherever the mask row is not empty; the run is deterministic
    nonempty = pat.m_rowptr.diff() > 0
    rs = torch.zeros(N, Bs, dtype=dtype, device="cuda").index_add(0, pat.m_row, out.detach())
    assert torch.allclose(rs[nonempty], torch.ones_like(rs[nonempty]), atol=10 * _tol(dtype))
    out2 = eg._run_attention(s2, m2, pat)
    gs3, gm3 = torch.autograd.grad((out2 * da.to(dtype)).sum(), (s2, m2))
    assert torch.equal(out, out2) and torch.equal(gs2, gs3) and torch.equal(gm2, gm3)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("Bs,C", [(1, 1), (7, 1), (5, 3), (6, 4), (3, 12), (10, 2), (9, 8)])
def test_gated_hop_kernels_vs_fp64_restatement(dtype, Bs, C):
    """Both lane mappings (16-byte vectors when C is a multiple of 4 floats / 2 doubles, scalar otherwise) and a gate
    read through a strided view (sample stride != 1), as the hidden filter reads one time slab."""
    from gnn_b200 import edgegated as eg
    rng = np.random.default_rng(2000 + 10 * Bs + C)
    N = 900
    rows, cols, vals = _random_graph(rng, N)
    pat = _pattern_from_coo(N, rows, cols, vals, "cuda")
    T = 3
    store = torch.tensor(rng.uniform(0.1, 1.0, (pat.nnz, T, Bs)), device="cuda")       # [nnz, T, Bs] like q_check
    u = torch.tensor(rng.standard_normal((N, Bs, C)), device="cuda", requires_grad=True)
    dd = torch.tensor(rng.standard_normal((N, Bs, C)), device="cuda")
    for gate_full in (store.permute(2, 1, 0), store.permute(1, 2, 0)):            # sample stride 1 and T*Bs*..
        g = gate_full[:, 1] if gate_full.shape[0] == Bs else gate_full[1]
        g = g.detach().requires_grad_(True)
        ref = _gated_hop_torch(u, g, pat)
        gu, gg = torch.autograd.grad((ref * dd).sum(), (u, g))
        u2 = u.detach().to(dtype).requires_grad_(True)
        base = gate_full.detach().to(dtype)
        g2 = (base[:, 1] if base.shape[0] == Bs else base[1]).requires_grad_(True)
        out = eg._run_gated_hop(u2, g2, pat)
        gu2, gg2 = torch.autograd.grad((out * dd.to(dtype)).sum(), (u2, g2))
        for got, want in ((out, ref), (gu2, gu), (gg2, gg)):
            assert _rel(got.detach().double().cpu().numpy(), want.detach().cpu().numpy()) < _tol(dtype)
        # entries outside the mask carry a zero gradient, bitwise-repeatable backward
        out2 = eg._run_gated_hop(u2, g2, pat)
        gu3, gg3 = torch.autograd.grad((out2 * dd.to(dtype)).sum(), (u2, g2))
        assert torch.equal(out, out2) and torch.equal(gu2, gu3) and torch.equal(gg2, gg3)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-10), (torch.float32, 1e-4)])
@pytest.mark.parametrize("tag", TAGS)
def test_fixtures_on_gpu(tag, dtype, tol):
    _run_and_compare(tag, dtype, "cuda", tol)


@pytest.mark.gpu
def test_sparse_gso_fixture_on_gpu():
    import gnn_b200
    _run_and_compare("diag", torch.float64, "cuda", 1e-10, S=gnn_b200.SparseGSO.from_dense(torch.tensor(GOLD["diag_S"])))


def _scale_problem(N=50_000, deg=16, B=8, T=4, F=1, H=12, K=5, seed=77):
    import gnn_b200
    import scipy.sparse as sp
    rng = np.random.default_rng(seed)
    nnz = N * deg
    rows = rng.integers(0, N, nnz)
    cols = rng.integers(0, N, nnz)
    m = sp.csr_matrix((rng.standard_normal(nnz), (rows, cols)), shape=(N, N))
    m.sum_duplicates()
    m = sp.diags(1.0 / np.maximum(np.abs(m).sum(axis=1).A.ravel(), 1.0)) @ m          # spectral radius <= 1
    m = sp.csr_matrix(m, dtype=np.float32)                  # the fp32 layer's GSO; the oracle reads the same values
    m.sort_indices()
    S = gnn_b200.SparseGSO([(m.indptr, m.indices, m.data)], N)
    torch.manual_seed(seed)
    layer = gnn_b200.EdgeGatedHiddenState(F, H, K)
    layer.addGSO(S)
    with torch.no_grad():                              # larger weights so that the gates are far from uniform
        for gat in (layer.inputGateGAT, layer.forgetGateGAT):
            gat.weight.mul_(4.0)
            gat.mixer.mul_(4.0)
    x = rng.standard_normal((B, T, F, N))
    z0 = rng.standard_normal((B, H, N))
    dz = rng.standard_normal((B, T, H, N))
    coo = m.tocoo()
    return layer, S, x, z0, dz, (coo.row, coo.col, coo.data.astype(np.float64))


@pytest.mark.gpu
def test_at_scale_vs_fp64_oracle():
    """N = 50 000, average degree 16, B = 8, T = 4, F = 1, H = 12, K = 5: the fp32 layer against the fp64 restatement
    (forward and the gradients of every input and parameter)."""
    layer, S, x, z0, dz, (rows, cols, vals) = _scale_problem()
    N = S.shape[1]
    layer = layer.cuda()
    xt = torch.tensor(x, dtype=torch.float32, device="cuda", requires_grad=True)
    zt = torch.tensor(z0, dtype=torch.float32, device="cuda", requires_grad=True)
    z, _ = layer(xt, zt)
    z.backward(torch.tensor(dz, dtype=torch.float32, device="cuda"))
    p = {k: v.detach().double().requires_grad_(True) for k, v in layer.state_dict().items()}
    x64 = torch.tensor(x, device="cuda", requires_grad=True)
    z64 = torch.tensor(z0, device="cuda", requires_grad=True)
    zr, _, _, _ = ego.edge_gated_hidden_state_coo(p, N, rows, cols, vals, x64, z64, torch.tanh)
    zr.backward(torch.tensor(dz, device="cuda"))
    assert _rel(z.detach().cpu().numpy(), zr.detach().cpu().numpy()) < 1e-4
    assert _rel(xt.grad.cpu().numpy(), x64.grad.cpu().numpy()) < 1e-4
    assert _rel(zt.grad.cpu().numpy(), z64.grad.cpu().numpy()) < 1e-4
    for name, prm in layer.named_parameters():
        assert _rel(prm.grad.cpu().numpy(), p[name].grad.cpu().numpy()) < 1e-4, name


@pytest.mark.gpu
def test_backward_is_bitwise_reproducible_and_graphed_forward_is_bit_identical():
    import gnn_b200
    layer, S, x, z0, dz, _ = _scale_problem(N=20_000, B=5, T=3)
    layer = layer.cuda()
    grads = []
    for _ in range(2):
        layer.zero_grad(set_to_none=True)
        xt = torch.tensor(x, dtype=torch.float32, device="cuda", requires_grad=True)
        zt = torch.tensor(z0, dtype=torch.float32, device="cuda", requires_grad=True)
        z, _ = layer(xt, zt)
        z.backward(torch.tensor(dz, dtype=torch.float32, device="cuda"))
        grads.append([xt.grad.clone(), zt.grad.clone()] + [p.grad.clone() for p in layer.parameters()])
    assert all(torch.equal(a, b) for a, b in zip(*grads))
    xt = torch.tensor(x, dtype=torch.float32, device="cuda")
    zt = torch.tensor(z0, dtype=torch.float32, device="cuda")
    with torch.no_grad():
        eager = layer(xt, zt)[0].clone()
        fn = gnn_b200.graphed(lambda a, b: layer(a, b)[0], xt, zt)
        replay = fn(xt, zt).clone()
    assert torch.equal(eager, replay)


# one-, two- and three-node graphs: S = [[-1]] has an empty mask (every gate is empty, every S entry is gated off)
TINY_S = {
    "N1": [[0.5]],
    "N1-empty-mask": [[-1.0]],
    "N2": [[0.0, 0.5], [-0.25, 0.0]],
    "N3": [[0.3, 0.0, -0.5], [0.0, -1.0, 0.25], [0.75, 0.0, 0.0]],
}


@pytest.mark.gpu
@pytest.mark.parametrize("tag", list(TINY_S))
def test_tiny_graph_layer_vs_fp64_oracle(tag):
    """K = 3, B = 2, H = 3 in fp64 against egate_oracle.edge_gated_hidden_state_coo: z, zT and the gradients of x, z0
    and every parameter.  With N = 1 a node-major hidden state reports a row stride of 1, below Bs*C."""
    import gnn_b200
    S = np.array(TINY_S[tag])
    N = S.shape[0]
    B, T, F, H, K = 2, 3, 2, 3, 3
    torch.manual_seed(N)
    layer = gnn_b200.EdgeGatedHiddenState(F, H, K)
    layer.addGSO(torch.tensor(S, device="cuda").reshape(1, N, N))
    layer = layer.double().cuda()
    rng = np.random.default_rng(N)
    x, z0, dz = rng.standard_normal((B, T, F, N)), rng.standard_normal((B, H, N)), rng.standard_normal((B, T, H, N))
    xt = torch.tensor(x, device="cuda", requires_grad=True)
    zt = torch.tensor(z0, device="cuda", requires_grad=True)
    z, zT = layer(xt, zt)
    z.backward(torch.tensor(dz, device="cuda"))
    p = {k: v.detach().cpu().requires_grad_(True) for k, v in layer.state_dict().items()}
    x64, z64 = torch.tensor(x, requires_grad=True), torch.tensor(z0, requires_grad=True)
    rows, cols = np.nonzero(S)
    zr, _, _, _ = ego.edge_gated_hidden_state_coo(p, N, rows, cols, S[rows, cols], x64, z64, torch.tanh)
    zr.backward(torch.tensor(dz))
    assert _rel(z.detach().cpu().numpy(), zr.detach().numpy()) < 1e-10
    assert _rel(zT.detach().cpu().numpy()[:, 0, 0], zr.detach().numpy()[:, -1]) < 1e-10
    assert _rel(xt.grad.cpu().numpy(), x64.grad.numpy()) < 1e-10
    assert _rel(zt.grad.cpu().numpy(), z64.grad.numpy()) < 1e-10
    for name, prm in layer.named_parameters():
        ref = np.zeros(tuple(prm.shape)) if p[name].grad is None else p[name].grad.numpy()
        got = np.zeros(tuple(prm.shape)) if prm.grad is None else prm.grad.cpu().numpy()
        if not np.any(ref):                                   # an empty mask: the gates reach nothing
            assert np.abs(got).max(initial=0) < 1e-12, name
        else:
            assert _rel(got, ref) < 1e-10, name
