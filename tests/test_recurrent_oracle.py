"""The fp64 recurrent-layer oracle with error bounds (oracle/recurrent_oracle.py), checked on the CPU.

* Its values reproduce the reference's fixtures (grnn_cases / grnn_db_cases / lsigf_db_cases.npz) to 1e-12.
* Its fp32 bounds admit two legitimate fp32 implementations: the layers' own host logic in float32 with the dense torch
  filter standing in for the kernels, and the reference's formulation (dense per-step products) in float32.
* Its fp32 bounds reject plausible bugs: each planted defect exceeds the bound by 10x somewhere.
* The bounds are not vacuous: in fp32 the median of beta / |v| is <= 1e-4 for every output, and every gradient's
  median is pinned just above its measured value (MEDIAN_LIMITS).

The case builders and layer runners here are shared with the GPU table of tests/test_recurrent_bounds.py.
"""
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import lsigf_oracle as orc
import recurrent_oracle as ro

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = {n: np.load(os.path.join(HERE, "golden", n + ".npz")) for n in ("grnn_cases", "grnn_db_cases", "lsigf_db_cases")}
SIGMA = {"tanh": torch.tanh, "relu": torch.relu, "identity": lambda v: v}
NPD = {torch.float32: np.float32, torch.float64: np.float64}


# ------------------------------------------------------------------------------------------------ case builders
# Operands are chosen so that error propagation through the recursion cannot blow up: every GSO is scaled so that the
# row and the column sums of |S| are <= 1, and the hidden-to-hidden taps so that LSIGF(|b|, |S|, .) contracts (the sum
# of |b| over (e, k, g) for every output h, and over (h, e, k) for every input g, is <= 0.8).  Then the absolute-value
# runs the bounds are built on stay of the size of the values themselves, time step after time step.
def scaled(m, dtype):
    """scipy CSR scaled so that the row and column sums of |S| are <= 1, rounded to dtype."""
    m = sp.csr_matrix(m, dtype=np.float64)
    a = abs(m)
    s = max(float(np.asarray(a.sum(1)).max(initial=0)), float(np.asarray(a.sum(0)).max(initial=0)), 1e-300)
    m = m / s
    m.data = ro.rounded(m.data, dtype)
    m.sort_indices()
    return m


def contracting(w, rho=0.8):
    """hidden taps [H, E, K, H'] scaled so that LSIGF(|w|, |S|, .) and its adjoint contract by rho on such S."""
    a = np.abs(w)
    return w * rho / max(a.sum(axis=(1, 2, 3)).max(), a.sum(axis=(0, 1, 2)).max())


def random_gso(rng, N, deg=4):
    mask = rng.random((N, N)) < deg / N
    return sp.csr_matrix(np.where(mask, rng.standard_normal((N, N)), 0.0))


def grnn_params(rng, F, H, K, E, dtype, bias=True):
    s = 1.0 / np.sqrt(F * K)
    p = dict(a=ro.rounded(s * orc.biased_uniform(rng, (H, E, K, F)), dtype),
             b=ro.rounded(contracting(orc.biased_uniform(rng, (H, E, K, H))), dtype))
    if bias:
        p["xb"] = ro.rounded(rng.uniform(-s, s, (H, 1)), dtype)
        p["zb"] = ro.rounded(rng.uniform(-s, s, (H, 1)), dtype)
    return p


def grnn_case(seed, N, B, T, F, H, K, E=1, sigma="tanh", gates=None, dtype=np.float32, gso=None, bias=True):
    """GatedGRNN inputs: gates None, "scalar", "time" ([B, T, 1, 1]) or "node" ([1, T, 1, N], shared by the batch)."""
    rng = np.random.default_rng(seed)
    ops = [scaled(gso if (gso is not None and e == 0) else random_gso(rng, N), dtype) for e in range(E)]
    c = dict(S=ops, p=grnn_params(rng, F, H, K, E, dtype, bias), sigma=sigma,
             x=ro.rounded(orc.biased_uniform(rng, (B, T, F, N)), dtype), z0=ro.rounded(orc.biased_uniform(rng, (B, H, N)), dtype),
             dz=ro.rounded(orc.biased_uniform(rng, (B, T, H, N)), dtype))
    shape = dict(scalar=(1,), time=(B, T, 1, 1), node=(1, T, 1, N)).get(gates)
    c["q_hat"] = None if gates is None else ro.rounded(rng.uniform(0.2, 1.0, shape), dtype)
    c["q_check"] = None if gates is None else ro.rounded(rng.uniform(0.2, 1.0, shape), dtype)
    return c


def hidden_case(seed, kind, N, B, T, F, H, K, dtype=np.float32, gso=None):
    """HiddenState ("plain"), TimeGatedHiddenState ("time") or NodeGatedHiddenState ("node") inputs; parameters drawn
    by the layer's own initialisation (seeded), the GRNN taps with signs biased positive like orc.biased_uniform (the gate
    maps keep theirs, so that the gates do not saturate), hidden taps rescaled as above, all rounded to dtype."""
    import gnn_b200
    from gnn_b200 import recurrent as rec
    rng = np.random.default_rng(seed)
    S = scaled(gso if gso is not None else random_gso(rng, N), dtype)
    torch.manual_seed(seed)
    cls = dict(plain=rec.HiddenState, time=rec.TimeGatedHiddenState, node=rec.NodeGatedHiddenState)[kind]
    layer = cls(F, H, K).double()
    layer.addGSO(gnn_b200.SparseGSO.from_scipy([S]))              # draws the gate maps
    p = {k: v.detach().numpy().copy() for k, v in layer.state_dict().items()}
    for k in p:
        if k.endswith("Weights"):                                 # GRNN taps: the layer's magnitudes, signs biased positive
            p[k] = np.abs(p[k]) * np.where(rng.random(p[k].shape) < 0.2, -1.0, 1.0)
        if k.endswith("bWeights"):
            p[k] = contracting(p[k])
        p[k] = ro.rounded(p[k], dtype)
    return dict(kind=kind, S=[S], p=p, sigma="tanh", x=ro.rounded(orc.biased_uniform(rng, (B, T, F, N)), dtype),
                z0=ro.rounded(orc.biased_uniform(rng, (B, H, N)), dtype), dz=ro.rounded(orc.biased_uniform(rng, (B, T, H, N)), dtype))


def db_gso(rng, B, T, E, N, dtype, density=0.15, zero=()):
    """[B, T, E, N, N] time-varying GSO, every S(b, t, e) scaled as above; (b, t) in `zero` are all-zero blocks."""
    S = np.zeros((B, T, E, N, N))
    for b in range(B):
        for t in range(T):
            if (b, t) in zero:
                continue
            for e in range(E):
                S[b, t, e] = scaled(np.where(rng.random((N, N)) < density, rng.standard_normal((N, N)), 0.0),
                                    dtype).toarray()
    return S


def lsigf_db_case(seed, B, T, N, G, F, K, E=1, bias="F1", dtype=np.float32, zero=()):
    rng = np.random.default_rng(seed)
    s = 1.0 / np.sqrt(G * K)
    c = dict(S=db_gso(rng, B, T, E, N, dtype, zero=zero), h=ro.rounded(rng.uniform(-s, s, (F, E, K, G)), dtype),
             x=ro.rounded(orc.biased_uniform(rng, (B, T, G, N)), dtype), dy=ro.rounded(orc.biased_uniform(rng, (B, T, F, N)), dtype))
    c["b"] = None if bias is None else ro.rounded(rng.uniform(-s, s, (F, 1) if bias == "F1" else (F, N)), dtype)
    return c


def grnn_db_case(seed, B, T, N, F, H, K, E=1, sigma="tanh", dtype=np.float32, bias=True, zero=()):
    rng = np.random.default_rng(seed)
    c = dict(S=db_gso(rng, B, T, E, N, dtype, zero=zero), sigma=sigma, x=ro.rounded(orc.biased_uniform(rng, (B, T, F, N)), dtype),
             z0=ro.rounded(orc.biased_uniform(rng, (B, H, N)), dtype), dz=ro.rounded(orc.biased_uniform(rng, (B, T, H, N)), dtype))
    c.update(grnn_params(rng, F, H, K, E, dtype, bias))
    return c


# ------------------------------------------------------------------------------------------------ oracle and runners
def oracle_grnn(c, dt, bug=None, grads=True):
    q = lambda k: None if c[k] is None else ro.exact(c[k])          # noqa: E731
    return ro.grnn(c["p"], c["S"], c["x"], c["z0"], c["sigma"], dt, q("q_hat"), q("q_check"),
                   c["dz"] if grads else None, bug)


def oracle_hidden(c, dt, bug=None, grads=True):
    return ro.hidden_state(c["kind"], c["p"], c["S"], c["x"], c["z0"], c["sigma"], dt, c["dz"] if grads else None, bug)


def oracle_lsigf_db(c, dt, bug=None, grads=True):
    return ro.lsigf_db(c["h"], c["S"], c["x"], c["b"], dt, c["dy"] if grads else None, bug)


def oracle_grnn_db(c, dt, bug=None, grads=True):
    return ro.grnn_db(c["a"], c["b"], c["S"], c["x"], c["z0"], c["sigma"], dt, c.get("xb"), c.get("zb"),
                      c["dz"] if grads else None, bug)


def _t(a, dtype, device, grad=False):
    return torch.tensor(a, dtype=dtype, device=device).requires_grad_(grad)


def run_grnn(c, dtype, device, S):
    """GatedGRNN forward + backward; S: the GSO argument (dense tensor, SparseGSO).  -> {name: tensor} named as the oracle."""
    from gnn_b200 import recurrent as rec
    p = {k: _t(v, dtype, device, True) for k, v in c["p"].items()}
    x, z0 = _t(c["x"], dtype, device, True), _t(c["z0"], dtype, device, True)
    q = lambda k: None if c[k] is None else _t(c[k], dtype, device)  # noqa: E731
    z = rec.GatedGRNN(p["a"], p["b"], S, x, z0, SIGMA[c["sigma"]], q("q_hat"), q("q_check"), p.get("xb"), p.get("zb"))
    z.backward(_t(c["dz"], dtype, device))
    out = dict(z=z, dx=x.grad, dz0=z0.grad)
    out.update({k: v.grad for k, v in p.items()})
    return out


def run_hidden(c, dtype, device, S):
    from gnn_b200 import recurrent as rec
    B, T, F, N = c["x"].shape
    H, _, K, _ = c["p"]["aWeights"].shape
    cls = dict(plain=rec.HiddenState, time=rec.TimeGatedHiddenState, node=rec.NodeGatedHiddenState)[c["kind"]]
    layer = cls(F, H, K).to(device=device, dtype=dtype)
    layer.addGSO(S)
    layer = layer.to(device=device, dtype=dtype)
    layer.load_state_dict({k: torch.tensor(v) for k, v in c["p"].items()})
    x, z0 = _t(c["x"], dtype, device, True), _t(c["z0"], dtype, device, True)
    z, zT = layer(x, z0)
    z.backward(_t(c["dz"], dtype, device))
    out = dict(z=z, zT=zT, dx=x.grad, dz0=z0.grad)
    out.update({"g_" + k: v.grad for k, v in layer.named_parameters()})
    return out


def run_lsigf_db(c, dtype, device):
    from gnn_b200 import delayed
    h, x = _t(c["h"], dtype, device, True), _t(c["x"], dtype, device, True)
    b = None if c["b"] is None else _t(c["b"], dtype, device, True)
    y = delayed.LSIGF_DB(h, _t(c["S"], dtype, device), x, b)
    y.backward(_t(c["dy"], dtype, device))
    out = dict(y=y, dh=h.grad, dx=x.grad)
    if b is not None:
        out["db"] = b.grad
    return out


def run_grnn_db(c, dtype, device):
    from gnn_b200 import delayed
    p = {k: _t(c[k], dtype, device, True) for k in ("a", "b", "xb", "zb") if k in c}
    x, z0 = _t(c["x"], dtype, device, True), _t(c["z0"], dtype, device, True)
    z = delayed.GRNN_DB(p["a"], p["b"], _t(c["S"], dtype, device), x, z0, SIGMA[c["sigma"]], p.get("xb"), p.get("zb"))
    z.backward(_t(c["dz"], dtype, device))
    out = dict(z=z, dx=x.grad, dz0=z0.grad, da=p["a"].grad, db=p["b"].grad)
    if "xb" in p:
        out["dxb"], out["dzb"] = p["xb"].grad, p["zb"].grad
    return out


def violations(got, ref):
    """{name: max |got - v| / beta} over the oracle's outputs the run produced."""
    return {k: orc.bound_violation(got[k].detach().double().cpu().numpy().reshape(ref[k][0].shape), ref[k][0], ref[k][1])
            for k in ref if k in got}


def test_oracle_rules_cover_every_output_of_the_runners():
    """Every tensor a runner hands back has its (v, beta) in the oracle, so a GPU row checks all of them."""
    c = grnn_case(1, 20, 2, 3, 2, 3, 3, gates="node")
    assert set(oracle_grnn(c, np.float64)) == {"z", "dx", "dz0", "a", "b", "xb", "zb", "dq_hat", "dq_check"}
    h = hidden_case(1, "time", 12, 2, 3, 2, 3, 2)
    assert {"g_" + k for k in h["p"]} | {"z", "zT", "dx", "dz0"} == set(oracle_hidden(h, np.float64))


def test_slab_operators_match_the_product_plan_inputs():
    """ro.slab_ops (scipy block_diag, the reference of the _SlabOps rows) has exactly the pattern and values of
    delayed.slab_csr, including an operator left empty by an all-zero S[:, t]."""
    from gnn_b200 import delayed
    rng = np.random.default_rng(3)
    S = db_gso(rng, 3, 5, 2, 7, np.float32, zero={(b, 2) for b in range(3)})
    A = ro.slab_ops(S)
    fwd, bwd, R = delayed.slab_csr(torch.tensor(S))
    assert len(A) == len(bwd) == 8 and R == 21
    for o, (rowptr, col, val) in enumerate(bwd):
        assert np.array_equal(A[o].indptr, rowptr.numpy()) and np.array_equal(A[o].indices, col.numpy())
        assert np.array_equal(A[o].data, val.numpy())
    assert A[2].nnz == A[3].nnz == 0 and all(A[o].nnz > 0 for o in (0, 1, 4, 5, 6, 7))


# ------------------------------------------------------------------------------------------------ pinned values
def test_values_reproduce_the_static_recurrent_fixtures():
    g = GOLD["grnn_cases"]
    for tag, kind in (("plain", "plain"), ("nobias", "plain"), ("time", "time"), ("node", "node")):
        p = {k[len(tag) + 3:]: g[k] for k in g.files if k.startswith(tag + "_p_")}
        r = ro.hidden_state(kind, p, list(g[tag + "_S"]), g[tag + "_x"], g[tag + "_z0"], "tanh", np.float64,
                            dz=g[tag + "_dz"])
        want = {n: g["%s_%s" % (tag, n)] for n in ("z", "zT", "dx", "dz0")}
        want.update({"g_" + k: g["%s_g_%s" % (tag, k)] for k in p})
        assert set(want) <= set(r)
        for n, w in want.items():
            assert np.abs(r[n][0].reshape(w.shape) - w).max() <= 1e-12 * max(1.0, np.abs(w).max()), (tag, n)


@pytest.mark.parametrize("tag", ["ga", "gb", "gc", "gd", "ge", "gf"])
def test_values_reproduce_the_grnn_db_fixtures(tag):
    g = GOLD["grnn_db_cases"]
    B, T, N, F, H, K, E, bias, sg = (int(v) for v in g[tag + "_meta"])
    f = lambda n: g[tag + "_" + n]                                   # noqa: E731
    r = ro.grnn_db(f("a"), f("b"), f("S"), f("x"), f("z0"), ["tanh", "relu"][sg], np.float64,
                   f("xb") if bias else None, f("zb") if bias else None, dz=f("dz"))
    names = ["z", "da", "db", "dx", "dz0"] + (["dxb", "dzb"] if bias else [])
    for n in names:
        assert np.abs(r[n][0] - f(n)).max() <= 1e-12 * max(1.0, np.abs(f(n)).max()), (tag, n)


@pytest.mark.parametrize("tag", ["fa", "fb", "fc", "fd", "fe"])
def test_values_reproduce_the_lsigf_db_fixtures(tag):
    g = GOLD["lsigf_db_cases"]
    bias = int(g[tag + "_meta"][7])
    f = lambda n: g[tag + "_" + n]                                   # noqa: E731
    r = ro.lsigf_db(f("h"), f("S"), f("x"), f("b") if bias else None, np.float64, dy=f("dy"))
    for n in ["y", "dh", "dx"] + (["db"] if bias else []):
        assert np.abs(r[n][0] - f(n)).max() <= 1e-12 * max(1.0, np.abs(f(n)).max()), (tag, n)


# ------------------------------------------------------------------------------------------------ fp32 admission
@pytest.fixture
def dense_filters(monkeypatch):
    """The layers' filters on the CPU: the dense torch restatement for LSIGF, the space-time operator densified for
    LSIGF_DB and torch.sparse over slab_csr for the delay-line hops (as the test_widen_* host-logic tests do)."""
    import gnn_b200
    from gnn_b200 import delayed
    from gnn_b200 import recurrent as rec
    from host_filters import SparseSlabOps, dense_from_csr
    monkeypatch.setattr(rec, "_lsigf", orc.lsigf_dense_torch)
    monkeypatch.setattr(gnn_b200.graphML, "LSIGF", orc.lsigf_dense_torch)

    def apply(h, S, x_big, b_big):
        csr, M = delayed.block_delay_csr(S)
        return orc.lsigf_dense_torch(h, dense_from_csr(csr, M, S.dtype), x_big, b_big)
    monkeypatch.setattr(delayed, "_apply", apply)
    monkeypatch.setattr(delayed, "_slab_ops", SparseSlabOps)


def _dense(c):
    return torch.tensor(np.stack([m.toarray() for m in c["S"]]), dtype=torch.float32)


CPU_GRNN = {
    "grnn-ungated-tanh": lambda: grnn_case(2, 60, 2, 4, 3, 5, 3),
    "grnn-relu-E2": lambda: grnn_case(3, 50, 3, 5, 4, 6, 3, E=2, sigma="relu"),
    "grnn-scalar": lambda: grnn_case(4, 40, 2, 4, 2, 4, 2, gates="scalar"),
    "grnn-time": lambda: grnn_case(5, 40, 2, 4, 2, 4, 3, gates="time"),
    "grnn-node": lambda: grnn_case(6, 40, 2, 4, 2, 4, 3, gates="node"),
}
CPU_HIDDEN = {k: (lambda k=k: hidden_case(7, k, 30, 2, 4, 3, 5, 3)) for k in ("plain", "time", "node")}
CPU_LSIGF_DB = {
    "lsigf-db-F1": lambda: lsigf_db_case(8, 3, 5, 12, 3, 4, 3),
    "lsigf-db-FN-E2": lambda: lsigf_db_case(9, 2, 4, 10, 3, 5, 3, E=2, bias="FN"),
    "lsigf-db-zero-block": lambda: lsigf_db_case(10, 2, 4, 10, 2, 3, 3, zero=((1, 2),)),
}
CPU_GRNN_DB = {
    "grnn-db-K3-E2": lambda: grnn_db_case(11, 3, 6, 10, 2, 4, 3, E=2),
    "grnn-db-K4-relu": lambda: grnn_db_case(12, 2, 5, 9, 3, 5, 4, sigma="relu"),
}


@pytest.mark.parametrize("cid", sorted(CPU_GRNN))
def test_fp32_host_logic_lies_within_the_bound_grnn(cid, dense_filters):
    c = CPU_GRNN[cid]()
    got = run_grnn(c, torch.float32, "cpu", _dense(c))
    v = violations(got, oracle_grnn(c, np.float32))
    assert max(v.values()) <= 1.0, v


@pytest.mark.parametrize("kind", sorted(CPU_HIDDEN))
def test_fp32_host_logic_lies_within_the_bound_hidden_state(kind, dense_filters):
    c = CPU_HIDDEN[kind]()
    got = run_hidden(c, torch.float32, "cpu", _dense(c))
    v = violations(got, oracle_hidden(c, np.float32))
    assert len(v) == 4 + len(c["p"])
    assert max(v.values()) <= 1.0, v


@pytest.mark.parametrize("cid", sorted(CPU_LSIGF_DB))
def test_fp32_host_logic_lies_within_the_bound_lsigf_db(cid, dense_filters):
    c = CPU_LSIGF_DB[cid]()
    v = violations(run_lsigf_db(c, torch.float32, "cpu"), oracle_lsigf_db(c, np.float32))
    assert max(v.values()) <= 1.0, v


@pytest.mark.parametrize("cid", sorted(CPU_GRNN_DB))
def test_fp32_host_logic_lies_within_the_bound_grnn_db(cid, dense_filters):
    c = CPU_GRNN_DB[cid]()
    v = violations(run_grnn_db(c, torch.float32, "cpu"), oracle_grnn_db(c, np.float32))
    assert max(v.values()) <= 1.0, v


def _reference_grnn_db(a, b, S, x, z0, sigma, xb, zb, E, K):
    """The reference's formulation of GRNN_DB (graphML.py:1096-1290): per-(b, t) dense products x(t-k) S(t-k+1)..S(t)."""
    T = x.shape[1]
    zs, hist = [], [z0]
    for t in range(T):
        acc = xb.reshape(1, -1, 1) + zb.reshape(1, -1, 1)
        for e in range(E):
            for k in range(K):
                if t - k < 0:
                    continue
                xs, zz = x[:, t - k], hist[t - k]
                for s in range(t - k + 1, t + 1):
                    xs, zz = torch.matmul(xs, S[:, s, e]), torch.matmul(zz, S[:, s, e])
                acc = acc + torch.einsum("hf,bfn->bhn", a[:, e, k], xs) + torch.einsum("hg,bgn->bhn", b[:, e, k], zz)
        zs.append(sigma(acc))
        hist.append(zs[-1])
    return torch.stack(zs, 1)


def test_fp32_reference_formulations_lie_within_the_bound():
    """The reference's own dense formulations, in float32 with autograd: the GRNN as per-step LSIGF products
    (graphML.py:1403, :1461), LSIGF_DB as per-(b, t) products with a unit delay (the flocking restatement), GRNN_DB as
    the per-(b, t) delayed products.  They sum in other orders than the layers; all lie within the bound."""
    f32 = torch.float32
    # GatedGRNN with node gates
    c = CPU_GRNN["grnn-node"]()
    S = _dense(c)
    p = {k: _t(v, f32, "cpu", True) for k, v in c["p"].items()}
    x, z0 = _t(c["x"], f32, "cpu", True), _t(c["z0"], f32, "cpu", True)
    qh, qc = _t(c["q_hat"], f32, "cpu"), _t(c["q_check"], f32, "cpu")
    B, T, F, N = x.shape
    H = p["a"].shape[0]
    Ax = orc.lsigf_dense_torch(p["a"], S, x.reshape(B * T, F, N), p["xb"]).reshape(B, T, H, N)
    zt, zs = z0, []
    for t in range(T):
        zt = torch.tanh(qh[:, t] * Ax[:, t] + qc[:, t] * orc.lsigf_dense_torch(p["b"], S, zt, p["zb"]))
        zs.append(zt)
    z = torch.stack(zs, 1)
    z.backward(_t(c["dz"], f32, "cpu"))
    got = dict(z=z, dx=x.grad, dz0=z0.grad, **{k: v.grad for k, v in p.items()})
    v = violations(got, oracle_grnn(c, np.float32))
    assert len(v) == 7 and max(v.values()) <= 1.0, v
    # LSIGF_DB, flocking-style unit-delay products
    c = CPU_LSIGF_DB["lsigf-db-FN-E2"]()
    h, x, bb = _t(c["h"], f32, "cpu", True), _t(c["x"], f32, "cpu", True), _t(c["b"], f32, "cpu", True)
    S = _t(c["S"], f32, "cpu")
    B, T, G, N = x.shape
    F, E, K, _ = h.shape
    zz, y = x.unsqueeze(2).expand(B, T, E, G, N), 0.0
    for k in range(K):
        if k > 0:
            zz = torch.matmul(torch.cat((torch.zeros_like(zz[:, :1]), zz[:, :-1]), 1), S)
        y = y + torch.einsum("feg,btegn->btfn", h[:, :, k], zz)
    y = y + bb
    y.backward(_t(c["dy"], f32, "cpu"))
    v = violations(dict(y=y, dh=h.grad, dx=x.grad, db=bb.grad), oracle_lsigf_db(c, np.float32))
    assert len(v) == 4 and max(v.values()) <= 1.0, v
    # GRNN_DB, per-(b, t) delayed products
    c = CPU_GRNN_DB["grnn-db-K3-E2"]()
    p = {k: _t(c[k], f32, "cpu", True) for k in ("a", "b", "xb", "zb")}
    x, z0 = _t(c["x"], f32, "cpu", True), _t(c["z0"], f32, "cpu", True)
    z = _reference_grnn_db(p["a"], p["b"], _t(c["S"], f32, "cpu"), x, z0, torch.tanh, p["xb"], p["zb"],
                           c["a"].shape[1], c["a"].shape[2])
    z.backward(_t(c["dz"], f32, "cpu"))
    got = dict(z=z, dx=x.grad, dz0=z0.grad, da=p["a"].grad, db=p["b"].grad, dxb=p["xb"].grad, dzb=p["zb"].grad)
    v = violations(got, oracle_grnn_db(c, np.float32))
    assert len(v) == 7 and max(v.values()) <= 1.0, v


# ------------------------------------------------------------------------------------------------ mutants
MUTANTS = [
    # (layer, case, bug, output that must show it)
    ("grnn", "grnn-ungated-tanh", "S^T", "z"),
    ("grnn", "grnn-ungated-tanh", "z_t-2", "z"),
    ("grnn", "grnn-time", "gate_t+1", "z"),
    ("grnn", "grnn-ungated-tanh", "no_zBias", "z"),
    ("grnn", "grnn-ungated-tanh", "dW_last", "b"),
    ("grnn", "grnn-ungated-tanh", "dz0_hop1", "dz0"),
    ("lsigf_db", "lsigf-db-F1", "S_t", "y"),
    ("lsigf_db", "lsigf-db-F1", "history", "y"),
    ("lsigf_db", "lsigf-db-FN-E2", "bias_interleaved", "y"),
    ("grnn_db", "grnn-db-K3-E2", "op+1", "z"),
    ("grnn_db", "grnn-db-K3-E2", "slot", "z"),
    ("grnn_db", "grnn-db-K3-E2", "swap_e", "z"),
    ("grnn_db", "grnn-db-K3-E2", "dW_last", "db"),
    ("grnn_db", "grnn-db-K3-E2", "dz0_hop1", "dz0"),
]
_LAYER = dict(grnn=(CPU_GRNN, oracle_grnn), lsigf_db=(CPU_LSIGF_DB, oracle_lsigf_db), grnn_db=(CPU_GRNN_DB, oracle_grnn_db))


@pytest.mark.parametrize("layer,cid,bug,out", MUTANTS, ids=["%s-%s" % (m[0], m[2]) for m in MUTANTS])
def test_planted_bug_exceeds_the_fp32_bound_tenfold(layer, cid, bug, out):
    cases, oracle = _LAYER[layer]
    c = cases[cid]()
    grads = out not in ("z", "y")
    ref = oracle(c, np.float32, grads=grads)
    bad = oracle(c, np.float64, bug=bug, grads=grads)
    v = orc.bound_violation(bad[out][0], ref[out][0], ref[out][1])
    assert v >= 10.0, "%s/%s: the planted bug is only %.3g x the bound" % (cid, bug, v)


# ------------------------------------------------------------------------------------------------ non-vacuity
# The median of beta / |v| of every output, pinned 25 % above its measured value (two digits, rounded up): a rule that
# loosens fails here.  The outputs (z, zT, y) sit near 1e-5.  Gradients that sum N*B*T products of a state and an
# adjoint of both signs sit higher, up to 2e-3 for the gate GRNNs of the gated layers: their bound carries the worst case
# gamma_n of those sums (and, for the gates, sigmoid', the gate map's adjoint and a second reverse recursion), while the
# error of an actual sum grows like sqrt(n) u.
MEDIAN_LIMITS = {'grnn-db-K3-E2': {'da': 0.00023,
                   'db': 0.00017,
                   'dx': 2.4e-05,
                   'dxb': 2.4e-05,
                   'dz0': 1.2e-05,
                   'dzb': 1.2e-05,
                   'z': 1.3e-05},
 'grnn-db-K4-relu': {'da': 2.3e-05,
                     'db': 1.8e-05,
                     'dx': 9.2e-06,
                     'dxb': 7.6e-06,
                     'dz0': 9.5e-07,
                     'dzb': 2e-06,
                     'z': 1.6e-05},
 'grnn-node': {'a': 0.00017,
               'b': 0.00015,
               'dq_check': 6.1e-05,
               'dq_hat': 4.8e-05,
               'dx': 1.9e-05,
               'dz0': 1.7e-05,
               'xb': 3.2e-05,
               'z': 1.8e-05,
               'zb': 1.3e-05},
 'grnn-relu-E2': {'a': 0.00096,
                  'b': 0.00066,
                  'dx': 2.3e-05,
                  'dz0': 2.4e-05,
                  'xb': 6.4e-05,
                  'z': 3.1e-05,
                  'zb': 1.6e-05},
 'grnn-scalar': {'a': 0.00022,
                 'b': 0.00048,
                 'dq_check': 0.00027,
                 'dq_hat': 0.00027,
                 'dx': 2.2e-05,
                 'dz0': 1.9e-05,
                 'xb': 3.3e-05,
                 'z': 2.8e-05,
                 'zb': 1.5e-05},
 'grnn-time': {'a': 0.00022,
               'b': 0.00017,
               'dq_check': 7.7e-05,
               'dq_hat': 4e-05,
               'dx': 2.6e-05,
               'dz0': 1.7e-05,
               'xb': 3e-05,
               'z': 1.6e-05,
               'zb': 1.1e-05},
 'grnn-ungated-tanh': {'a': 0.00056,
                       'b': 0.00042,
                       'dx': 2.6e-05,
                       'dz0': 2.9e-05,
                       'xb': 4.8e-05,
                       'z': 2.3e-05,
                       'zb': 1.9e-05},
 'hidden-node': {'dx': 4.7e-05,
                 'dz0': 6.1e-05,
                 'g_aWeights': 0.00068,
                 'g_bWeights': 0.00048,
                 'g_forgetGateGRNN.aWeights': 0.0019,
                 'g_forgetGateGRNN.bWeights': 0.0011,
                 'g_forgetGateGRNN.xBias': 0.00017,
                 'g_forgetGateGRNN.zBias': 0.00015,
                 'g_forgetGateGraphFilter.bias': 4.4e-05,
                 'g_forgetGateGraphFilter.weight': 0.0015,
                 'g_inputGateGRNN.aWeights': 0.0017,
                 'g_inputGateGRNN.bWeights': 0.0025,
                 'g_inputGateGRNN.xBias': 9.9e-05,
                 'g_inputGateGRNN.zBias': 8.4e-05,
                 'g_inputGateGraphFilter.bias': 5.1e-05,
                 'g_inputGateGraphFilter.weight': 0.0013,
                 'g_xBias': 3.1e-05,
                 'g_zBias': 1.6e-05,
                 'z': 2.3e-05,
                 'zT': 2.6e-05},
 'hidden-plain': {'dx': 2.7e-05,
                  'dz0': 3.6e-05,
                  'g_aWeights': 0.00058,
                  'g_bWeights': 0.00047,
                  'g_xBias': 2.7e-05,
                  'g_zBias': 1.3e-05,
                  'z': 3.3e-05,
                  'zT': 3.7e-05},
 'hidden-time': {'dx': 0.00023,
                 'dz0': 0.00033,
                 'g_aWeights': 0.0015,
                 'g_bWeights': 0.0013,
                 'g_forgetGateFC.bias': 5.7e-05,
                 'g_forgetGateFC.weight': 8.4e-05,
                 'g_forgetGateGRNN.aWeights': 0.0018,
                 'g_forgetGateGRNN.bWeights': 0.0024,
                 'g_forgetGateGRNN.xBias': 0.00083,
                 'g_forgetGateGRNN.zBias': 0.00072,
                 'g_inputGateFC.bias': 5.6e-05,
                 'g_inputGateFC.weight': 8.2e-05,
                 'g_inputGateGRNN.aWeights': 0.0021,
                 'g_inputGateGRNN.bWeights': 0.002,
                 'g_inputGateGRNN.xBias': 0.00072,
                 'g_inputGateGRNN.zBias': 0.00063,
                 'g_xBias': 6.8e-05,
                 'g_zBias': 5.4e-05,
                 'z': 5.5e-05,
                 'zT': 6e-05},
 'lsigf-db-F1': {'db': 1.6e-05, 'dh': 7.4e-05, 'dx': 1.6e-05, 'y': 1.5e-05},
 'lsigf-db-FN-E2': {'db': 7.4e-06, 'dh': 2.7e-05, 'dx': 1.6e-05, 'y': 1.7e-05},
 'lsigf-db-zero-block': {'db': 6.7e-06, 'dh': 1.8e-05, 'dx': 1.6e-05, 'y': 1.6e-05}}


def _median_rel(ref):
    out = {}
    for k, (v, b) in ref.items():
        nz = np.abs(v) > 0
        out[k] = float(np.median(b[nz] / np.abs(v[nz]))) if nz.any() else 0.0
    return out


@pytest.mark.parametrize("cid", sorted(MEDIAN_LIMITS))
def test_fp32_bound_is_not_vacuous(cid):
    if cid in CPU_GRNN:
        ref = oracle_grnn(CPU_GRNN[cid](), np.float32)
    elif cid.startswith("hidden-"):
        ref = oracle_hidden(CPU_HIDDEN[cid[7:]](), np.float32)
    elif cid in CPU_LSIGF_DB:
        ref = oracle_lsigf_db(CPU_LSIGF_DB[cid](), np.float32)
    else:
        ref = oracle_grnn_db(CPU_GRNN_DB[cid](), np.float32)
    med = _median_rel(ref)
    assert sorted(med) == sorted(MEDIAN_LIMITS[cid])
    assert max(m for k, m in med.items() if k in ("z", "zT", "y")) <= 1e-4, med
    loose = {k: (m, MEDIAN_LIMITS[cid][k]) for k, m in med.items() if m > MEDIAN_LIMITS[cid][k]}
    assert not loose, loose


def test_every_cpu_case_has_median_limits():
    assert set(MEDIAN_LIMITS) == set(CPU_GRNN) | {"hidden-" + k for k in CPU_HIDDEN} | set(CPU_LSIGF_DB) | set(CPU_GRNN_DB)
