"""The CPU oracle and the package's CPU-side logic against the UNMODIFIED reference.  The reference's results are stored
in tests/golden (oracle/ref_golden.py); the reference itself runs only when they are recorded."""
import numpy as np
import pytest
import torch

import lsigf_oracle as orc
import ref_import
from ref_golden import reference

def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


@pytest.mark.parametrize("seed", range(6))
def test_lsigf_random_cases_vs_reference(seed):
    rng = np.random.default_rng(seed)
    N = int(rng.integers(5, 40)); B = int(rng.integers(1, 4)); G = int(rng.integers(1, 6)); F = int(rng.integers(1, 6))
    K = int(rng.integers(1, 6)); E = int(rng.integers(1, 4))
    c = orc.random_case(1000 + seed, N, B, G, F, K, E, avg_deg=4, bias=["F1", "FN", None][seed % 3])
    t = lambda a: None if a is None else torch.tensor(a)  # noqa: E731

    def run_reference():
        gml = ref_import.import_reference()
        h, x = t(c["h"]).requires_grad_(True), t(c["x"]).requires_grad_(True)
        y = gml.LSIGF(h, t(c["S"]), x, t(c["b"]))
        y.backward(t(c["dy"]))
        return dict(y=y.detach().numpy(), dh=h.grad.numpy(), dx=x.grad.numpy())

    r = reference("lsigf_random_%d" % seed, run_reference)
    assert _rel(orc.lsigf_dense(c["h"], c["S"], c["x"], c["b"]), r["y"]) < 1e-12
    dh, dx, _ = orc.lsigf_grads_dense(c["h"], c["S"], c["x"], c["dy"])
    assert _rel(dh, r["dh"]) < 1e-12 and _rel(dx, r["dx"]) < 1e-12
    ys = orc.lsigf_sparse(c["h"], list(c["S"]), c["x"], c["b"])
    assert _rel(ys, r["y"]) < 1e-12


@pytest.mark.parametrize("kind", ["HiddenState", "TimeGatedHiddenState", "NodeGatedHiddenState"])
@pytest.mark.parametrize("seed", range(3))
def test_recurrent_layers_vs_reference_live(kind, seed, monkeypatch):
    """gnn_b200.recurrent against the reference layers (graphML.py:3540-4031) on random shapes.  The dense CPU oracle
    stands in for the CUDA filter, so this checks the recursion / gating / autograd wiring, not the kernels.  Seeded
    construction + addGSO consume the RNG in the reference's order, so both layers hold identical parameters."""
    import gnn_b200
    from gnn_b200 import recurrent as rec
    lsigf = lambda h, S, x, b=None: orc.lsigf_dense_torch(h, S, x, b)  # noqa: E731
    monkeypatch.setattr(rec, "_lsigf", lsigf)
    monkeypatch.setattr(gnn_b200.graphML, "LSIGF", lsigf)
    rng = np.random.default_rng(7000 + seed)
    N, B, T = int(rng.integers(4, 20)), int(rng.integers(1, 4)), int(rng.integers(1, 6))
    F, H, K = int(rng.integers(1, 4)), int(rng.integers(1, 5)), int(rng.integers(1, 4))
    E = int(rng.integers(1, 3)) if kind == "HiddenState" else 1     # the gate GRNNs are built with E = 1 (:3757)
    bias = bool(seed % 2 == 0)
    S = torch.tensor(orc.random_sparse_gso(rng, N, 4, E))
    x, z0 = rng.standard_normal((B, T, F, N)), rng.standard_normal((B, H, N))
    dz = rng.standard_normal((B, T, H, N))

    def run(mod):
        torch.manual_seed(seed)
        torch.set_default_dtype(torch.float64)
        try:
            layer = getattr(mod, kind)(F, H, K, E=E, bias=bias)
            layer.addGSO(S)
        finally:
            torch.set_default_dtype(torch.float32)
        xt, zt = torch.tensor(x, requires_grad=True), torch.tensor(z0, requires_grad=True)
        z, zT = layer(xt, zt)
        z.backward(torch.tensor(dz))
        out = dict(z=z.detach().numpy(), zT=zT.detach().numpy(), dx=xt.grad.numpy(), dz0=zt.grad.numpy())
        for n, p in layer.named_parameters():
            out["p:" + n], out["g:" + n] = p.detach().numpy(), p.grad.numpy()
        return out

    r = reference("recurrent_%s_%d" % (kind, seed), lambda: run(ref_import.import_reference()))
    m = run(rec)
    assert sorted(k for k in r if k.startswith("p:")) == sorted(k for k in m if k.startswith("p:"))
    for k in (k for k in r if k.startswith("p:")):
        assert np.array_equal(r[k], m[k]), k                      # same init
        g = "g:" + k[2:]
        assert _rel(m[g], r[g]) < 1e-11, g
    assert m["z"].shape == r["z"].shape and m["zT"].shape == r["zT"].shape
    assert _rel(m["z"], r["z"]) < 1e-12 and _rel(m["zT"], r["zT"]) < 1e-12
    assert _rel(m["dx"], r["dx"]) < 1e-11 and _rel(m["dz0"], r["dz0"]) < 1e-11


@pytest.mark.parametrize("dataType", [np.float64, torch.float64])
def test_sparse_source_localization_matches_reference_dataset(dataType):
    """gnn_b200.datasets_sparse.SourceLocalization (sparse mat-vec diffusion) == the reference data class
    (dataTools.py:472-592, dense matrix powers) for the same numpy seed: signals, labels, splits and the helper methods.
    The graph is the reference's SBM draw, stored with its results."""
    import scipy.sparse as sp
    from gnn_b200 import datasets_sparse
    sources = [2, 11, 23]
    scores = np.random.default_rng(0).standard_normal((7, 3))
    yhat = torch.tensor(scores) if dataType is torch.float64 else scores
    num = lambda a: a.numpy() if isinstance(a, torch.Tensor) else np.asarray(a)  # noqa: E731

    def make(cls, graph):
        np.random.seed(5)
        d = cls(graph, 20, 6, 7, sources, tMax=9, dataType=dataType)
        d.expandDims()
        np.random.seed(6)
        return d, (d.getSamples("train", 5), d.getSamples("test", [1, 3]), d.getSamples("valid", 2))

    def flatten(d, draws):
        out = {}
        for part in ("train", "valid", "test"):
            xs, ys = d.samples[part]["signals"], d.samples[part]["targets"]
            out[part + ":x"], out[part + ":y"] = num(xs), num(ys)
            out[part + ":types"] = np.array([type(xs).__name__, str(xs.dtype), str(ys.dtype)])
        for i, (xa, ya) in enumerate(draws):
            out["draw%d:x" % i], out["draw%d:y" % i] = num(xa), num(ya)
        out["evaluate"] = np.float64(float(d.evaluate(yhat, d.samples["test"]["targets"])))
        return out

    def run_reference():
        ref_import.import_reference()
        import alegnn.utils.graphTools as graphTools
        import alegnn.utils.dataTools as dataTools
        np.random.seed(3)
        G = graphTools.Graph("SBM", 30, {"nCommunities": 3, "probIntra": 0.7, "probInter": 0.2})
        return dict(W=G.W, **flatten(*make(dataTools.SourceLocalization, G)))

    r = reference("source_localization_%s" % ("torch" if dataType is torch.float64 else "numpy"), run_reference)

    class SparseG:                                   # what a large-graph caller would hold: no dense W anywhere
        N, W = r["W"].shape[0], sp.csr_matrix(r["W"])

    m = flatten(*make(datasets_sparse.SourceLocalization, SparseG))
    for part in ("train", "valid", "test"):
        assert m[part + ":types"].tolist() == r[part + ":types"].tolist()
        assert m[part + ":x"].shape == r[part + ":x"].shape
        assert np.abs(m[part + ":x"] - r[part + ":x"]).max() < 1e-13 and np.array_equal(m[part + ":y"], r[part + ":y"])
    for i in range(3):
        xa, xb = m["draw%d:x" % i], r["draw%d:x" % i]
        assert xa.shape == xb.shape and np.abs(xa - xb).max() < 1e-13 and np.array_equal(m["draw%d:y" % i], r["draw%d:y" % i])
    assert float(m["evaluate"]) == float(r["evaluate"])


# ------------------------------------------------------------------------------------------------ install()
# install() rebinds names of a module object; the tests below install into a stand-in module that carries the names the
# reference's alegnn.utils.graphML exposes, and rebuild each reference architecture from the layers found on it after
# install() (the way the architectures look them up), with the reference's stored parameters.  The reference
# architecture's own output and gradients (recorded by `run_reference`) are the expected values.
_INSTALLED = ("LSIGF", "GraphFilter", "EVGF", "EdgeVariantGF", "MaxPoolLocal", "MaxLocalActivation",
              "MedianLocalActivation", "HiddenState", "TimeGatedHiddenState", "NodeGatedHiddenState", "LSIGF_DB",
              "GraphFilter_DB", "GRNN_DB", "HiddenState_DB")
_LEFT_ALONE = ("GatedGRNN", "EdgeGatedHiddenState", "NoPool")


def _standin():
    import types
    mod = types.ModuleType("graphML_standin")
    for n in _INSTALLED + _LEFT_ALONE:
        setattr(mod, n, type(n, (), {}))
    return mod


def _params(net, prefix="p:"):
    return {prefix + n: p.detach().numpy() for n, p in net.state_dict().items()}


def _grads(net):
    return {"g:" + n: p.grad.numpy() for n, p in net.named_parameters()}


def _load(net, r):
    keys = sorted(k[2:] for k in r if k.startswith("p:"))
    assert sorted(net.state_dict().keys()) == keys                 # the reference architecture's parameter names
    net.load_state_dict({k: torch.tensor(r["p:" + k]) for k in keys})


def _dense_apply(h, S_, x_big, b_big):
    """delayed._apply stand-in: the dense CPU oracle on the space-time CSR operator."""
    from gnn_b200 import delayed
    csr, M = delayed.block_delay_csr(S_)
    dense = torch.zeros(len(csr), M, M, dtype=S_.dtype)
    for e, (rowptr, col, val) in enumerate(csr):
        dense[e, torch.repeat_interleave(torch.arange(M), rowptr[1:] - rowptr[:-1]), col.long()] = val
    return orc.lsigf_dense_torch(h, dense, x_big, b_big)


def _z0_drawn_next(shape):
    """The tensor the next torch.randn(shape) call will return, without consuming it."""
    state = torch.get_rng_state()
    z0 = torch.randn(shape)
    torch.set_rng_state(state)
    return z0


def test_install_retargets_reference_module():
    import gnn_b200
    gml = _standin()
    orig = {n: getattr(gml, n) for n in _INSTALLED + _LEFT_ALONE}
    S = np.eye(8) * 0.5 + np.diag(np.ones(7), 1) * 0.25

    def run_reference():
        import torch.nn as nn
        ref = ref_import.import_reference()
        import alegnn.modules.architectures as archit
        net = archit.SelectionGNN([1, 4], [3], True, nn.ReLU, [8], ref.NoPool, [1], [2], S)
        return {"shape:" + n: np.array(p.shape) for n, p in net.state_dict().items()}

    r = reference("install_selectiongnn_parameters", run_reference)
    try:
        assert gnn_b200.install(gml) is gml
        assert gml.LSIGF is gnn_b200.LSIGF and gml.GraphFilter is gnn_b200.GraphFilter
        assert gml.EVGF is gnn_b200.EVGF and gml.EdgeVariantGF is gnn_b200.EdgeVariantGF
        assert gml.MaxPoolLocal is gnn_b200.MaxPoolLocal
        assert all(getattr(gml, n) is not orig[n] for n in _INSTALLED)
        assert all(getattr(gml, n) is orig[n] for n in _LEFT_ALONE)
        # the first layer SelectionGNN([1, 4], [3], ...) builds from the module is this package's, with the reference's
        # parameter names and shapes
        layer = gml.GraphFilter(1, 4, 3, 1, True)
        assert {"GFL.0." + n: tuple(p.shape) for n, p in layer.state_dict().items()} == \
            {k[6:]: tuple(v.tolist()) for k, v in r.items() if k.startswith("shape:GFL.0.")}
        assert tuple(layer.weight.shape) == (4, 1, 3, 1)
        layer.addGSO(torch.tensor(S).reshape(1, 8, 8))
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            layer(torch.zeros(2, 1, 8, dtype=torch.float64))
    finally:
        gnn_b200.uninstall(gml)
    assert {n: getattr(gml, n) for n in orig} == orig


def test_install_retargets_recurrent_layers(monkeypatch):
    """GraphRecurrentNN (architectures.py:4357-4560: HiddenState -> GraphFilter -> relu -> per-node readout) rebuilt from
    the retargeted module equals the reference architecture; the dense CPU oracle stands in for the CUDA filter."""
    import torch.nn as nn
    import gnn_b200
    from gnn_b200 import recurrent as rec
    S = np.eye(6) * 0.5 + np.diag(np.ones(5), 1) * 0.25
    x = torch.tensor(np.random.default_rng(0).standard_normal((3, 4, 2, 6)), dtype=torch.float32)
    B, T, F, G, H, N = 3, 4, 2, 3, 3, 6

    def run_reference():
        ref_import.import_reference()
        import alegnn.modules.architectures as archit
        torch.manual_seed(11)
        net = archit.GraphRecurrentNN(F, G, H, [2, 2], True, torch.tanh, torch.relu, nn.ReLU, [2], S.astype(np.float32))
        torch.manual_seed(12)                       # z0 is drawn inside splitForward (architectures.py:4547)
        z0 = _z0_drawn_next((B, H, N))
        return dict(y=net(x).detach().numpy(), z0=z0.numpy(), **_params(net))

    r = reference("install_graph_recurrent_nn", run_reference)
    lsigf = lambda h, S_, x_, b=None: orc.lsigf_dense_torch(h, S_, x_, b)  # noqa: E731
    monkeypatch.setattr(rec, "_lsigf", lsigf)
    monkeypatch.setattr(gnn_b200.graphML, "LSIGF", lsigf)
    gml = gnn_b200.install(_standin())
    try:
        St = torch.tensor(S.astype(np.float32)).reshape(1, N, N)
        net = nn.Module()
        net.hiddenState = gml.HiddenState(F, H, 2, nonlinearity=torch.tanh, E=1, bias=True)
        net.outputState = gml.GraphFilter(H, G, 2, E=1, bias=True)
        net.Readout = nn.Sequential(nn.Linear(G, 2, bias=True))
        net.hiddenState.addGSO(St)
        net.outputState.addGSO(St)
        _load(net, r)
        assert isinstance(net.hiddenState, gnn_b200.HiddenState) and isinstance(net.outputState, gnn_b200.GraphFilter)
        z, _ = net.hiddenState(x, torch.tensor(r["z0"]))
        y_out = torch.relu(net.outputState(z.reshape(B * T, H, N))).reshape(B, T, G, N)
        y = net.Readout(y_out.permute(0, 1, 3, 2)).permute(0, 1, 3, 2)
    finally:
        gnn_b200.uninstall(gml)
    y_ref = torch.tensor(r["y"])
    assert y.shape == y_ref.shape and torch.allclose(y, y_ref, rtol=1e-5, atol=1e-6)


def test_install_retargets_batch_delay_filter(monkeypatch):
    """LocalGNN_DB (architecturesTime.py:33-205: two GraphFilter_DB layers + tanh + per-node readout) rebuilt from the
    retargeted module equals the reference architecture, output and every parameter gradient; the dense CPU oracle
    applied to the space-time CSR stands in for the CUDA filter."""
    import torch.nn as nn
    import gnn_b200
    from gnn_b200 import delayed
    rng = np.random.default_rng(3)
    B, T, N, E = 3, 5, 7, 2
    S = torch.tensor(np.stack([np.stack([orc.random_sparse_gso(rng, N, 3, E) for _ in range(T)]) for _ in range(B)]),
                     dtype=torch.float32)
    x = torch.tensor(rng.standard_normal((B, T, 2, N)), dtype=torch.float32)

    def run_reference():
        ref_import.import_reference()
        import alegnn.modules.architecturesTime as architTime
        torch.manual_seed(21)
        net = architTime.LocalGNN_DB([2, 4, 3], [3, 2], True, nn.Tanh, [5, 2], E)
        y = net(x, S)
        y.sum().backward()
        return dict(y=y.detach().numpy(), **_params(net), **_grads(net))

    r = reference("install_local_gnn_db", run_reference)
    monkeypatch.setattr(delayed, "_apply", _dense_apply)
    gml = gnn_b200.install(_standin())
    try:
        net = nn.Module()
        net.GFL = nn.Sequential(gml.GraphFilter_DB(2, 4, 3, E, True), nn.Tanh(), gml.GraphFilter_DB(4, 3, 2, E, True), nn.Tanh())
        net.Readout = nn.Sequential(nn.Linear(3, 5, bias=True), nn.Tanh(), nn.Linear(5, 2, bias=True))
        _load(net, r)
        assert isinstance(net.GFL[0], gnn_b200.GraphFilter_DB) and isinstance(net.GFL[2], gnn_b200.GraphFilter_DB)
        net.GFL[0].addGSO(S)
        net.GFL[2].addGSO(S)
        y = net.Readout(net.GFL(x).permute(0, 1, 3, 2)).permute(0, 1, 3, 2)
        y.sum().backward()
    finally:
        gnn_b200.uninstall(gml)
    assert y.shape == r["y"].shape and torch.allclose(y, torch.tensor(r["y"]), rtol=1e-5, atol=1e-6)
    for n, p in net.named_parameters():
        assert torch.allclose(p.grad, torch.tensor(r["g:" + n]), rtol=1e-4, atol=1e-5), n


def test_install_retargets_batch_delay_recurrence(monkeypatch):
    """GraphRecurrentNN_DB (architecturesTime.py:273-470: HiddenState_DB -> GraphFilter_DB -> tanh -> per-node readout)
    rebuilt from the retargeted module equals the reference architecture, output and every parameter gradient; torch.sparse
    on the per-time-step CSR operators stands in for the hop kernel, the dense CPU oracle for the filters."""
    import torch.nn as nn
    import gnn_b200
    from gnn_b200 import delayed
    rng = np.random.default_rng(4)
    B, T, N, E, F, G, H = 2, 6, 7, 2, 2, 3, 4
    S = torch.tensor(np.stack([np.stack([orc.random_sparse_gso(rng, N, 3, E) for _ in range(T)]) for _ in range(B)]),
                     dtype=torch.float32)
    x = torch.tensor(rng.standard_normal((B, T, F, N)), dtype=torch.float32)

    def run_reference():
        ref_import.import_reference()
        import alegnn.modules.architecturesTime as architTime
        torch.manual_seed(22)                       # parameters, then the random initial hidden state (:447)
        net = architTime.GraphRecurrentNN_DB(F, G, H, [3, 2], True, torch.tanh, torch.tanh, nn.Tanh, [5, 2], E)
        z0 = _z0_drawn_next((B, H, N))
        y = net(x, S)
        y.sum().backward()
        return dict(y=y.detach().numpy(), z0=z0.numpy(), **_params(net), **_grads(net))

    r = reference("install_graph_recurrent_nn_db", run_reference)

    class SparseSlabOps:
        def __init__(self, S_):
            fwd, _, R = delayed.slab_csr(S_)
            self.A = [torch.sparse_coo_tensor(torch.stack((torch.repeat_interleave(torch.arange(R), rp[1:] - rp[:-1]), col.long())),
                                              val, (R, R)) for (rp, col, val) in fwd]

        def hop(self, o, src):
            return torch.sparse.mm(self.A[o], src)

    monkeypatch.setattr(delayed, "_apply", _dense_apply)
    monkeypatch.setattr(delayed, "_slab_ops", SparseSlabOps)
    gml = gnn_b200.install(_standin())
    try:
        net = nn.Module()
        net.hiddenState = gml.HiddenState_DB(F, H, 3, nonlinearity=torch.tanh, E=E, bias=True)
        net.outputState = gml.GraphFilter_DB(H, G, 2, E=E, bias=True)
        net.Readout = nn.Sequential(nn.Linear(G, 5, bias=True), nn.Tanh(), nn.Linear(5, 2, bias=True))
        _load(net, r)
        assert isinstance(net.hiddenState, gnn_b200.HiddenState_DB) and isinstance(net.outputState, gnn_b200.GraphFilter_DB)
        net.hiddenState.addGSO(S)
        net.outputState.addGSO(S)
        z, _ = net.hiddenState(x, torch.tensor(r["z0"]))
        y_out = torch.tanh(net.outputState(z))
        y = net.Readout(y_out.permute(0, 1, 3, 2)).permute(0, 1, 3, 2)
        y.sum().backward()
    finally:
        gnn_b200.uninstall(gml)
    assert y.shape == r["y"].shape and torch.allclose(y, torch.tensor(r["y"]), rtol=1e-5, atol=1e-6)
    for n, p in net.named_parameters():
        assert torch.allclose(p.grad, torch.tensor(r["g:" + n]), rtol=1e-4, atol=1e-5), n


def test_reference_gatedgrnn_with_biases_after_install(monkeypatch):
    """The reference's GatedGRNN (graphML.py:1292-1527) reshapes its biases to (1, H, 1) before calling the module-global
    LSIGF (:1394-1404, :1461); after install() that call lands in gnn_b200.LSIGF, whose argument handling must accept
    what the reference's broadcast add accepts.  The dense CPU oracle stands in for the CUDA dispatch
    (`graphML._dispatch`), so the shape handling of the product function itself is what runs here; the recursion itself
    is this package's GatedGRNN, against the reference function's stored output."""
    import gnn_b200
    from gnn_b200 import recurrent as rec
    seen = []

    def dispatch(h, S, x, b):
        seen.append(None if b is None else tuple(b.shape))
        return orc.lsigf_dense_torch(h, S, x, b)

    rng = np.random.default_rng(5)
    B, T, F, H, N, K, E = 2, 3, 2, 4, 7, 3, 1
    a = torch.tensor(rng.standard_normal((H, E, K, F)))
    bt = torch.tensor(rng.standard_normal((H, E, K, H)))
    S = torch.tensor(orc.random_sparse_gso(rng, N, 3, E))
    x = torch.tensor(rng.standard_normal((B, T, F, N)))
    z0 = torch.tensor(rng.standard_normal((B, H, N)))
    xb, zb = torch.tensor(rng.standard_normal((H, 1))), torch.tensor(rng.standard_normal((H, 1)))

    def run_reference():
        ref = ref_import.import_reference()
        return dict(z=ref.GatedGRNN(a, bt, S, x, z0, torch.tanh, xBias=xb, zBias=zb).numpy())

    r = reference("gatedgrnn_with_biases", run_reference)
    monkeypatch.setattr(gnn_b200.graphML, "_dispatch", dispatch)
    monkeypatch.setattr(rec, "_lsigf", gnn_b200.LSIGF)
    # the call the reference makes: bias reshaped to (1, H, 1), normalised to the [F, 1] the C ABI takes
    y = gnn_b200.LSIGF(a, S, x[:, 0], xb.reshape(1, H, 1))
    assert seen == [(H, 1)]
    assert _rel(y.numpy(), orc.lsigf_dense_torch(a, S, x[:, 0], xb).numpy()) < 1e-14
    got = rec.GatedGRNN(a, bt, S, x, z0, torch.tanh, xBias=xb.reshape(1, H, 1), zBias=zb.reshape(1, H, 1))
    assert seen and all(s == (H, 1) for s in seen)
    assert got.shape == r["z"].shape and _rel(got.numpy(), r["z"]) < 1e-12
    # shapes the reference's broadcast would reject are still rejected loudly
    with pytest.raises(RuntimeError, match="bias must broadcast"):
        gnn_b200.LSIGF(a, S, x[:, 0], torch.zeros(H + 1, 1, dtype=torch.float64))


def test_fuse_layers_on_a_reference_architecture(monkeypatch):
    """SURVEY.md §8 f-1 at the architecture level: the reference's `SelectionGNN` with two graph-convolutional layers and
    `MaxPoolLocal` (architectures.py:166-296, 422-460), rebuilt from the retargeted module's layers (GraphFilter -> ReLU
    -> MaxPoolLocal per layer, one linear readout on the flattened output) and loaded with the reference network's
    parameters, then fuse_layers().  Output, input gradient and every parameter gradient must agree with the reference
    network's; the state_dict keys must not change.  CPU: the oracle / a torch gather stand in for the two CUDA dispatch
    hooks, everything else (fused-activation plumbing, Identity rewiring, neighbourhoods) is product code."""
    import torch.nn as nn
    import gnn_b200
    from gnn_b200 import graphML, pooling

    def dispatch(h, S, x, b, act=0):
        y = orc.lsigf_dense_torch(h, S, x, b)
        return torch.relu(y) if act else y

    def gather_max(x, nb32, n_out, max_nb):
        B, F, _ = x.shape
        return x.index_select(2, nb32.reshape(-1).long()).reshape(B, F, n_out, max_nb).max(dim=3)[0]

    rng = np.random.default_rng(21)
    N = 24
    A = (rng.random((N, N)) < 0.2).astype(np.float64)
    A = np.maximum(A, A.T)
    np.fill_diagonal(A, 0)
    S = A / max(np.abs(np.linalg.eigvalsh(A)).max(), 1e-9)
    x = torch.tensor(rng.standard_normal((3, 2, N)))

    def run_reference():
        ref = ref_import.import_reference()
        import alegnn.modules.architectures as archit
        torch.manual_seed(5)
        torch.set_default_dtype(torch.float64)
        try:
            net = archit.SelectionGNN([2, 4, 3], [3, 2], True, nn.ReLU, [10, 6], ref.MaxPoolLocal, [1, 2], [5], S)
        finally:
            torch.set_default_dtype(torch.float32)
        xr = x.clone().requires_grad_(True)
        y = net(xr)
        y.sum().backward()
        return dict(y=y.detach().numpy(), dx=xr.grad.numpy(), **_params(net), **_grads(net))

    r = reference("fuse_layers_selectiongnn", run_reference)
    monkeypatch.setattr(graphML, "_dispatch", dispatch)
    monkeypatch.setattr(pooling, "_gather_max", gather_max)
    gml = gnn_b200.install(_standin())
    try:
        St = torch.tensor(S).reshape(1, N, N)
        torch.set_default_dtype(torch.float64)
        try:
            net = nn.Module()
            net.GFL = nn.Sequential(gml.GraphFilter(2, 4, 3, 1, True), nn.ReLU(), gml.MaxPoolLocal(N, 10, 1),
                                    gml.GraphFilter(4, 3, 2, 1, True), nn.ReLU(), gml.MaxPoolLocal(10, 6, 2))
            net.MLP = nn.Sequential(nn.Linear(3 * 6, 5, bias=True))
        finally:
            torch.set_default_dtype(torch.float32)
        for i in (0, 2, 3, 5):
            net.GFL[i].addGSO(St)
        assert isinstance(net.GFL[0], gnn_b200.GraphFilter) and isinstance(net.GFL[2], gnn_b200.MaxPoolLocal)
        _load(net, r)
        keys = sorted(net.state_dict().keys())
        assert gnn_b200.fuse_layers(net) == 2
        assert isinstance(net.GFL[1], nn.Identity) and isinstance(net.GFL[4], nn.Identity)
        assert sorted(net.state_dict().keys()) == keys
        xm = x.clone().requires_grad_(True)
        y = net.MLP(net.GFL(xm).reshape(3, 3 * 6))
        y.sum().backward()
    finally:
        gnn_b200.uninstall(gml)
    assert _rel(y.detach().numpy(), r["y"]) < 1e-12
    assert _rel(xm.grad.numpy(), r["dx"]) < 1e-11
    for n, p in net.named_parameters():
        assert _rel(p.grad.numpy(), r["g:" + n]) < 1e-11, n
