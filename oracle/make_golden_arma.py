"""Generate tests/golden/arma_cases.npz by running the UNMODIFIED reference (alegnn).

TEST INFRASTRUCTURE.  Run once (`B200GF_REFERENCE_ROOT=<alegnn checkout> python oracle/make_golden_arma.py`); the fixture
is committed so that the tests need no reference checkout.  Every array in it is either a seeded input or an output of
the reference's own code, in fp64.  Every GSO is non-symmetric, so the column convention of the Jacobi chains (S~ v) is
told apart from LSIGF's row convention (x S):

  arma_<tag>_*    the functional jARMA (graphML.py:490-638): forward, gradients of x, psi, varphi, phi and b
  armal_<tag>_*   GraphFilterARMA (graphML.py:2714-2847): forward, gradients of x and of every parameter
  armagnn_*       a two-layer ARMAfilterGNN (alegnn/modules/architectures.py:2243-2555) with MaxPoolLocal and an MLP
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_import  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")
BIAS_KINDS = {"none": 0, "F1": 1, "FN": 2}
DIAG_KINDS = {"zero": 0, "const": 1, "vary": 2, "mixed": 3}


def arma_gso(rng, N, E, diag):
    """E non-symmetric GSOs, entries uniform in [-0.5, 0.5] on 40 % of the positions; diagonal zero, constant (0.7 + e),
    varying (uniform in [-1, 1]) or mixed (zero in e = 0, varying in the others)."""
    S = rng.uniform(-0.5, 0.5, (E, N, N)) * (rng.uniform(size=(E, N, N)) < 0.4)
    for e in range(E):
        kind = diag if diag != "mixed" else ("zero" if e == 0 else "vary")
        np.fill_diagonal(S[e], {"zero": lambda: 0.0, "const": lambda: 0.7 + e,
                                "vary": lambda: rng.uniform(-1, 1, N)}[kind]())
    return S


def arma_params(rng, F, E, P, K, G):
    stdv = 1. / np.sqrt(G * P)                       # the ranges of GraphFilterARMA.reset_parameters
    return (rng.uniform(1 + 1 / stdv, 1 + 2 / stdv, (F, E, P, G)), rng.uniform(-stdv, stdv, (F, E, P, G)),
            rng.uniform(-stdv, stdv, (F, E, K, G)))


def gen_jarma(gml, out):
    # (tag, seed, N, B, G, F, P, K, E, tMax, diag, bias)
    cases = [("zt0", 2101, 9, 2, 3, 2, 1, 1, 1, 0, "zero", "none"),
             ("ct1", 2102, 8, 2, 2, 3, 2, 3, 2, 1, "const", "F1"),
             ("vt4", 2103, 10, 3, 2, 2, 2, 3, 1, 4, "vary", "FN"),
             ("vt5", 2104, 7, 1, 2, 2, 1, 1, 2, 5, "vary", "F1"),
             ("mt1", 2105, 9, 2, 2, 2, 2, 3, 2, 1, "mixed", "FN"),
             ("zt4", 2106, 8, 2, 2, 2, 2, 1, 1, 4, "zero", "F1"),
             ("ct5", 2107, 6, 2, 1, 2, 1, 3, 1, 5, "const", "none"),
             ("vt0", 2108, 6, 2, 2, 2, 2, 1, 2, 0, "vary", "none")]
    for (tag, seed, N, B, G, F, P, K, E, tMax, diag, bias) in cases:
        rng = np.random.default_rng(seed)
        S = arma_gso(rng, N, E, diag)
        psi, varphi, phi = arma_params(rng, F, E, P, K, G)
        x = rng.standard_normal((B, G, N))
        b = None if bias == "none" else rng.uniform(-0.5, 0.5, (F, 1) if bias == "F1" else (F, N))
        ts = {k: torch.tensor(v, requires_grad=True) for k, v in (("psi", psi), ("varphi", varphi), ("phi", phi),
                                                                  ("x", x))}
        bt = None if b is None else torch.tensor(b, requires_grad=True)
        u = gml.jARMA(ts["psi"], ts["varphi"], ts["phi"], torch.tensor(S), ts["x"], bt, tMax=tMax)
        dU = rng.standard_normal(tuple(u.shape))
        u.backward(torch.tensor(dU))
        p = "arma_%s_" % tag
        out[p + "meta"] = np.array([seed, N, B, G, F, P, K, E, tMax, DIAG_KINDS[diag], BIAS_KINDS[bias]])
        for name, val in (("S", S), ("psi", psi), ("varphi", varphi), ("phi", phi), ("x", x), ("dU", dU),
                          ("u", u.detach().numpy())):
            out[p + name] = val
        for k, t in ts.items():
            out[p + "d" + k] = t.grad.numpy()
        if b is not None:
            out[p + "b"] = b
            out[p + "db"] = bt.grad.numpy()


def gen_layer(gml, out):
    # (tag, seed, N, B, G, F, P, K, E, bias, tMax, Nin, diag)
    cases = [("nin", 2201, 10, 2, 2, 3, 2, 2, 1, True, 3, 7, "vary"),
             ("e2", 2202, 9, 2, 3, 2, 1, 3, 2, False, 4, 9, "mixed")]
    for (tag, seed, N, B, G, F, P, K, E, bias, tMax, Nin, diag) in cases:
        rng = np.random.default_rng(seed)
        S = arma_gso(rng, N, E, diag)
        torch.manual_seed(seed)
        layer = gml.GraphFilterARMA(G, F, P, K, E, bias, tMax)
        layer.double()
        layer.addGSO(torch.tensor(S))
        x = rng.standard_normal((B, G, Nin))
        xt = torch.tensor(x, requires_grad=True)
        y = layer(xt)
        dy = rng.standard_normal(tuple(y.shape))
        y.backward(torch.tensor(dy))
        p = "armal_%s_" % tag
        out[p + "meta"] = np.array([seed, N, B, G, F, P, K, E, int(bias), tMax, Nin])
        for name, val in (("S", S), ("x", x), ("dy", dy), ("y", y.detach().numpy()), ("dx", xt.grad.numpy())):
            out[p + name] = val
        for name, prm in layer.named_parameters():
            out[p + "p_" + name] = prm.detach().numpy()
            out[p + "g_" + name] = prm.grad.numpy()


def gen_gnn(gml, out):
    import torch.nn as nn
    import alegnn.modules.architectures as archit
    seed, N, B = 2301, 14, 3
    rng = np.random.default_rng(seed)
    # non-negative and symmetric off the diagonal, as the other GNN fixtures (MaxPoolLocal's neighbourhoods are those of
    # S's pattern), with a varying diagonal so that the layers take the general path
    A = np.abs(arma_gso(rng, N, 1, "zero")[0])
    S = (A + A.T) / 2 + np.diag(rng.uniform(0.1, 0.9, N))
    torch.manual_seed(seed)
    torch.set_default_dtype(torch.float64)
    try:
        net = archit.ARMAfilterGNN([2, 4, 3], [2, 1], [3, 2], True, nn.ReLU, [10, 6], gml.MaxPoolLocal, [1, 2], [5], S,
                                   tMax=3)
    finally:
        torch.set_default_dtype(torch.float32)
    x = rng.standard_normal((B, 2, N))
    xt = torch.tensor(x, requires_grad=True)
    y = net(xt)
    dy = rng.standard_normal(tuple(y.shape))
    y.backward(torch.tensor(dy))
    out["armagnn_meta"] = np.array([seed, N, B])
    for name, val in (("S", S), ("x", x), ("dy", dy), ("y", y.detach().numpy()), ("dx", xt.grad.numpy())):
        out["armagnn_" + name] = val
    for name, prm in net.named_parameters():
        out["armagnn_p_" + name] = prm.detach().numpy()
        out["armagnn_g_" + name] = prm.grad.numpy()


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    gml = ref_import.import_reference()
    out = {}
    gen_jarma(gml, out)
    gen_layer(gml, out)
    gen_gnn(gml, out)
    np.savez_compressed(os.path.join(OUT, "arma_cases.npz"), **out)
    print("arma_cases.npz:", len(out), "arrays")
