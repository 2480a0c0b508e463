"""Generate tests/golden/nvgf_cases.npz by running the UNMODIFIED reference (alegnn).

TEST INFRASTRUCTURE.  Run once (`B200GF_REFERENCE_ROOT=<alegnn checkout> python oracle/make_golden_nv.py`); the fixture
is committed so that the tests need no reference checkout.  Every array in it is either a seeded input or an output of
the reference's own code, in fp64:

  nvgf_<tag>_*   the functional NVGF (graphML.py:293-387): forward, gradients of x, h and b
  nvl_<tag>_*    NodeVariantGF (graphML.py:2317-2509): forward, gradients of x, weight and bias, copyNodes
  nvgnn_*        a two-layer NodeVariantGNN (alegnn/modules/architectures.py:1485-1719) with MaxPoolLocal and an MLP
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_import  # noqa: E402
import lsigf_oracle as orc  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")
BIAS_KINDS = {"none": 0, "F1": 1, "FN": 2}


def connected_gso(rng, N, E, chord=None, avg_deg=2):
    """E weighted GSOs whose pattern contains the undirected path 0 - 1 - ... - N-1 (so every node reaches node 0, and
    NodeVariantGF's search ends), plus random directed entries (avg_deg per row); `chord` = (i, j) adds the undirected
    edge i - j."""
    S = orc.random_sparse_gso(rng, N, avg_deg, E)
    for e in range(E):
        for i in range(N - 1):
            S[e, i, i + 1] = rng.uniform(0.2, 0.5)
            S[e, i + 1, i] = rng.uniform(0.2, 0.5)
        if chord is not None:
            S[e, chord[0], chord[1]] = rng.uniform(0.2, 0.5)
            S[e, chord[1], chord[0]] = rng.uniform(0.2, 0.5)
    return S


def gen_nvgf(gml, out):
    # (tag, seed, N, B, G, F, K, E, bias)
    cases = [("e1k3", 1101, 9, 2, 3, 4, 3, 1, "none"),
             ("e2k3", 1102, 8, 3, 2, 3, 3, 2, "F1"),
             ("e1k1", 1103, 7, 2, 3, 2, 1, 1, "FN"),
             ("e2k1", 1104, 6, 1, 2, 3, 1, 2, "F1"),
             ("e2k3fn", 1105, 10, 2, 2, 2, 3, 2, "FN")]
    for (tag, seed, N, B, G, F, K, E, bias) in cases:
        rng = np.random.default_rng(seed)
        S = orc.random_sparse_gso(rng, N, 3, E)
        h = rng.uniform(-1, 1, (F, E, K, G, N))
        x = rng.standard_normal((B, G, N))
        b = None if bias == "none" else rng.uniform(-0.5, 0.5, (F, 1) if bias == "F1" else (F, N))
        ht, xt = torch.tensor(h, requires_grad=True), torch.tensor(x, requires_grad=True)
        bt = None if b is None else torch.tensor(b, requires_grad=True)
        y = gml.NVGF(ht, torch.tensor(S), xt, bt)
        dy = rng.standard_normal(tuple(y.shape))
        y.backward(torch.tensor(dy))
        p = "nvgf_%s_" % tag
        out[p + "meta"] = np.array([seed, N, B, G, F, K, E, BIAS_KINDS[bias]])
        for name, val in (("S", S), ("h", h), ("x", x), ("dy", dy), ("y", y.detach().numpy()), ("dx", xt.grad.numpy()),
                          ("dh", ht.grad.numpy())):
            out[p + name] = val
        if b is not None:
            out[p + "b"] = b
            out[p + "db"] = bt.grad.numpy()


def gen_layer(gml, out):
    # (tag, seed, N, B, G, F, K, M, E, bias, Nin, chord, random entries per row)
    cases = [("mlt", 1201, 10, 2, 2, 3, 3, 4, 1, True, 10, (0, 6), 0),   # path + chord: copyNodes [0,1,2,3,3,0,0,0,0,0]
             ("mlt2", 1202, 16, 3, 3, 2, 2, 5, 2, True, 16, (2, 11), 2),
             ("meq", 1203, 9, 2, 2, 3, 3, 9, 2, False, 9, None, 2),
             ("mgt", 1204, 7, 2, 3, 2, 2, 11, 1, True, 7, None, 2),
             ("nin", 1205, 12, 2, 2, 2, 3, 3, 1, True, 8, (1, 9), 2)]
    for (tag, seed, N, B, G, F, K, M, E, bias, Nin, chord, deg) in cases:
        rng = np.random.default_rng(seed)
        S = connected_gso(rng, N, E, chord, deg)
        torch.manual_seed(seed)
        layer = gml.NodeVariantGF(G, F, K, M, E, bias)
        layer.double()
        layer.addGSO(torch.tensor(S))
        x = rng.standard_normal((B, G, Nin))
        xt = torch.tensor(x, requires_grad=True)
        y = layer(xt)
        dy = rng.standard_normal(tuple(y.shape))
        y.backward(torch.tensor(dy))
        p = "nvl_%s_" % tag
        out[p + "meta"] = np.array([seed, N, B, G, F, K, M, E, int(bias), Nin])
        for name, val in (("S", S), ("x", x), ("dy", dy), ("y", y.detach().numpy()), ("dx", xt.grad.numpy()),
                          ("copyNodes", layer.copyNodes.numpy())):
            out[p + name] = val
        for name, prm in layer.named_parameters():
            out[p + "p_" + name] = prm.detach().numpy()
            out[p + "g_" + name] = prm.grad.numpy()


def gen_gnn(gml, out):
    import torch.nn as nn
    import alegnn.modules.architectures as archit
    seed, N, B = 1301, 14, 3
    rng = np.random.default_rng(seed)
    # symmetric and non-negative, as the SelectionGNN fixtures: MaxPoolLocal's neighbourhoods are those of S's pattern
    A = np.abs(connected_gso(rng, N, 1, (0, 8))[0])
    S = (A + A.T) / 2
    torch.manual_seed(seed)
    torch.set_default_dtype(torch.float64)
    try:
        net = archit.NodeVariantGNN([2, 4, 3], [3, 2], [5, 6], True, nn.ReLU, [10, 6], gml.MaxPoolLocal, [1, 2], [5], S)
    finally:
        torch.set_default_dtype(torch.float32)
    x = rng.standard_normal((B, 2, N))
    xt = torch.tensor(x, requires_grad=True)
    y = net(xt)
    dy = rng.standard_normal(tuple(y.shape))
    y.backward(torch.tensor(dy))
    out["nvgnn_meta"] = np.array([seed, N, B])
    for name, val in (("S", S), ("x", x), ("dy", dy), ("y", y.detach().numpy()), ("dx", xt.grad.numpy()),
                      ("copy0", net.NVGFL[0].copyNodes.numpy()), ("copy3", net.NVGFL[3].copyNodes.numpy())):
        out["nvgnn_" + name] = val
    for name, prm in net.named_parameters():
        out["nvgnn_p_" + name] = prm.detach().numpy()
        out["nvgnn_g_" + name] = prm.grad.numpy()


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    gml = ref_import.import_reference()
    out = {}
    gen_nvgf(gml, out)
    gen_layer(gml, out)
    gen_gnn(gml, out)
    np.savez_compressed(os.path.join(OUT, "nvgf_cases.npz"), **out)
    print("nvgf_cases.npz:", len(out), "arrays;", {k: list(v) for k, v in out.items() if k.endswith("copyNodes")})
