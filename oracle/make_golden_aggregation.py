"""Generate tests/golden/aggregation_cases.npz by running the UNMODIFIED reference (alegnn).

TEST INFRASTRUCTURE.  Run once (`B200GF_REFERENCE_ROOT=<alegnn checkout> python oracle/make_golden_aggregation.py`); the
fixture is committed so that the tests need no reference checkout.  The reference runs on the CPU in float64 after
`.double()` (its SN is float64 whatever the GSO's dtype).  For every case <c>:

  <c>_meta      [kind (0 AggregationGNN, 1 MultiNodeAggregationGNN), B, N, E]
  <c>_S         the GSO [E, N, N] as our layers receive it (original numbering)
  <c>_x, <c>_dy, <c>_y, <c>_dx     input, the fixed loss's output gradient, output and input gradient
  <c>_p_<name>, <c>_g_<name>       state_dict and the gradient of every parameter

  agg_n1        nNodes = 1, maxN = None, E = 1, two conv layers, MLP, no AggMLP
  agg_n3_aggmlp nNodes = 3, maxN = 5, E = 2, non-empty AggMLP
  agg_n3        nNodes = 3, maxN = None, E = 1, empty AggMLP (output [B, MLP, nNodes])
  agg_n1_e2     nNodes = 1, maxN = 3, E = 2
  agg_degree    order='Degree', nNodes = 2, maxN = 4: the reference with order=None on the GSO reordered by
                graphTools.permDegree (its order='Degree' raises NameError), x and dx mapped back to the original
                numbering; <c>_order is that ordering
  multi         MultiNodeAggregationGNN, P = [3, 2], Q = [3, 2]
The constructor arguments of every case are CASES below, which the tests import.
"""
import copy
import os
import sys

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import lsigf_oracle as orc  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")

# name: (kind, seed, B, N, E, constructor keyword arguments without GSO / nonlinearity / poolingFunction)
CASES = {
    "agg_n1": ("agg", 2101, 3, 10, 1, dict(dimFeatures=[2, 3, 2], nFilterTaps=[3, 2], bias=True, poolingSize=[2, 1],
                                           dimLayersMLP=[4], maxN=None, nNodes=1, dimLayersAggMLP=[])),
    "agg_n3_aggmlp": ("agg", 2102, 2, 12, 2, dict(dimFeatures=[2, 3], nFilterTaps=[2], bias=True, poolingSize=[2],
                                                  dimLayersMLP=[4], maxN=5, nNodes=3, dimLayersAggMLP=[5, 2])),
    "agg_n3": ("agg", 2103, 2, 12, 1, dict(dimFeatures=[1, 2], nFilterTaps=[3], bias=True, poolingSize=[2],
                                           dimLayersMLP=[3], maxN=None, nNodes=3, dimLayersAggMLP=[])),
    "agg_n1_e2": ("agg", 2104, 3, 9, 2, dict(dimFeatures=[2, 2], nFilterTaps=[2], bias=False, poolingSize=[1],
                                             dimLayersMLP=[2], maxN=3, nNodes=1, dimLayersAggMLP=[])),
    "agg_degree": ("agg", 2105, 2, 12, 1, dict(dimFeatures=[2, 3], nFilterTaps=[2], bias=True, poolingSize=[1],
                                               dimLayersMLP=[3], maxN=4, nNodes=2, dimLayersAggMLP=[], order="Degree")),
    "multi": ("multi", 2106, 2, 10, 1, dict(nSelectedNodes=[3, 2], nShifts=[3, 2], dimFeatures=[[2, 3], [3, 2]],
                                            nFilterTaps=[[2], [1]], bias=True, poolingSize=[[1], [1]],
                                            dimLayersMLP=[4])),
}


def gso(seed, N, E):
    """Positive random weights (no ties in the degree order) on a sparse pattern, plus a path so that every node is
    reached within a few hops."""
    rng = np.random.default_rng(seed)
    S = np.abs(orc.random_sparse_gso(rng, N, 2, E))
    for e in range(E):
        for i in range(N - 1):
            S[e, i, i + 1] = rng.uniform(0.2, 0.6)
    return S / np.abs(S).sum(axis=2).max()


def build(archit, kind, kw, S):
    kw = copy.deepcopy(kw)                       # MultiNodeAggregationGNN appends to the caller's dimFeatures
    if kind == "agg":
        return archit.AggregationGNN(nonlinearity=nn.ReLU, poolingFunction=nn.MaxPool1d, GSO=S, **kw)
    return archit.MultiNodeAggregationGNN(nonlinearity=nn.ReLU, poolingFunction=nn.MaxPool1d, GSO=S, **kw)


def gen(archit, graphTools, name, out):
    kind, seed, B, N, E, kw = CASES[name]
    S = gso(seed, N, E)
    rng = np.random.default_rng(seed + 1)
    F0 = kw["dimFeatures"][0] if kind == "agg" else kw["dimFeatures"][0][0]
    x = rng.standard_normal((B, F0, N))
    S_ref, x_ref, order = S, x, np.arange(N)
    ref_kw = dict(kw)
    if kw.get("order") == "Degree":
        S_ref, order = graphTools.permDegree(S)
        order = np.asarray(order)
        x_ref = x[:, :, order]
        ref_kw["order"] = None
    torch.manual_seed(seed)
    net = build(archit, kind, ref_kw, S_ref).double()
    xt = torch.tensor(x_ref, requires_grad=True)
    y = net(xt)
    dy = rng.standard_normal(tuple(y.shape))
    y.backward(torch.tensor(dy))
    dx = np.empty_like(x)
    dx[:, :, order] = xt.grad.numpy()
    p = name + "_"
    out[p + "meta"] = np.array([kind == "multi", B, N, E])
    for k, v in (("S", S), ("x", x), ("dy", dy), ("y", y.detach().numpy()), ("dx", dx), ("order", order)):
        out[p + k] = v
    for k, v in net.state_dict().items():
        out[p + "p_" + k] = v.numpy()
    for k, prm in net.named_parameters():
        out[p + "g_" + k] = prm.grad.numpy()


if __name__ == "__main__":
    import ref_import
    ref_import.import_reference()
    import alegnn.modules.architectures as archit
    import alegnn.utils.graphTools as graphTools
    os.makedirs(OUT, exist_ok=True)
    out = {}
    for name in CASES:
        gen(archit, graphTools, name, out)
    np.savez_compressed(os.path.join(OUT, "aggregation_cases.npz"), **out)
    print("aggregation_cases.npz:", len(out), "arrays")
