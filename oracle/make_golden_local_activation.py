"""Generate tests/golden/local_activation_cases.npz by running the UNMODIFIED reference (alegnn).

TEST INFRASTRUCTURE.  Run once (`B200GF_REFERENCE_ROOT=<alegnn checkout> python oracle/make_golden_local_activation.py`);
the fixture is committed so that the tests need no reference checkout.  Every array in it is either a seeded input or
an output of the reference's own code, in fp64, on inputs without ties (standard normal draws):

  la_<Max|Median>_E<e>_K<k>_*   MaxLocalActivation / MedianLocalActivation (graphML.py:1535-1810), K = 1..3, E = 1..2:
                                S, weight, x, dy, y, dx, dw
  lagnn_*                        a two-layer LocalActivationGNN (alegnn/modules/architectures.py:481-780): GraphFilter,
                                 MaxLocalActivation (layer 0) / MedianLocalActivation (layer 1, put in place of the
                                 Max one the constructor builds), MaxPoolLocal, and a linear readout: S, x, dy, y, dx,
                                 p_<name> (state_dict) and g_<name> (every parameter gradient)
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
N_LAYER, B, F = 13, 2, 3


def gen_layers(gml, out):
    for kind in ("Max", "Median"):
        for E in (1, 2):
            for K in (1, 2, 3):
                seed = 1500 + 100 * (kind == "Median") + 10 * E + K
                rng = np.random.default_rng(seed)
                S = orc.random_sparse_gso(rng, N_LAYER, 2, E, symmetric=(E == 1))
                S[:, 0, :] = 0.0                    # node 0 has no out-neighbours: a one-node 1-hop list
                torch.manual_seed(seed)
                layer = getattr(gml, kind + "LocalActivation")(K).double()
                layer.addGSO(torch.tensor(S))
                x = rng.standard_normal((B, F, N_LAYER))
                xt = torch.tensor(x, requires_grad=True)
                y = layer(xt)
                dy = rng.standard_normal(tuple(y.shape))
                y.backward(torch.tensor(dy))
                p = "la_%s_E%d_K%d_" % (kind, E, K)
                for name, val in (("S", S), ("weight", layer.weight.detach().numpy()), ("x", x), ("dy", dy),
                                  ("y", y.detach().numpy()), ("dx", xt.grad.numpy()), ("dw", layer.weight.grad.numpy())):
                    out[p + name] = val


def gen_gnn(gml, out):
    import torch.nn as nn  # noqa: F401
    import alegnn.modules.architectures as archit
    seed, N, Bg = 1601, 12, 3
    rng = np.random.default_rng(seed)
    A = np.abs(orc.random_sparse_gso(rng, N, 2, 1)[0])
    S = (A + A.T) / 2
    for i in range(N - 1):                          # a path keeps every node in a neighbourhood of more than itself
        S[i, i + 1] = S[i + 1, i] = rng.uniform(0.2, 0.5)
    torch.manual_seed(seed)
    torch.set_default_dtype(torch.float64)
    try:
        net = archit.LocalActivationGNN([2, 3, 2], [2, 3], True, gml.MaxLocalActivation, [2, 1], [N, N],
                                        gml.MaxPoolLocal, [1, 2], [4], S)
        net.GFL[4] = gml.MedianLocalActivation(1)
        net.GFL[4].addGSO(net.S)
    finally:
        torch.set_default_dtype(torch.float32)
    x = rng.standard_normal((Bg, 2, N))
    xt = torch.tensor(x, requires_grad=True)
    y = net(xt)
    dy = rng.standard_normal(tuple(y.shape))
    y.backward(torch.tensor(dy))
    out["lagnn_meta"] = np.array([seed, N, Bg])
    for name, val in (("S", S), ("x", x), ("dy", dy), ("y", y.detach().numpy()), ("dx", xt.grad.numpy())):
        out["lagnn_" + name] = val
    for name, prm in net.named_parameters():
        out["lagnn_p_" + name] = prm.detach().numpy()
        out["lagnn_g_" + name] = prm.grad.numpy()


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    gml = ref_import.import_reference()
    out = {}
    gen_layers(gml, out)
    gen_gnn(gml, out)
    np.savez_compressed(os.path.join(OUT, "local_activation_cases.npz"), **out)
    print("local_activation_cases.npz:", len(out), "arrays;", sorted(k for k in out if k.startswith("lagnn_p_")))
