"""Generate tests/golden/grnn_edge_cases.npz by running the UNMODIFIED reference (alegnn).

TEST INFRASTRUCTURE.  Run once (`B200GF_REFERENCE_ROOT=<alegnn checkout> python oracle/make_golden_edge.py`); the
fixture is committed so that the tests need no reference checkout.  Every array in it is either a seeded input or an
output of the reference's own code:

  grnn_edge_cases.npz – `EdgeGatedHiddenState` (graphML.py:4033-4209) forward + all gradients in fp64, and the
                        reference's dense gates qHat / qCheck for one case.
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


def _edge_gso(rng, N, mode):
    """random_sparse_gso plus the diagonal of each edge-gating case: "plain" (as drawn), "diag" (non-zero S_ii on every
    node), "neg" (S_ii = -1 on some nodes, so the mask drops their diagonal; node 1 keeps only S_11 = -1, an empty mask
    row, and node 2 has no entry at all, a mask row holding only the diagonal)."""
    S = orc.random_sparse_gso(rng, N, 3)
    if mode == "diag":
        S[0][np.arange(N), np.arange(N)] = rng.uniform(0.2, 0.6, N) * rng.choice([-1.0, 1.0], N)
    elif mode == "neg":
        S[0][1, :] = 0.0
        S[0][:, 1] = 0.0
        S[0][2, :] = 0.0
        S[0][[1, 4, 7], [1, 4, 7]] = -1.0
    return S


def gen_grnn_edge(gml):
    """EdgeGatedHiddenState (graphML.py:4033-4209): GatedGRNN's edge path (:1410-1451, :1474-1514) on gates from
    learnAttentionGSO (:640-737), fp64: trajectory, input gradients and the gradients of all 16 parameters; the first
    case also stores the reference's dense gates qHat / qCheck [B, T, 1, N, N]."""
    out = {}
    # (tag, seed, N, B, T, F, H, K, bias, sigma, gso)
    cases = [("base", 901, 10, 2, 3, 2, 3, 3, True, "tanh", "plain"),
             ("nobias", 902, 9, 3, 2, 1, 4, 2, False, "tanh", "plain"),
             ("k1", 903, 8, 2, 3, 2, 3, 1, True, "tanh", "plain"),
             ("kgt", 904, 11, 2, 2, 1, 3, 4, True, "tanh", "plain"),          # more taps than time steps
             ("relu", 905, 10, 2, 3, 2, 2, 3, True, "relu", "plain"),
             ("diag", 906, 12, 2, 3, 1, 3, 3, True, "tanh", "diag"),          # non-zero S_ii
             ("neg", 907, 10, 3, 2, 2, 3, 3, True, "tanh", "neg")]            # S_ii = -1: diagonal outside the mask
    for (tag, seed, N, B, T, F, H, K, bias, sg, mode) in cases:
        rng = np.random.default_rng(seed)
        S = _edge_gso(rng, N, mode)
        torch.manual_seed(seed)
        layer = gml.EdgeGatedHiddenState(F, H, K, getattr(torch, sg), 1, bias)
        layer.addGSO(torch.tensor(S))
        layer.double()                                     # the gate attentions are created inside addGSO
        x = rng.standard_normal((B, T, F, N))
        z0 = rng.standard_normal((B, H, N))
        xt = torch.tensor(x, requires_grad=True)
        z0t = torch.tensor(z0, requires_grad=True)
        z, zT = layer(xt, z0t)
        dz = rng.standard_normal(tuple(z.shape))
        z.backward(torch.tensor(dz))
        out[tag + "_meta"] = np.array([seed, N, B, T, F, H, K, int(bias), {"tanh": 0, "relu": 1}[sg]])
        for name, val in (("S", S), ("x", x), ("z0", z0), ("dz", dz), ("z", z.detach().numpy()),
                          ("zT", zT.detach().numpy()), ("dx", xt.grad.numpy()), ("dz0", z0t.grad.numpy())):
            out[tag + "_" + name] = val
        for name, p in layer.named_parameters():
            out[tag + "_p_" + name] = p.detach().numpy()
            # K = 1 has no hop, so the gates reach nothing and autograd leaves their parameters without a gradient
            out[tag + "_g_" + name] = np.zeros(tuple(p.shape)) if p.grad is None else p.grad.numpy()
        if tag == "base":
            with torch.no_grad():
                for gate, grnn, gat in (("qHat", layer.inputGateGRNN, layer.inputGateGAT),
                                        ("qCheck", layer.forgetGateGRNN, layer.forgetGateGAT)):
                    zg, _ = grnn(xt, z0t)
                    q = gml.learnAttentionGSO(zg.reshape(B * T, H, N), gat.mixer, gat.weight, gat.S)
                    out[tag + "_" + gate] = q.reshape(B, T, 1, N, N).numpy()
    np.savez_compressed(os.path.join(OUT, "grnn_edge_cases.npz"), **out)
    print("grnn_edge_cases.npz:", sorted(k for k in out if k.endswith("_z")))


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    gen_grnn_edge(ref_import.import_reference())
