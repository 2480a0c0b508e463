"""Generate tests/golden/attention_cases.npz by running the UNMODIFIED reference (alegnn).

TEST INFRASTRUCTURE.  Run once (`B200GF_REFERENCE_ROOT=<alegnn checkout> python oracle/make_golden_attention.py`); the
fixture is committed so that the tests need no reference checkout.  Every array in it is either a seeded input or an
output of the reference's own code, in fp64:

  ga_<tag>_*       graphAttention (graphML.py:739-809): forward, gradients of x, a and W
  gl_<tag>_*       graphAttentionLSIGF (graphML.py:811-895): forward, gradients of h, x, a, W (and b)
  ge_<tag>_*       graphAttentionEVGF (graphML.py:897-969): forward, gradients of x, a, W (and b)
  l<kind>_<tag>_*  GraphAttentional / GraphFilterAttentional / EdgeVariantAttentional (graphML.py:2849-3270): forward,
                   gradients of x and of every parameter, concatenating and averaging heads, with and without bias,
                   Nin < N
  net_<arch>_*     a two-layer GraphAttentionNetwork, GraphConvolutionAttentionNetwork and EdgeVariantAttention
                   (alegnn/modules/architectures.py:3575, :3815, :4088) with NoPool and an MLP

Every GSO is non-symmetric (LSIGF's row convention x S is told apart from S x) and has a node whose only entry is
S_ii = -1 in every edge feature (its diagonal leaves the mask |S + I| > 1e-9, an empty mask row, while S_ii stays a hop
entry), S_ii = -1 on one more node that keeps its other entries, and the pair (0, 2) at 6e-10 in every edge feature:
below the tolerance alone (E = 1: a hop entry outside the mask), above it summed over E = 2.  "n1" cases run on a
one-node graph.
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
SIGMAS = {"relu": 0, "tanh": 1}


def attention_gso(rng, N, E):
    if N == 1:
        return np.full((E, 1, 1), 0.7) * (1 + np.arange(E)).reshape(E, 1, 1)
    S = orc.random_sparse_gso(rng, N, 3, E)
    S[:, 1, :] = 0.0                               # node 1: S_11 = -1 its only entry, an empty mask row
    S[:, 1, 1] = -1.0
    S[:, 4, 4] = -1.0                              # node 4: diagonal outside the mask, other entries kept
    S[:, 4, 5] = rng.uniform(0.3, 0.6, E)
    S[:, 0, 2] = 6e-10                             # summed over e: in the mask only when E = 2
    return S


def _t(a):
    return torch.tensor(a, requires_grad=True)


def _store(out, p, meta, inputs, y, dy, grads):
    out[p + "meta"] = np.array(meta)
    for k, v in inputs.items():
        out[p + k] = v
    out[p + "y"] = y.detach().numpy()
    out[p + "dy"] = dy
    for k, v in grads.items():
        out[p + "d" + k] = np.zeros(v.shape) if v.grad is None else v.grad.numpy()


def gen_functionals(gml, out):
    # graphAttention: (tag, seed, N, B, G, F, P, E)
    for tag, seed, N, B, G, F, P, E in [("e1p1", 3101, 9, 2, 3, 2, 1, 1), ("e2p3", 3102, 10, 2, 2, 3, 3, 2),
                                        ("e1p3", 3103, 8, 3, 2, 2, 3, 1), ("n1", 3104, 1, 2, 2, 3, 2, 2)]:
        rng = np.random.default_rng(seed)
        S = attention_gso(rng, N, E)
        stdv = 1. / np.sqrt(G * P)
        inp = dict(S=S, x=rng.standard_normal((B, G, N)), a=rng.uniform(-stdv, stdv, (P, E, 2 * F)),
                   W=rng.uniform(-stdv, stdv, (P, E, F, G)))
        ts = {k: _t(inp[k]) for k in ("x", "a", "W")}
        y = gml.graphAttention(ts["x"], ts["a"], ts["W"], torch.tensor(S))
        dy = rng.standard_normal(tuple(y.shape))
        y.backward(torch.tensor(dy))
        _store(out, "ga_%s_" % tag, [seed, N, B, G, F, P, E], inp, y, dy, ts)
    # graphAttentionLSIGF: (tag, seed, N, B, G, F, P, E, K, bias)
    for tag, seed, N, B, G, F, P, E, K, bias in [("k1", 3201, 8, 2, 3, 2, 1, 1, 1, True),
                                                 ("k3e2", 3202, 9, 2, 2, 3, 3, 2, 3, False),
                                                 ("k3p1", 3203, 7, 1, 3, 2, 1, 1, 3, True),
                                                 ("k2p3", 3204, 8, 2, 2, 3, 3, 1, 2, True),
                                                 ("n1", 3205, 1, 2, 2, 3, 2, 2, 3, True)]:
        rng = np.random.default_rng(seed)
        S = attention_gso(rng, N, E)
        stdv = 1. / np.sqrt(G * P)
        inp = dict(S=S, x=rng.standard_normal((B, G, N)), a=rng.uniform(-stdv, stdv, (P, E, 2 * F)),
                   W=rng.uniform(-stdv, stdv, (P, E, F, G)), h=rng.uniform(-1, 1, (E, K)))
        names = ("h", "x", "a", "W")
        if bias:
            inp["b"] = rng.uniform(-stdv, stdv, (F, 1))
            names += ("b",)
        ts = {k: _t(inp[k]) for k in names}
        y = gml.graphAttentionLSIGF(ts["h"], ts["x"], ts["a"], ts["W"], torch.tensor(S), b=ts.get("b"))
        dy = rng.standard_normal(tuple(y.shape))
        y.backward(torch.tensor(dy))
        _store(out, "gl_%s_" % tag, [seed, N, B, G, F, P, E, K, int(bias)], inp, y, dy, ts)
    # graphAttentionEVGF: (tag, seed, N, B, G, F, P, E, K, bias)
    for tag, seed, N, B, G, F, P, E, K, bias in [("k1", 3301, 8, 2, 3, 2, 1, 1, 1, True),
                                                 ("k3e2", 3302, 9, 2, 2, 3, 3, 2, 3, False),
                                                 ("k3p1", 3303, 7, 1, 3, 2, 1, 1, 3, True),
                                                 ("k2e2", 3304, 8, 2, 2, 3, 1, 2, 2, True),
                                                 ("n1", 3305, 1, 2, 2, 3, 2, 2, 3, True)]:
        rng = np.random.default_rng(seed)
        S = attention_gso(rng, N, E)
        stdv = 1. / np.sqrt(G * K)
        inp = dict(S=S, x=rng.standard_normal((B, G, N)), a=rng.uniform(-stdv, stdv, (P, K, E, 2 * F)),
                   W=rng.uniform(-stdv, stdv, (P, K, E, F, G)))
        names = ("x", "a", "W")
        if bias:
            inp["b"] = rng.uniform(-stdv, stdv, (F, 1))
            names += ("b",)
        ts = {k: _t(inp[k]) for k in names}
        y = gml.graphAttentionEVGF(ts["x"], ts["a"], ts["W"], torch.tensor(S), b=ts.get("b"))
        dy = rng.standard_normal(tuple(y.shape))
        y.backward(torch.tensor(dy))
        _store(out, "ge_%s_" % tag, [seed, N, B, G, F, P, E, K, int(bias)], inp, y, dy, ts)


# (kind, tag, seed, N, B, G, F, K, P, E, bias, concatenate, Nin, sigma)
LAYER_CASES = [("ga", "cat", 3401, 10, 2, 3, 2, 3, 0, 2, False, True, 7, "relu"),
               ("ga", "mean", 3402, 9, 2, 2, 3, 1, 0, 1, False, False, 9, "tanh"),
               ("gl", "cat", 3403, 10, 2, 3, 2, 3, 2, 2, True, True, 8, "relu"),
               ("gl", "mean", 3404, 9, 2, 2, 3, 1, 3, 1, False, False, 9, "tanh"),
               ("ge", "cat", 3405, 10, 2, 3, 2, 2, 2, 2, True, True, 8, "relu"),
               ("ge", "mean", 3406, 9, 2, 2, 3, 3, 1, 1, False, False, 9, "tanh"),
               ("ge", "n1", 3407, 1, 2, 2, 3, 2, 2, 1, True, True, 1, "relu")]


def make_layer(mod, kind, G, F, K, P, E, bias, concatenate, sigma):
    sg = {"relu": torch.nn.functional.relu, "tanh": torch.tanh}[sigma]
    if kind == "ga":
        return mod.GraphAttentional(G, F, K, E, sg, concatenate)
    if kind == "gl":
        return mod.GraphFilterAttentional(G, F, K, P, E, bias, sg, concatenate)
    return mod.EdgeVariantAttentional(G, F, K, P, E, bias, sg, concatenate)


def gen_layers(gml, out):
    for kind, tag, seed, N, B, G, F, K, P, E, bias, cat, Nin, sigma in LAYER_CASES:
        rng = np.random.default_rng(seed)
        S = attention_gso(rng, N, E)
        torch.manual_seed(seed)
        layer = make_layer(gml, kind, G, F, K, P, E, bias, cat, sigma).double()
        layer.addGSO(torch.tensor(S))
        x = rng.standard_normal((B, G, Nin))
        xt = _t(x)
        y = layer(xt)
        dy = rng.standard_normal(tuple(y.shape))
        y.backward(torch.tensor(dy))
        p = "l%s_%s_" % (kind, tag)
        out[p + "meta"] = np.array([seed, N, B, G, F, K, P, E, int(bias), int(cat), Nin, SIGMAS[sigma]])
        for name, val in (("S", S), ("x", x), ("dy", dy), ("y", y.detach().numpy()), ("dx", xt.grad.numpy())):
            out[p + name] = val
        for name, prm in layer.named_parameters():
            out[p + "p_" + name] = prm.detach().numpy()
            # K = 1 in GraphFilterAttentional: no hop, so the attention reaches nothing and its mixer has no gradient
            out[p + "g_" + name] = np.zeros(tuple(prm.shape)) if prm.grad is None else prm.grad.numpy()


# (arch, seed, N, B, E): GraphAttentionNetwork([2, 4, 3], [2, 2], relu, [N, N], NoPool, [1, 1], [5], True, S);
# the two filter networks ([2, 4, 3], taps [2, 3], heads [2, 2], bias True, relu, ...)
NET_CASES = [("gat", 3501, 11, 3, 2), ("gcat", 3502, 10, 2, 1), ("eva", 3503, 9, 2, 2)]


def build_net(archit, gml, arch, N, S):
    relu = torch.nn.functional.relu
    if arch == "gat":
        return archit.GraphAttentionNetwork([2, 4, 3], [2, 2], relu, [N, N], gml.NoPool, [1, 1], [5], True, S)
    cls = archit.GraphConvolutionAttentionNetwork if arch == "gcat" else archit.EdgeVariantAttention
    return cls([2, 4, 3], [2, 3] if arch == "gcat" else [2, 2], [2, 2], True, relu, [N, N], gml.NoPool, [1, 1], [5], S)


def gen_nets(gml, out):
    import alegnn.modules.architectures as archit
    for arch, seed, N, B, E in NET_CASES:
        rng = np.random.default_rng(seed)
        S = attention_gso(rng, N, E)
        torch.manual_seed(seed)
        torch.set_default_dtype(torch.float64)
        try:
            net = build_net(archit, gml, arch, N, S)
        finally:
            torch.set_default_dtype(torch.float32)
        x = rng.standard_normal((B, 2, N))
        xt = _t(x)
        y = net(xt)
        dy = rng.standard_normal(tuple(y.shape))
        y.backward(torch.tensor(dy))
        p = "net_%s_" % arch
        out[p + "meta"] = np.array([seed, N, B, E])
        for name, val in (("S", S), ("x", x), ("dy", dy), ("y", y.detach().numpy()), ("dx", xt.grad.numpy())):
            out[p + name] = val
        for name, prm in net.named_parameters():
            out[p + "p_" + name] = prm.detach().numpy()
            # K = 1 in GraphFilterAttentional: no hop, so the attention reaches nothing and its mixer has no gradient
            out[p + "g_" + name] = np.zeros(tuple(prm.shape)) if prm.grad is None else prm.grad.numpy()


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    gml = ref_import.import_reference()
    out = {}
    gen_functionals(gml, out)
    gen_layers(gml, out)
    gen_nets(gml, out)
    np.savez_compressed(os.path.join(OUT, "attention_cases.npz"), **out)
    print("attention_cases.npz:", len(out), "arrays")
