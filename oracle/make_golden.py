"""Generate tests/golden/*.npz by running the UNMODIFIED reference (alegnn).

TEST INFRASTRUCTURE.  Run once (`B200GF_REFERENCE_ROOT=<alegnn checkout> python oracle/make_golden.py`); the fixtures are
committed so that the tests need no reference checkout.  Every array in a fixture is either a seeded input or an
output of the reference's own code:

  lsigf_cases.npz   – `alegnn.utils.graphML.LSIGF` (graphML.py:83-176) forward in fp64 and its autograd
                      gradients (dh, dx, db) for a sweep of shapes (E>1, K in {1,2,3,5}, bias None / Fx1 / FxN,
                      non-symmetric GSOs), plus the reference's own fp32 forward (its noise floor).
  graphfilter_cases.npz – `alegnn.utils.graphML.GraphFilter` (graphML.py:2036-2155) incl. the N_in < N
                      zero-pad / truncate path (:2131-2143).
  layer_cases.npz   – the layer the selection architectures stack (architectures.py:274-296):
                      `GraphFilter` -> `nn.ReLU` -> `MaxPoolLocal` (graphML.py:1968-2019), forward + all gradients and
                      the reference's neighbourhood matrix.
  selectiongnn_cfg1.npz – BASELINE.json configs[0]: reference `Graph('SBM',50,...)`, `S = W/lambda_max`,
                      `SelectionGNN([1,32],[5],...)` (architectures.py:166-180) forward + backward in fp64;
                      state_dict, input batch, output and the parameter gradients.
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

# (seed, N, B, G, F, K, E, avg_deg, bias, symmetric)
LSIGF_CASES = [
    (101, 12, 2, 3, 4, 3, 1, 4, "F1", False),
    (102, 17, 3, 2, 5, 5, 2, 5, "FN", False),
    (103, 9, 1, 1, 6, 1, 1, 3, "F1", False),     # K = 1: no hops
    (104, 20, 4, 4, 4, 2, 3, 6, None, False),
    (105, 33, 2, 8, 8, 5, 1, 8, "F1", True),
    (106, 50, 5, 1, 32, 5, 1, 10, "F1", True),   # cfg1-shaped layer
    (107, 64, 2, 16, 12, 4, 2, 7, "FN", False),
    (108, 41, 3, 5, 7, 3, 1, 41, "F1", False),   # fully dense GSO
]

GF_CASES = [
    # (seed, N, Nin, B, G, F, K, E, bias)
    (201, 24, 24, 3, 2, 4, 3, 1, True),
    (202, 24, 15, 2, 3, 5, 4, 2, True),          # zero-pad + truncate
    (203, 30, 7, 4, 1, 3, 2, 1, False),
]


def gen_lsigf(gml):
    out = {}
    for (seed, N, B, G, F, K, E, deg, bias, sym) in LSIGF_CASES:
        c = orc.random_case(seed, N, B, G, F, K, E, deg, bias, sym)
        h = torch.tensor(c["h"], dtype=torch.float64, requires_grad=True)
        x = torch.tensor(c["x"], dtype=torch.float64, requires_grad=True)
        S = torch.tensor(c["S"], dtype=torch.float64)
        b = None if c["b"] is None else torch.tensor(c["b"], dtype=torch.float64, requires_grad=True)
        y = gml.LSIGF(h, S, x, b)
        dy = torch.tensor(c["dy"], dtype=torch.float64)
        y.backward(dy)
        y32 = gml.LSIGF(h.detach().float(), S.float(), x.detach().float(),
                        None if b is None else b.detach().float())
        key = "c%d" % seed
        out[key + "_meta"] = np.array([seed, N, B, G, F, K, E, deg, {"F1": 1, "FN": 2, None: 0}[bias], int(sym)])
        for name, val in (("h", c["h"]), ("S", c["S"]), ("x", c["x"]), ("dy", c["dy"])):
            out[key + "_" + name] = val
        if c["b"] is not None:
            out[key + "_b"] = c["b"]
            out[key + "_db"] = b.grad.numpy()
        out[key + "_y"] = y.detach().numpy()
        out[key + "_y32"] = y32.numpy()
        out[key + "_dh"] = h.grad.numpy()
        out[key + "_dx"] = x.grad.numpy()
    np.savez_compressed(os.path.join(OUT, "lsigf_cases.npz"), **out)
    print("lsigf_cases.npz:", len(LSIGF_CASES), "cases")


def gen_graphfilter(gml):
    out = {}
    for (seed, N, Nin, B, G, F, K, E, bias) in GF_CASES:
        rng = np.random.default_rng(seed)
        S = orc.random_sparse_gso(rng, N, 5, E)
        x = rng.standard_normal((B, G, Nin))
        torch.manual_seed(seed)
        layer = gml.GraphFilter(G, F, K, E, bias).double()
        layer.addGSO(torch.tensor(S))
        xt = torch.tensor(x, requires_grad=True)
        y = layer(xt)
        dy = rng.standard_normal(tuple(y.shape))
        y.backward(torch.tensor(dy))
        key = "g%d" % seed
        out[key + "_meta"] = np.array([seed, N, Nin, B, G, F, K, E, int(bias)])
        out[key + "_S"] = S
        out[key + "_x"] = x
        out[key + "_dy"] = dy
        out[key + "_weight"] = layer.weight.detach().numpy()
        out[key + "_dweight"] = layer.weight.grad.numpy()
        if bias:
            out[key + "_bias"] = layer.bias.detach().numpy()
            out[key + "_dbias"] = layer.bias.grad.numpy()
        out[key + "_y"] = y.detach().numpy()
        out[key + "_dx"] = xt.grad.numpy()
    np.savez_compressed(os.path.join(OUT, "graphfilter_cases.npz"), **out)
    print("graphfilter_cases.npz:", len(GF_CASES), "cases")


def gen_selectiongnn_cfg1(gml):
    import torch.nn as nn
    import alegnn.utils.graphTools as graphTools
    import alegnn.modules.architectures as archit
    np.random.seed(0)
    torch.manual_seed(0)
    torch.set_default_dtype(torch.float64)
    try:
        G = graphTools.Graph("SBM", 50, {"nCommunities": 5, "probIntra": 0.8, "probInter": 0.2})
        G.computeGFT()
        S = G.W / np.max(np.real(G.E))  # examples/sourceLocGNN.py:752
        net = archit.SelectionGNN([1, 32], [5], True, nn.ReLU, [50], gml.NoPool, [1], [5], S)
        x = np.random.randn(20, 1, 50)
        xt = torch.tensor(x, requires_grad=True)
        y = net(xt)
        dy = np.random.randn(*y.shape)
        y.backward(torch.tensor(dy))
        out = {"S": S, "x": x, "dy": dy, "y": y.detach().numpy(), "dx": xt.grad.numpy()}
        for k, v in net.state_dict().items():
            out["sd_" + k] = v.numpy()
        for k, p in net.named_parameters():
            out["grad_" + k] = p.grad.numpy()
    finally:
        torch.set_default_dtype(torch.float32)
    np.savez_compressed(os.path.join(OUT, "selectiongnn_cfg1.npz"), **out)
    print("selectiongnn_cfg1.npz: keys", sorted(out.keys()))


# GraphFilter -> nn.ReLU -> MaxPoolLocal, the layer of the selection architectures (architectures.py:274-296)
LAYER_CASES = [
    # (seed, N, Nout, B, G, F, K, E, hops)
    (301, 30, 30, 2, 3, 5, 3, 1, 1),
    (302, 40, 17, 3, 4, 6, 4, 2, 2),
    (303, 25, 9, 1, 2, 8, 2, 1, 3),
]


def gen_layer(gml):
    import torch.nn as nn
    out = {}
    for (seed, N, Nout, B, G, F, K, E, hops) in LAYER_CASES:
        rng = np.random.default_rng(seed)
        S = np.abs(orc.random_sparse_gso(rng, N, 4, E, symmetric=True))
        torch.manual_seed(seed)
        gf = gml.GraphFilter(G, F, K, E, True).double()
        gf.addGSO(torch.tensor(S))
        pool = gml.MaxPoolLocal(N, Nout, hops)
        pool.addGSO(torch.tensor(S))
        net = nn.Sequential(gf, nn.ReLU(), pool)
        x = torch.tensor(rng.standard_normal((B, G, N)), requires_grad=True)
        y = net(x)
        dy = torch.tensor(rng.standard_normal(tuple(y.shape)))
        y.backward(dy)
        c = "l%d" % seed
        out.update({c + "_S": S, c + "_x": x.detach().numpy(), c + "_dy": dy.numpy(), c + "_y": y.detach().numpy(),
                    c + "_weight": gf.weight.detach().numpy(), c + "_bias": gf.bias.detach().numpy(),
                    c + "_dx": x.grad.numpy(), c + "_dweight": gf.weight.grad.numpy(), c + "_dbias": gf.bias.grad.numpy(),
                    c + "_neighborhood": pool.neighborhood.numpy(), c + "_meta": np.array([N, Nout, B, G, F, K, E, hops])})
    np.savez_compressed(os.path.join(OUT, "layer_cases.npz"), **out)
    print("layer_cases.npz:", len(LAYER_CASES), "cases")


def gen_evgf(gml):
    """EVGF (graphML.py:389-488) and EdgeVariantGF (graphML.py:2511-2712), full (M = N) and hybrid (M < N), fp64."""
    out = {}
    # (a) the functional on arbitrary masked filter matrices
    rng = np.random.default_rng(301)
    F, E, K, G, N, B = 3, 2, 3, 2, 10, 2
    mask = (rng.random((1, E, 1, 1, N, N)) < 0.3) | np.eye(N, dtype=bool)[None, None, None, None]
    Phi = rng.standard_normal((F, E, K, G, N, N)) * mask
    x = rng.standard_normal((B, G, N))
    b = rng.standard_normal((F, 1))
    Pt = torch.tensor(Phi, requires_grad=True)
    xt = torch.tensor(x, requires_grad=True)
    bt = torch.tensor(b, requires_grad=True)
    y = gml.EVGF(Pt, xt, bt)
    dy = rng.standard_normal(tuple(y.shape))
    y.backward(torch.tensor(dy))
    out.update({"f_Phi": Phi, "f_x": x, "f_b": b, "f_dy": dy, "f_y": y.detach().numpy(),
                "f_dPhi": Pt.grad.numpy() * mask, "f_dx": xt.grad.numpy(), "f_db": bt.grad.numpy()})
    # (b) the layer: full and hybrid
    for tag, (N, M, E, K, G, F, B, Nin) in {"full": (9, 9, 1, 3, 2, 3, 2, 9), "hyb": (12, 5, 2, 3, 3, 2, 3, 10)}.items():
        rng = np.random.default_rng(310 + N)
        S = orc.random_sparse_gso(rng, N, 3, E)
        torch.manual_seed(N)
        layer = gml.EdgeVariantGF(G, F, K, M, N, E, True).double()
        with torch.no_grad():  # larger weights than the 1/sqrt(GKN) init so that the comparison is not all bias
            layer.weightEV.mul_(5.0)
        layer.addGSO(torch.tensor(S))
        x = rng.standard_normal((B, G, Nin))
        xt = torch.tensor(x, requires_grad=True)
        y = layer(xt)
        dy = rng.standard_normal(tuple(y.shape))
        y.backward(torch.tensor(dy))
        out[tag + "_meta"] = np.array([N, M, E, K, G, F, B, Nin])
        out[tag + "_S"] = S
        out[tag + "_x"] = x
        out[tag + "_dy"] = dy
        out[tag + "_y"] = y.detach().numpy()
        out[tag + "_dx"] = xt.grad.numpy()
        for name, p in layer.named_parameters():
            out[tag + "_p_" + name] = p.detach().numpy()
            out[tag + "_g_" + name] = p.grad.numpy()
    np.savez_compressed(os.path.join(OUT, "evgf_cases.npz"), **out)
    print("evgf_cases.npz:", sorted(k for k in out if k.endswith("_y")))


def gen_grnn(gml):
    """GatedGRNN (graphML.py:1292-1527) through the reference's HiddenState / TimeGatedHiddenState /
    NodeGatedHiddenState layers (graphML.py:3540-4031), fp64: trajectory, input gradient and parameter gradients."""
    out = {}
    cases = {"plain": (gml.HiddenState, 14, 3, 5, 2, 4, 3, 2, True),      # (layer, N, B, T, F, H, K, E, bias)
             "nobias": (gml.HiddenState, 11, 2, 4, 3, 3, 2, 1, False),
             "time": (gml.TimeGatedHiddenState, 12, 3, 4, 2, 3, 3, 1, True),
             "node": (gml.NodeGatedHiddenState, 13, 2, 5, 2, 4, 3, 1, True)}
    for tag, (cls, N, B, T, F, H, K, E, bias) in cases.items():
        rng = np.random.default_rng(400 + N)
        S = orc.random_sparse_gso(rng, N, 4, E)
        torch.manual_seed(N)
        layer = cls(F, H, K, E=E, bias=bias).double()
        layer.addGSO(torch.tensor(S))
        layer.double()                                     # the gate maps are created inside addGSO
        x = rng.standard_normal((B, T, F, N))
        z0 = rng.standard_normal((B, H, N))
        xt = torch.tensor(x, requires_grad=True)
        z0t = torch.tensor(z0, requires_grad=True)
        z, zT = layer(xt, z0t)
        dz = rng.standard_normal(tuple(z.shape))
        z.backward(torch.tensor(dz))
        out[tag + "_meta"] = np.array([N, B, T, F, H, K, E, int(bias)])
        out[tag + "_S"] = S
        out[tag + "_x"] = x
        out[tag + "_z0"] = z0
        out[tag + "_dz"] = dz
        out[tag + "_z"] = z.detach().numpy()
        out[tag + "_zT"] = zT.detach().numpy()
        out[tag + "_dx"] = xt.grad.numpy()
        out[tag + "_dz0"] = z0t.grad.numpy()
        for name, p in layer.named_parameters():
            out[tag + "_p_" + name] = p.detach().numpy()
            out[tag + "_g_" + name] = p.grad.numpy()
    np.savez_compressed(os.path.join(OUT, "grnn_cases.npz"), **out)
    print("grnn_cases.npz:", sorted(k for k in out if k.endswith("_z")))


def gen_lsigf_db(gml):
    """LSIGF_DB (graphML.py:977-1094) and GraphFilter_DB (graphML.py:3278-3393): a different GSO per batch element
    and time step, unit delay per tap; fp64 forward and autograd gradients."""
    out = {}
    # (tag, B, T, N, G, F, K, E, bias)
    cases = [("a", 3, 5, 7, 2, 3, 3, 1, "F1"), ("b", 2, 4, 6, 3, 2, 4, 2, "FN"), ("c", 2, 1, 5, 2, 2, 3, 1, "F1"),
             ("d", 1, 6, 8, 1, 4, 1, 1, None), ("e", 2, 3, 9, 4, 5, 6, 1, "F1")]      # e: more taps than time steps
    for (tag, B, T, N, G, F, K, E, bias) in cases:
        rng = np.random.default_rng(500 + ord(tag))
        S = np.stack([np.stack([orc.random_sparse_gso(rng, N, 3, E) for _ in range(T)]) for _ in range(B)])  # B,T,E,N,N
        x = rng.standard_normal((B, T, G, N))
        bound = 1.0 / np.sqrt(G * K)
        h = rng.uniform(-bound, bound, (F, E, K, G))
        b = None if bias is None else rng.uniform(-bound, bound, (F, 1 if bias == "F1" else N))
        ht, xt = torch.tensor(h, requires_grad=True), torch.tensor(x, requires_grad=True)
        bt = None if b is None else torch.tensor(b, requires_grad=True)
        y = gml.LSIGF_DB(ht, torch.tensor(S), xt, bt)
        dy = rng.standard_normal(tuple(y.shape))
        y.backward(torch.tensor(dy))
        key = "f" + tag
        out[key + "_meta"] = np.array([B, T, N, G, F, K, E, {"F1": 1, "FN": 2, None: 0}[bias]])
        for name, val in (("S", S), ("x", x), ("h", h), ("dy", dy), ("y", y.detach().numpy()),
                          ("dh", ht.grad.numpy()), ("dx", xt.grad.numpy())):
            out[key + "_" + name] = val
        if b is not None:
            out[key + "_b"] = b
            out[key + "_db"] = bt.grad.numpy()
    # the layer
    B, T, N, G, F, K, E = 3, 4, 6, 2, 3, 3, 2
    rng = np.random.default_rng(560)
    S = np.stack([np.stack([orc.random_sparse_gso(rng, N, 3, E) for _ in range(T)]) for _ in range(B)])
    torch.manual_seed(560)
    layer = gml.GraphFilter_DB(G, F, K, E, True).double()
    layer.addGSO(torch.tensor(S))
    x = rng.standard_normal((B, T, G, N))
    xt = torch.tensor(x, requires_grad=True)
    y = layer(xt)
    dy = rng.standard_normal(tuple(y.shape))
    y.backward(torch.tensor(dy))
    out.update({"layer_meta": np.array([B, T, N, G, F, K, E]), "layer_S": S, "layer_x": x, "layer_dy": dy,
                "layer_y": y.detach().numpy(), "layer_dx": xt.grad.numpy(),
                "layer_weight": layer.weight.detach().numpy(), "layer_bias": layer.bias.detach().numpy(),
                "layer_dweight": layer.weight.grad.numpy(), "layer_dbias": layer.bias.grad.numpy()})
    np.savez_compressed(os.path.join(OUT, "lsigf_db_cases.npz"), **out)
    print("lsigf_db_cases.npz:", sorted(k for k in out if k.endswith("_y")))


def gen_grnn_db(gml):
    """GRNN_DB (graphML.py:1096-1290) and HiddenState_DB (graphML.py:3395-3538): hidden-state recursion on a GSO that
    changes with the batch element and the time step; fp64 forward and autograd gradients of every input.
    The reference builds its K x (K-1) selection matrix with the default dtype (:1176), so it runs in fp64 only with the
    default dtype set accordingly."""
    out = {}
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        # (tag, B, T, N, F, H, K, E, bias, sigma)
        cases = [("a", 3, 5, 7, 2, 3, 3, 1, True, "tanh"), ("b", 2, 6, 6, 3, 2, 4, 2, True, "tanh"),
                 ("c", 2, 1, 5, 2, 2, 3, 1, True, "tanh"),       # a single time step: no shift at all
                 ("d", 1, 6, 8, 1, 4, 1, 1, False, "relu"),      # K = 1: no delay line
                 ("e", 2, 3, 9, 4, 5, 6, 1, True, "tanh"),       # more taps than time steps
                 ("f", 2, 7, 6, 2, 3, 2, 2, False, "relu")]      # K = 2, E = 2
        for (tag, B, T, N, F, H, K, E, bias, sg) in cases:
            rng = np.random.default_rng(700 + ord(tag))
            S = np.stack([np.stack([orc.random_sparse_gso(rng, N, 3, E) for _ in range(T)]) for _ in range(B)])
            x = rng.standard_normal((B, T, F, N))
            z0 = rng.standard_normal((B, H, N))
            a = rng.uniform(-0.5, 0.5, (H, E, K, F))
            b = rng.uniform(-0.5, 0.5, (H, E, K, H))
            xb = rng.uniform(-0.5, 0.5, (H, 1)) if bias else None
            zb = rng.uniform(-0.5, 0.5, (H, 1)) if bias else None
            ts = [torch.tensor(v, requires_grad=True) for v in (a, b, x, z0)]
            bs = [None if v is None else torch.tensor(v, requires_grad=True) for v in (xb, zb)]
            z = gml.GRNN_DB(ts[0], ts[1], torch.tensor(S), ts[2], ts[3], getattr(torch, sg), bs[0], bs[1])
            dz = rng.standard_normal(tuple(z.shape))
            z.backward(torch.tensor(dz))
            key = "g" + tag
            out[key + "_meta"] = np.array([B, T, N, F, H, K, E, int(bias), {"tanh": 0, "relu": 1}[sg]])
            for name, val in (("S", S), ("x", x), ("z0", z0), ("a", a), ("b", b), ("dz", dz), ("z", z.detach().numpy()),
                              ("da", ts[0].grad.numpy()), ("db", ts[1].grad.numpy()), ("dx", ts[2].grad.numpy()),
                              ("dz0", ts[3].grad.numpy())):
                out[key + "_" + name] = val
            if bias:
                out[key + "_xb"], out[key + "_zb"] = xb, zb
                out[key + "_dxb"], out[key + "_dzb"] = bs[0].grad.numpy(), bs[1].grad.numpy()
        # the layer
        B, T, N, F, H, K, E = 3, 5, 6, 2, 4, 3, 2
        rng = np.random.default_rng(760)
        S = np.stack([np.stack([orc.random_sparse_gso(rng, N, 3, E) for _ in range(T)]) for _ in range(B)])
        torch.manual_seed(760)
        layer = gml.HiddenState_DB(F, H, K, torch.tanh, E, True).double()
        layer.addGSO(torch.tensor(S))
        x, z0 = rng.standard_normal((B, T, F, N)), rng.standard_normal((B, H, N))
        xt, zt = torch.tensor(x, requires_grad=True), torch.tensor(z0, requires_grad=True)
        z, zT = layer(xt, zt)
        dz, dzT = rng.standard_normal(tuple(z.shape)), rng.standard_normal(tuple(zT.shape))
        ((z * torch.tensor(dz)).sum() + (zT * torch.tensor(dzT)).sum()).backward()
        out.update({"layer_meta": np.array([B, T, N, F, H, K, E]), "layer_S": S, "layer_x": x, "layer_z0": z0,
                    "layer_dz": dz, "layer_dzT": dzT, "layer_z": z.detach().numpy(), "layer_zT": zT.detach().numpy(),
                    "layer_dx": xt.grad.numpy(), "layer_dz0": zt.grad.numpy()})
        for name, prm in layer.named_parameters():
            out["layer_p_" + name] = prm.detach().numpy()
            out["layer_g_" + name] = prm.grad.numpy()
    finally:
        torch.set_default_dtype(prev)
    np.savez_compressed(os.path.join(OUT, "grnn_db_cases.npz"), **out)
    print("grnn_db_cases.npz:", sorted(k for k in out if k.endswith("_z")))


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    gml = ref_import.import_reference()
    only = set(sys.argv[1:])                               # e.g. `python oracle/make_golden.py grnn`
    for name, gen in (("lsigf", gen_lsigf), ("graphfilter", gen_graphfilter), ("selectiongnn_cfg1", gen_selectiongnn_cfg1),
                      ("evgf", gen_evgf), ("grnn", gen_grnn), ("lsigf_db", gen_lsigf_db), ("layer", gen_layer),
                      ("grnn_db", gen_grnn_db)):
        if not only or name in only:
            gen(gml)
