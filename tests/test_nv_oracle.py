"""The node-variant filter's fp64 restatement (oracle/nv_oracle.py) against the reference's stored results, its copyNodes
search against the package's and against graphtools_sparse.compute_neighborhood, and its componentwise bound itself.
CPU only.

The bound tests follow tests/test_ev_oracle.py: an emulated correct fp32 kernel (float32 hops, float32 products and sums in
a shuffled order) must pass nv_envelope, and six emulated wrong kernels must fail it by a wide margin, at the shapes of
the GPU dispatch cases in tests/test_nv_dispatch.py."""
import os

import numpy as np
import pytest
import scipy.sparse as sp

import lsigf_oracle as orc
import nv_oracle as nvo

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "nvgf_cases.npz"))
NVGF_TAGS = sorted({k.split("_")[1] for k in GOLD.files if k.startswith("nvgf_")})
LAYER_TAGS = sorted({k.split("_")[1] for k in GOLD.files if k.startswith("nvl_")})


def _rel(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def _S(prefix):
    return [sp.csr_matrix(S) for S in GOLD[prefix + "S"]]


def test_fixture_set_is_complete():
    assert NVGF_TAGS == ["e1k1", "e1k3", "e2k1", "e2k3", "e2k3fn"]
    assert LAYER_TAGS == ["meq", "mgt", "mlt", "mlt2", "nin"]
    kinds = {(int(GOLD["nvgf_%s_meta" % t][6]), int(GOLD["nvgf_%s_meta" % t][5]), int(GOLD["nvgf_%s_meta" % t][7]))
             for t in NVGF_TAGS}
    assert {e for e, _, _ in kinds} == {1, 2} and {k for _, k, _ in kinds} == {1, 3} and {b for _, _, b in kinds} == {0, 1, 2}
    # the path with a chord at M = 4: ties and nodes several hops from any independent node
    assert list(GOLD["nvl_mlt_copyNodes"]) == [0, 1, 2, 3, 3, 0, 0, 0, 0, 0]


@pytest.mark.parametrize("tag", NVGF_TAGS)
def test_oracle_matches_reference_nvgf(tag):
    p = "nvgf_%s_" % tag
    b = GOLD[p + "b"] if p + "b" in GOLD.files else None
    N = GOLD[p + "x"].shape[2]
    y = nvo.nv_forward(GOLD[p + "h"], np.arange(N), _S(p), GOLD[p + "x"], b)
    dx, dh, db = nvo.nv_backward(GOLD[p + "h"], np.arange(N), _S(p), GOLD[p + "x"], GOLD[p + "dy"],
                                 None if b is None else b.shape)
    assert _rel(y, GOLD[p + "y"]) < 1e-12
    assert _rel(dx, GOLD[p + "dx"]) < 1e-12
    assert _rel(dh, GOLD[p + "dh"]) < 1e-12
    if b is not None:
        assert _rel(db, GOLD[p + "db"]) < 1e-12


@pytest.mark.parametrize("tag", LAYER_TAGS)
def test_oracle_matches_reference_layer(tag):
    """NodeVariantGF: weight [F,E,K,G,M] read through copyNodes; Nin < N pads x with zeros and keeps Nin outputs."""
    p = "nvl_%s_" % tag
    seed, N, B, G, F, K, M, E, bias, Nin = (int(v) for v in GOLD[p + "meta"])
    copy = GOLD[p + "copyNodes"]
    assert list(nvo.copy_nodes_search(_S(p), M)) == list(copy)
    h = GOLD[p + "p_weight"]
    b = GOLD[p + "p_bias"] if bias else None
    x = np.concatenate((GOLD[p + "x"], np.zeros((B, G, N - Nin))), axis=2)
    dy = np.concatenate((GOLD[p + "dy"], np.zeros((B, F, N - Nin))), axis=2)
    y = nvo.nv_forward(h, copy, _S(p), x, b)
    dx, dh, db = nvo.nv_backward(h, copy, _S(p), x, dy, None if b is None else b.shape)
    assert _rel(y[:, :, :Nin], GOLD[p + "y"]) < 1e-12
    assert _rel(dx[:, :, :Nin], GOLD[p + "dx"]) < 1e-12
    assert _rel(dh, GOLD[p + "g_weight"]) < 1e-12
    if bias:
        assert _rel(db, GOLD[p + "g_bias"]) < 1e-12
    if M > N:                                 # taps no node reads get no gradient
        assert not np.any(dh[..., N:])


# ------------------------------------------------------------------------------------------------------- copyNodes
def _connected(rng, N, deg, directed_extra=True):
    """A random graph that contains the undirected path 0 - ... - N-1 relabelled by a permutation, plus random entries."""
    perm = rng.permutation(N)
    rows = np.concatenate((perm[:-1], perm[1:]))
    cols = np.concatenate((perm[1:], perm[:-1]))
    if directed_extra:
        r = rng.integers(0, N, N * deg)
        c = rng.integers(0, N, N * deg)
        rows, cols = np.concatenate((rows, r)), np.concatenate((cols, c))
    vals = rng.standard_normal(rows.size)
    vals[vals == 0] = 1.0
    m = sp.csr_matrix((vals, (rows, cols)), shape=(N, N))
    m.sum_duplicates()
    return m


def _brute_force(S_list, M):
    """The reference's procedure on the CSR routine: compute_neighborhood(S, k, nb=M) for k = 1, 2, ... until every node
    has an independent node in its neighbourhood, then min (graphML.py:2413-2459)."""
    import gnn_b200
    N = S_list[0].shape[0]
    if M >= N:
        return list(range(N))
    lists = gnn_b200.graphtools_sparse.compute_neighborhood(S_list, 1, nb=M)
    k = 1
    while any(len(lists[n]) == 0 for n in range(N)):
        k += 1
        more = gnn_b200.graphtools_sparse.compute_neighborhood(S_list, k, nb=M)
        lists = [lists[n] if lists[n] else more[n] for n in range(N)]
    return list(range(M)) + [min(lists[n]) for n in range(M, N)]


@pytest.mark.parametrize("seed,N,deg,M,E", [(1, 40, 1, 3, 1), (2, 60, 2, 1, 1), (3, 50, 1, 7, 2), (4, 30, 0, 5, 1),
                                            (5, 45, 3, 45, 1), (6, 20, 1, 30, 2), (7, 80, 1, 12, 1)])
def test_copy_nodes_equals_brute_force_neighbourhoods(seed, N, deg, M, E):
    import gnn_b200
    rng = np.random.default_rng(seed)
    mats = [_connected(rng, N, deg) for _ in range(E)]
    ref = _brute_force(mats, M)
    got = gnn_b200.copy_nodes(gnn_b200.SparseGSO.from_scipy(mats), M)
    assert list(got) == ref
    assert list(nvo.copy_nodes_search(mats, M)) == ref
    dense = np.stack([m.toarray() for m in mats])
    import torch
    assert list(gnn_b200.copy_nodes(torch.tensor(dense), M)) == ref


def test_copy_nodes_matches_every_fixture():
    import gnn_b200
    import torch
    for tag in LAYER_TAGS:
        p = "nvl_%s_" % tag
        M = int(GOLD[p + "meta"][6])
        assert list(gnn_b200.copy_nodes(torch.tensor(GOLD[p + "S"]), M)) == list(GOLD[p + "copyNodes"]), tag
    for name, M in (("copy0", 5), ("copy3", 6)):
        assert list(gnn_b200.copy_nodes(torch.tensor(GOLD["nvgnn_S"])[None], M)) == list(GOLD["nvgnn_" + name])


def test_unreachable_node_raises():
    """Node 5 has no out-edge towards the independent nodes (the reference's search never ends there)."""
    import gnn_b200
    import torch
    N = 8
    S = np.zeros((1, N, N))
    for i in range(4):
        S[0, i, i + 1] = S[0, i + 1, i] = 0.5
    S[0, 5, 6] = S[0, 6, 5] = 0.5             # nodes 5, 6 form their own component
    S[0, 7, 0] = 0.5                          # 7 -> 0 only: reachable
    with pytest.raises(ValueError, match=r"2 node\(s\).*M = 2.*: 5, 6"):
        gnn_b200.copy_nodes(torch.tensor(S), 2)
    layer = gnn_b200.NodeVariantGF(1, 1, 2, 2)
    with pytest.raises(ValueError, match="cannot reach"):
        layer.addGSO(torch.tensor(S))
    assert list(gnn_b200.copy_nodes(torch.tensor(S), 8)) == list(range(8))


# ------------------------------------------------------------------------------------------------ the bound itself
def _problem(N, B, G, F, K, E, M, bias, seed, dtype=np.float32, graph_deg=6):
    rng = np.random.default_rng(seed)
    mats = []
    for _ in range(E):
        m = sp.random(N, N, density=graph_deg / N, format="csr", random_state=rng, data_rvs=rng.standard_normal)
        m = m / max(abs(m).sum(axis=1).max(), 1.0)
        mats.append(sp.csr_matrix(m.astype(dtype).astype(np.float64)))
    r = lambda shape: orc.biased_uniform(rng, shape).astype(dtype).astype(np.float64)   # noqa: E731
    copy = rng.integers(0, M, N) if M < N else np.arange(N)
    h, x, dy = r((F, E, K, G, M)), r((B, G, N)), r((B, F, N))
    b = None if bias is None else r((F, 1) if bias == "F1" else (F, N))
    return mats, h, copy, x, b, dy


def _emulate_fp32(mats, h, copy, x, b, dy, rng):
    """A correct fp32 kernel: float32 hops (scipy float32 CSR), float32 products, float32 sums in a shuffled order."""
    f32 = np.float32
    F, E, K, G, M = h.shape
    B, _, N = x.shape
    T = 1 + E * (K - 1)
    St = [sp.csr_matrix(m.T, dtype=f32) for m in mats]
    Sb = [sp.csr_matrix(m, dtype=f32) for m in mats]
    X = np.ascontiguousarray(np.transpose(x, (2, 0, 1)).reshape(N, B * G)).astype(f32)
    Z = [X]
    for e in range(E):
        z = X
        for _ in range(1, K):
            z = (St[e] @ z).astype(f32)
            Z.append(z)
    W = np.zeros((M, T, G, F), f32)
    W[:, 0] = np.transpose(h[:, :, 0].astype(f32).sum(axis=1, dtype=f32), (2, 1, 0))
    for e in range(E):
        for k in range(1, K):
            W[:, 1 + e * (K - 1) + k - 1] = np.transpose(h[:, e, k], (2, 1, 0)).astype(f32)
    Wn = W[copy]
    y = np.zeros((N, B, F), f32)
    for t, g in rng.permutation([(t, g) for t in range(T) for g in range(G)]):
        y += Z[t].reshape(N, B, G)[:, :, g, None] * Wn[:, t, g, None, :]
    if b is not None:
        y += (b.astype(f32).T[:, None, :] if b.shape[1] > 1 else b[:, 0].astype(f32)[None, None, :])
    dyn = np.transpose(dy, (2, 0, 1)).astype(f32)                          # [N, B, F]

    def dz(t):
        out = np.zeros((N, B, G), f32)
        for f in rng.permutation(F):
            out += dyn[:, :, f, None] * Wn[:, t, None, :, f]
        return out.reshape(N, B * G)
    dx = dz(0)
    for e in range(E):
        if K == 1:
            break
        acc = dz(1 + e * (K - 1) + K - 2)
        for k in range(K - 2, 0, -1):
            acc = ((Sb[e] @ acc).astype(f32) + dz(1 + e * (K - 1) + k - 1)).astype(f32)
        dx = (dx + (Sb[e] @ acc).astype(f32)).astype(f32)
    dW = np.zeros((M, T, G, F), f32)
    order = rng.permutation(N * B)
    for t in range(T):
        prod = Z[t].reshape(N * B, G)[:, :, None] * dyn.reshape(N * B, F)[:, None, :]
        np.add.at(dW[:, t], np.repeat(copy, B)[order], prod[order])
    dh = np.zeros((F, E, K, G, M), f32)
    for e in range(E):
        dh[:, e, 0] = np.transpose(dW[:, 0], (2, 1, 0))
        for k in range(1, K):
            dh[:, e, k] = np.transpose(dW[:, 1 + e * (K - 1) + k - 1], (2, 1, 0))
    return (np.transpose(y, (1, 2, 0)), np.transpose(dx.reshape(N, B, G), (1, 2, 0)), dh)


# the shapes of the GPU dispatch rows (tests/test_nv_dispatch.py, _nv_rows)
SHAPES = {"f32-B8-G9-F11": (3000, 8, 9, 11, 3, 1, 300, "F1"),
          "f32-B33-G17-F5-E2": (3000, 33, 17, 5, 3, 2, 3000, "FN"),
          "f32-B1-G13-F7-K4": (3000, 1, 13, 7, 4, 2, 700, "F1")}


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_emulated_fp32_kernel_passes(name):
    N, B, G, F, K, E, M, bias = SHAPES[name]
    mats, h, copy, x, b, dy = _problem(N, B, G, F, K, E, M, bias, seed=len(name))
    env = nvo.nv_envelope(h, copy, mats, x, b, dy, np.float32)
    y, dx, dh = _emulate_fp32(mats, h, copy, x, b, dy, np.random.default_rng(3))
    ry = nvo.nv_forward(h, copy, mats, x, b)
    rdx, rdh, _ = nvo.nv_backward(h, copy, mats, x, dy, None if b is None else b.shape)
    for out, ref, bound in ((y, ry, env["y"]), (dx, rdx, env["dx"]), (dh, rdh, env["dh"])):
        v = orc.bound_violation(out, ref, bound)
        assert 0 < v <= 0.5, v


def _wrong_margin(kind):
    """Error / bound of one emulated wrong kernel (the fp64 oracle on altered inputs or outputs, rounded to the dtype of
    the GPU case that runs that branch)."""
    if kind == "tap_chunk":                   # M = 1 at N > 20 000 (fp64 row): pieces of 32 members
        N, B, G, F, K, E, M, bias, dt = 24000, 2, 3, 5, 3, 1, 1, "F1", np.float64
    else:
        N, B, G, F, K, E, M, bias, dt = 3000, 8, 9, 11, 3, 2, 300, ("FN" if kind == "bias_as_F" else "F1"), np.float32
    mats, h, copy, x, b, dy = _problem(N, B, G, F, K, E, M, bias, seed=11, dtype=dt)
    env = nvo.nv_envelope(h, copy, mats, x, b, dy, dt)
    if kind == "neighbour_tap":
        n = int(np.nonzero(copy != copy[np.arange(N) + 1 - 2 * (np.arange(N) == N - 1)])[0][0])
        c2 = copy.copy()
        c2[n] = copy[n + 1]
        return orc.bound_violation(nvo.nv_forward(h, c2, mats, x, b), nvo.nv_forward(h, copy, mats, x, b), env["y"])
    if kind == "k0_not_merged":
        h2 = h.copy()
        h2[:, 1:, 0] = 0.0
        return orc.bound_violation(nvo.nv_forward(h2, copy, mats, x, b), nvo.nv_forward(h, copy, mats, x, b), env["y"])
    if kind == "lanes_swapped":
        y = nvo.nv_forward(h, copy, mats, x, b)
        return orc.bound_violation(y[[1, 0] + list(range(2, B))], y, env["y"])
    if kind == "bias_as_F":
        return orc.bound_violation(nvo.nv_forward(h, copy, mats, x, np.repeat(b[:, :1], N, 1)),
                                   nvo.nv_forward(h, copy, mats, x, b), env["y"])
    if kind == "horner_skip":               # chain e = 0 loses its dz_{0,1} add: dx misses S_0 dz_{0,1}
        ref, _, _ = nvo.nv_backward(h, copy, mats, x, dy)
        dz1 = np.einsum("fgn,bfn->ngb", h[:, 0, 1][..., copy], dy)        # [N, G, B]
        lost = mats[0] @ np.transpose(dz1, (0, 2, 1)).reshape(N, B * G)
        return orc.bound_violation(ref - np.transpose(lost.reshape(N, B, G), (1, 2, 0)), ref, env["dx"])
    if kind == "tap_chunk":
        _, ref, _ = nvo.nv_backward(h, copy, mats, x, dy)
        keep = np.ones(N, bool)
        keep[31] = False                      # the last member of the first piece of 32
        dy2 = dy * keep[None, None, :]
        _, wrong, _ = nvo.nv_backward(h, copy, mats, x, dy2)
        return orc.bound_violation(wrong, ref, env["dh"])
    raise ValueError(kind)


WRONG = ["neighbour_tap", "k0_not_merged", "tap_chunk", "horner_skip", "lanes_swapped", "bias_as_F"]


@pytest.mark.parametrize("kind", WRONG)
def test_emulated_wrong_kernel_fails_by_a_wide_margin(kind):
    v = _wrong_margin(kind)
    print("%s: %.3g x the bound" % (kind, v))
    assert v > 100.0, (kind, v)


# ------------------------------------------------------------------------------------------------------ the C ABI
def test_cabi_rejects_bad_arguments_before_any_cuda_call():
    """Every call below fails its argument checks before the library touches the device, so this holds on a machine
    without a GPU."""
    import ctypes
    import gnn_b200
    lib = gnn_b200._cabi.load()
    EINVAL, EUNSUPPORTED = -1, -2
    p = ctypes.c_void_p(0x1000)               # never dereferenced: the checks fail first
    assert lib.b200gf_nv_pack_taps(0, None, p, 2, 1, 2, 2, 3, None) == EINVAL
    assert lib.b200gf_nv_pack_taps(0, p, p, 2, 1, 0, 2, 3, None) == EINVAL        # K = 0
    assert lib.b200gf_nv_pack_taps(0, p, p, 2, 1, 2, 2, 0, None) == EINVAL        # M = 0
    assert lib.b200gf_nv_pack_taps(7, p, p, 2, 1, 2, 2, 3, None) == EUNSUPPORTED  # unknown dtype
    assert lib.b200gf_nv_workspace_bytes(None, 1, 1, 1, 1, 1, 1) == 0
    # no plan
    assert lib.b200gf_nv_forward(None, p, 4, p, p, 3, None, 0, p, 4, None, 0, 1, 4, 4, 2, None) == EINVAL
    assert lib.b200gf_nv_backward(None, p, 4, p, 4, p, p, 3, p, p, p, 4, p, None, 0, p, 1 << 20, 1, 4, 4, 2,
                                  None) == EINVAL
