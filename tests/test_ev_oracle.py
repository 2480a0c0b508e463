"""CPU tests of oracle/ev_oracle.py, the fp64 restatement and error envelope the edge-variant kernels (csrc/ev.cu) are
held to in tests/test_kernel_dispatch.py, and of the argument checks of b200gf_ev_forward / b200gf_ev_backward.

* The restatement is pinned: it reproduces the reference's stored EVGF results (forward and gradients) and the
  reference layer's output with its identity k = 0 mask, and its backward matches torch autograd through dense
  scatters of w.
* The envelope separates a correct kernel from subtly wrong ones.  An emulated correct fp32 kernel (float32 products
  and sums in a shuffled order, no FMA) meets it.  Emulations of wrong kernels miss it by at least WIDE at the shapes
  the GPU cases use (rows and columns of 0 .. 129 entries, G = 9, B = 8, K = 3).  The margins, measured on the CPU
  and independent of the GPU, are listed beside WRONG: every wrong kernel misses its bound by 1.5e4x or more."""
import ctypes
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import ev_oracle as evo
import lsigf_oracle as orc

WIDE = 3.0


def _rel(a, b):
    return np.abs(np.asarray(a) - b).max() / max(np.abs(b).max(), 1e-300)


# ------------------------------------------------------------------------------------------------ pinning
@pytest.fixture(scope="module")
def z(golden_dir):
    return np.load(os.path.join(golden_dir, "evgf_cases.npz"))


def _pattern_of(Phi_e):
    """CSR pattern (rowptr, col) and row-major (rows, cols) of the entries of Phi_e [F, K, G, N, N] that are non-zero
    for some (f, k, g)."""
    m = sp.csr_matrix((np.abs(Phi_e) > 0).any(axis=(0, 1, 2)).astype(np.float64))
    m.sort_indices()
    rows = np.repeat(np.arange(m.shape[0]), np.diff(m.indptr))
    return m.indptr.astype(np.int64), m.indices.astype(np.int64), rows


def test_oracle_matches_reference_evgf_forward_and_gradients(z):
    Phi, x, b, dy = z["f_Phi"], z["f_x"], z["f_b"], z["f_dy"]
    F, E, K, G, N, _ = Phi.shape
    xT = x.transpose(1, 2, 0)
    dY = dy.transpose(1, 2, 0)                                             # [F, N, B]
    y = np.zeros((F, N, x.shape[0]))
    dx = np.zeros_like(xT)
    dPhi = np.zeros_like(Phi)
    for e in range(E):
        rowptr, col, rows = _pattern_of(Phi[:, e])
        w = Phi[:, e][..., rows, col]                                     # [F, K, G, nnz]
        y += evo.ev_forward(rowptr, col, None, w, xT)[0]
        dw, dxT, _ = evo.ev_backward(rowptr, col, None, w, xT, dY)
        dx += dxT
        dPhi[:, e][..., rows, col] = dw
    y = y.transpose(2, 0, 1) + b[None]
    assert _rel(y, orc.evgf_dense(Phi, x, b)) < 1e-12
    assert _rel(y, z["f_y"]) < 1e-12
    assert _rel(dx.transpose(2, 0, 1), z["f_dx"]) < 1e-12
    on = np.abs(Phi) > 0                                                  # the gradient on the pattern
    assert _rel(dPhi[on], z["f_dPhi"][on]) < 1e-12


def test_oracle_diag_step_matches_reference_layer(z):
    """The layer's identity k = 0 mask (graphML.py:2653-2663) is the diag form of step 0: the reference layer's output."""
    N, M, E, K, G, F, B, Nin = [int(v) for v in z["full_meta"]]
    assert M == N and E == 1 and Nin == N
    S, W, bias = z["full_S"][0], z["full_p_weightEV"][:, 0], z["full_p_bias"]
    m = sp.csr_matrix(((np.abs(S) + np.eye(N)) > 1e-9).astype(np.float64))
    m.sort_indices()
    rowptr, col = m.indptr.astype(np.int64), m.indices.astype(np.int64)
    rows = np.repeat(np.arange(N), np.diff(rowptr))
    diag = np.full(N, -1)
    diag[rows[rows == col]] = np.nonzero(rows == col)[0]
    w = W[..., rows, col]                                                 # k = 0 off-diagonal slots non-zero: unused
    Y, _ = evo.ev_forward(rowptr, col, diag, w, z["full_x"].transpose(1, 2, 0))
    assert _rel(Y.transpose(2, 0, 1) + bias[None], z["full_y"]) < 1e-12


def _small_pattern(rng, NA, diag):
    m = sp.random(NA, NA, density=0.3, format="csr", random_state=rng)
    m = sp.csr_matrix(((m != 0) + sp.eye(NA)).astype(np.float64))
    m.sort_indices()
    rowptr, col = m.indptr.astype(np.int64), m.indices.astype(np.int64)
    rows = np.repeat(np.arange(NA), np.diff(rowptr))
    if not diag:
        return rowptr, col, rows, None
    d = np.full(NA, -1)
    d[rows[rows == col]] = np.nonzero(rows == col)[0]
    d[::4] = -1                                                           # rows whose k = 0 step is zero
    return rowptr, col, rows, d


@pytest.mark.parametrize("diag", [False, True])
def test_oracle_backward_matches_autograd(diag):
    rng = np.random.default_rng(7)
    NA, B, G, F, K = 12, 3, 2, 2, 3
    rowptr, col, rows, d = _small_pattern(rng, NA, diag)
    nnz = len(col)
    w, xT, dY = rng.standard_normal((F, K, G, nnz)), rng.standard_normal((G, NA, B)), rng.standard_normal((F, NA, B))
    wt = torch.tensor(w, requires_grad=True)
    xt = torch.tensor(xT, requires_grad=True)
    r, c = torch.from_numpy(rows), torch.from_numpy(col)
    if diag:
        i0, s0 = torch.from_numpy(np.nonzero(d >= 0)[0]), torch.from_numpy(d[d >= 0])
    Ys = []
    for f in range(F):
        yf = 0
        for g in range(G):
            u = xt[g]
            for k in range(K):
                Phi = torch.zeros(NA, NA, dtype=torch.float64)
                if k == 0 and diag:
                    Phi = Phi.index_put((i0, i0), wt[f, 0, g][s0])
                else:
                    Phi = Phi.index_put((r, c), wt[f, k, g])
                u = Phi @ u
                yf = yf + u
        Ys.append(yf)
    Yt = torch.stack(Ys)
    (Yt * torch.tensor(dY)).sum().backward()
    Y, U = evo.ev_forward(rowptr, col, d, w, xT)
    dw, dxT, lam = evo.ev_backward(rowptr, col, d, w, xT, dY)
    assert _rel(Y, Yt.detach().numpy()) < 1e-12
    assert _rel(dw, wt.grad.numpy()) < 1e-12
    assert _rel(dxT, xt.grad.numpy()) < 1e-12
    assert np.array_equal(lam[K - 1], np.repeat(dY, G, axis=0))
    if diag:
        off = np.ones(nnz, bool)
        off[d[d >= 0]] = False
        assert np.all(dw[:, 0][..., off] == 0)


# ------------------------------------------------------------------------------------------------ envelope
SPECIAL = [0, 1, 3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129]


def _dispatch_like_pattern(N=300, seed=0):
    """Rows and columns of the lengths test_kernel_dispatch.py's graph has (0, 1, 3..9, 15..17, 31..33, 63..65,
    127..129), the diagonal on most rows, diag[i] = -1 on every row i % 4 == 1."""
    rng = np.random.default_rng(seed)
    lens = list(rng.integers(0, 9, N))
    lens[:len(SPECIAL)] = SPECIAL
    rows, cols = [], []
    for r, L in enumerate(lens):
        rows += [r] * L
        cols += list(rng.choice(N, size=L, replace=False))
    for i, L in enumerate(SPECIAL):
        rows += list(rng.choice(N, size=L, replace=False))
        cols += [N - 1 - i] * L
    keep = np.arange(N) % 4 != 1
    rows += list(np.arange(N)[keep])
    cols += list(np.arange(N)[keep])
    m = sp.csr_matrix((np.ones(len(rows)), (rows, cols)), shape=(N, N))
    m.sum_duplicates()
    m.sort_indices()
    rowptr, col = m.indptr.astype(np.int64), m.indices.astype(np.int64)
    rw = np.repeat(np.arange(N), np.diff(rowptr))
    d = np.full(N, -1)
    d[rw[rw == col]] = np.nonzero(rw == col)[0]
    d[1::4] = -1
    return rowptr, col, d


def _acc_f32(ptr, idx, vals, u, init, rng):
    """out[r] = init[r] + sum over r's entries it of vals[it] * u[idx[it]], float32, one rounding per product and per
    sum, entries of a row in a random order."""
    n_rows = len(ptr) - 1
    rows = np.repeat(np.arange(n_rows), np.diff(ptr))
    order = np.argsort(rows + rng.random(len(rows)), kind="stable")
    pos = np.empty(len(rows), dtype=np.int64)
    pos[order] = np.arange(len(rows)) - ptr[rows[order]]
    acc = np.array(init, dtype=np.float32)
    for p in range(int(np.diff(ptr).max(initial=0))):
        sel = np.nonzero(pos == p)[0]
        acc[rows[sel]] = acc[rows[sel]] + vals[sel, None] * u[idx[sel]]
    return acc


def _ev_f32(rowptr, col, diag, w, xT, dY, rng, bug=None):
    """The EV forward and backward computed in float32 the way a correct kernel may (shuffled order), or with `bug`."""
    w, xT, dY = (np.asarray(a, dtype=np.float32) for a in (w, xT, dY))
    F, K, G, nnz = w.shape
    _, NA, B = xT.shape
    rows = np.repeat(np.arange(NA), np.diff(rowptr))
    permT = np.argsort(col * NA + rows, kind="stable")
    rowptrT = np.concatenate([[0], np.cumsum(np.bincount(col, minlength=NA))])
    colT = rows[permT]
    on = diag >= 0 if diag is not None else None
    zero = np.zeros((NA, B), np.float32)

    def step(k, wv, u):
        if k == 0 and diag is not None and bug != "k0_whole_row":
            coef = np.zeros(NA, np.float32)
            coef[on] = wv[diag[on]]
            return coef[:, None] * u
        return _acc_f32(rowptr, col, wv, u, zero, rng)

    Y = np.zeros((F, NA, B), np.float32)
    U = np.zeros((K, F * G, NA, B), np.float32)
    for f in range(F):
        for k in range(K):
            ysum = zero.copy()
            for g in range(G):
                U[k, f * G + g] = step(k, w[f, k, g], U[k - 1, f * G + g] if k else xT[g])
                if not (bug == "g_tail" and g >= G // 8 * 8):
                    ysum = ysum + U[k, f * G + g]
            Y[f] = ysum if k == 0 else ysum + Y[f]
    if bug == "lane_swap":                                  # lanes 1 and 2 of every 4-vector
        Y[..., 1::4], Y[..., 2::4] = Y[..., 2::4].copy(), Y[..., 1::4].copy()
    dw = np.zeros((F, K, G, nnz), np.float32)
    dxT = np.zeros((G, NA, B), np.float32)
    for f in range(F):
        for g in range(G):
            fg = f * G + g
            lk = dY[f]
            for k in range(K - 1, -1, -1):
                prev = U[k - 1, fg] if k else xT[g]
                prods = lk[rows] * prev[col]
                acc = np.zeros(nnz, np.float32)
                for b in rng.permutation(B):
                    acc = acc + prods[:, b]
                if k == 0 and diag is not None:
                    live = np.zeros(nnz, bool)
                    live[diag[on]] = True
                    acc[~live] = 0
                long_rows = np.nonzero(np.diff(rowptr) >= 33)[0]
                if bug == "wgrad_drop33":
                    acc[rowptr[long_rows] + 32] = 0
                elif bug == "wgrad_dup33":
                    acc[rowptr[long_rows] + 32] = acc[rowptr[long_rows] + 31]
                dw[f, k, g] = acc
                if k == 0:
                    break
                wk = w[f, k - 1 if bug == "adjoint_wkm1" else k, g]
                lk = _acc_f32(rowptrT, colT, wk[permT], lk, zero if bug == "adjoint_no_dy" else dY[f], rng)
            if diag is not None:
                coef = np.zeros(NA, np.float32)
                coef[on] = w[f, 0, g][diag[on]]
                dxT[g] = dxT[g] + coef[:, None] * lk
            else:
                dxT[g] = _acc_f32(rowptrT, colT, w[f, 0, g][permT], lk, dxT[g], rng)
    return dict(Y=Y, dw=dw, dxT=dxT)


@pytest.fixture(scope="module")
def env_case():
    """F = 3, G = 9 (one feature in the G-tail), B = 8, K = 3, diag given, k = 0 weights non-zero on every slot."""
    rng = np.random.default_rng(11)
    rowptr, col, d = _dispatch_like_pattern()
    F, K, G, B, NA = 3, 3, 9, 8, len(rowptr) - 1
    r32 = lambda a: orc.biased_uniform(rng, a).astype(np.float32).astype(np.float64)   # noqa: E731
    w, xT, dY = r32((F, K, G, len(col))), r32((G, NA, B)), r32((F, NA, B))
    Y, _ = evo.ev_forward(rowptr, col, d, w, xT)
    dw, dxT, _ = evo.ev_backward(rowptr, col, d, w, xT, dY)
    env = evo.ev_envelope(rowptr, col, d, w, xT, dY, np.float32)
    return dict(args=(rowptr, col, d, w, xT, dY), ref=dict(Y=Y, dw=dw, dxT=dxT), env=env)


@pytest.mark.parametrize("shape", [(3, 9, 8, 3, True), (3, 17, 7, 3, False), (2, 1, 33, 4, True)],
                         ids=["G9-B8-K3-diag", "G17-B7-K3", "G1-B33-K4-diag"])
def test_envelope_accepts_correct_fp32_kernel(shape):
    F, G, B, K, diag = shape
    rng = np.random.default_rng(F + G + B + K)
    rowptr, col, d = _dispatch_like_pattern(seed=G)
    d = d if diag else None
    NA = len(rowptr) - 1
    r32 = lambda a: orc.biased_uniform(rng, a).astype(np.float32).astype(np.float64)   # noqa: E731
    w, xT, dY = r32((F, K, G, len(col))), r32((G, NA, B)), r32((F, NA, B))
    Y, _ = evo.ev_forward(rowptr, col, d, w, xT)
    dw, dxT, _ = evo.ev_backward(rowptr, col, d, w, xT, dY)
    env = evo.ev_envelope(rowptr, col, d, w, xT, dY, np.float32)
    out = _ev_f32(rowptr, col, d, w, xT, dY, rng)
    for name, ref in (("Y", Y), ("dw", dw), ("dxT", dxT)):
        assert orc.bound_violation(out[name], ref, env[name]) <= 1.0, name


# (bug, the output it shows in); error / bound measured on the CPU with these seeds at the end of each line
WRONG = [
    ("wgrad_drop33", "dw"),         # the 33rd entry of a row (the second flush group) never stored: 3.0e4
    ("wgrad_dup33", "dw"),          # ... stored with the 32nd entry's value: 7.7e34 (a k = 0 slot that must be 0)
    ("adjoint_wkm1", "dw"),         # lam_{k-1} = dY + Phi_{k-1}^T lam_k: 1.7e5
    ("adjoint_no_dy", "dw"),        # lam_{k-1} = Phi_k^T lam_k: 2.7e4
    ("k0_whole_row", "Y"),          # k = 0 with diag sums the whole row instead of the diagonal slot: 5.9e5
    ("g_tail", "Y"),                # features g >= 8 (the G % 8 tail of the GB = 8 loop) dropped: 1.6e4
    ("lane_swap", "Y"),             # batch lanes 1 and 2 of each 4-vector exchanged: 7.5e4
]


@pytest.mark.parametrize("bug,out", WRONG, ids=[b for b, _ in WRONG])
def test_envelope_rejects_wrong_kernel(env_case, bug, out):
    rng = np.random.default_rng(3)
    got = _ev_f32(*env_case["args"], rng, bug=bug)
    v = orc.bound_violation(got[out], env_case["ref"][out], env_case["env"][out])
    print("%s: %s error / bound %.3g" % (bug, out, v))
    assert v > WIDE, (bug, v)


# ------------------------------------------------------------------------------------------------ C ABI checks
def test_ev_abi_rejects_bad_arguments_without_gpu():
    """Every call below returns before any CUDA call (the fake pointers are never dereferenced)."""
    import gnn_b200
    cabi = gnn_b200._cabi
    lib = cabi.load()
    EINVAL, EUNSUP = -1, -2
    p = ctypes.c_void_p(256)
    base = dict(dtype=cabi.F32, NA=10, B=4, G=2, F=3, K=3, rowptr=p, col=p, diag=None, nnz=20, w=p, xT=p, states=p,
                n_states=2, Y=p)

    def fwd(**kw):
        a = dict(base, **kw)
        return lib.b200gf_ev_forward(a["dtype"], a["NA"], a["B"], a["G"], a["F"], a["K"], a["rowptr"], a["col"],
                                     a["diag"], a["nnz"], a["w"], a["xT"], a["states"], a["n_states"], a["Y"], None)

    bbase = dict(base, rowptrT=p, colT=p, perm=p, dY=p, lam=p, dw=p, dxT=p)

    def bwd(**kw):
        a = dict(bbase, **kw)
        return lib.b200gf_ev_backward(a["dtype"], a["NA"], a["B"], a["G"], a["F"], a["K"], a["rowptr"], a["col"],
                                      a["rowptrT"], a["colT"], a["perm"], a["diag"], a["nnz"], a["w"], a["xT"],
                                      a["states"], a["dY"], a["lam"], a["dw"], a["dxT"], None)

    for call in (fwd, bwd):
        for name in ("B", "G", "F", "K"):
            for v in (0, -1):
                assert call(**{name: v}) == EINVAL, (call.__name__, name, v)
        assert call(NA=-1) == EINVAL and call(nnz=-1) == EINVAL
        for name in ("rowptr", "col", "xT"):
            assert call(**{name: None}) == EINVAL, (call.__name__, name)
        assert call(w=None) == EINVAL                                     # nnz > 0
        assert call(states=None) == EINVAL                                # K > 1
        assert call(NA=2 ** 31) == EUNSUP and call(nnz=2 ** 31) == EUNSUP
        assert call(dtype=7) == EUNSUP
    assert fwd(Y=None) == EINVAL
    assert fwd(K=4, n_states=1) == EINVAL                                 # neither K-1 states nor a ping-pong pair
    assert fwd(K=5, n_states=3) == EINVAL
    assert fwd(K=3, n_states=0) == EINVAL
    for name in ("rowptrT", "colT", "perm", "dY", "lam", "dxT", "dw"):
        assert bwd(**{name: None}) == EINVAL, name
    # nothing to do: OK and no launch
    n0 = lib.b200gf_launch_count(0)
    assert fwd(NA=0) == 0 and bwd(NA=0) == 0
    assert fwd(NA=0, K=1, states=None) == 0
    assert lib.b200gf_launch_count(0) == n0
