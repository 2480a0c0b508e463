"""The componentwise error bounds of oracle/lsigf_oracle.py are themselves tested here (CPU only): an emulated correct
fp32 kernel (float32 accumulation in a shuffled order) must meet them, and emulations of three subtly wrong kernels must
miss them by a wide margin at the shapes tests/test_kernel_dispatch.py runs on the GPU:
  * 1xTF32: both operands truncated to TF32 (10 explicit mantissa bits) instead of the 3xTF32 split,
  * 3xTF32 without the lo·hi term,
  * a hop that drops one neighbour of every row."""
import numpy as np
import pytest
import scipy.sparse as sp

import lsigf_oracle as orc

WIDE = 2.5      # a wrong kernel must exceed its bound at least this many times (3x at T*P = 1536, 75-150x at 32)


def _accumulate_f32(prods, order):
    """sum over axis 0 of float32 products, in `order`, rounding after every addition (no FMA: the worst case)."""
    acc = np.zeros(prods.shape[1:], dtype=np.float32)
    for k in order:
        acc = (acc + prods[k]).astype(np.float32)
    return acc


def _contract(A, W, rng, kind):
    """A [n, R] (one column per output row), W [n, Q] float32 -> float32 [R, Q] the way `kind` of kernel computes it."""
    n = A.shape[0]
    hi = lambda v: orc.tf32_truncate(v)                                    # noqa: E731
    lo = lambda v: orc.tf32_truncate((v - hi(v)).astype(np.float32))      # noqa: E731
    if kind == "fp32":
        prods = (A[:, :, None] * W[:, None, :]).astype(np.float32)
    elif kind == "3xtf32":
        prods = (hi(A)[:, :, None] * hi(W)[:, None, :] + lo(A)[:, :, None] * hi(W)[:, None, :]
                 + hi(A)[:, :, None] * lo(W)[:, None, :]).astype(np.float32)
    elif kind == "1xtf32":
        prods = (hi(A)[:, :, None] * hi(W)[:, None, :]).astype(np.float32)
    elif kind == "3xtf32_no_lohi":
        prods = (hi(A)[:, :, None] * hi(W)[:, None, :] + hi(A)[:, :, None] * lo(W)[:, None, :]).astype(np.float32)
    else:
        raise ValueError(kind)
    return _accumulate_f32(prods, rng.permutation(n))


# (T*P accumulation length, Q): the wgmma cases of test_kernel_dispatch.py (T = 1 / 16, P = 32 / 96 / 288)
CONTRACT_SHAPES = [(32, 16), (96, 48), (288, 96), (512, 80), (1536, 48)]


@pytest.mark.parametrize("n,Q", CONTRACT_SHAPES)
def test_contraction_bound_accepts_correct_and_rejects_wrong(n, Q):
    rng = np.random.default_rng(n + Q)
    R = 64
    A = orc.biased_uniform(rng, (n, R)).astype(np.float32)
    W = orc.biased_uniform(rng, (n, Q)).astype(np.float32)
    ref = A.astype(np.float64).T @ W.astype(np.float64)
    absp = np.abs(A.astype(np.float64)).T @ np.abs(W.astype(np.float64))
    plain = orc.dot_bound(n, absp, np.float32)
    tc = orc.dot_bound(n, absp, np.float32, tf32x3=True)
    assert orc.bound_violation(_contract(A, W, rng, "fp32"), ref, plain) <= 1.0
    assert orc.bound_violation(_contract(A, W, rng, "3xtf32"), ref, tc) <= 1.0
    for wrong in ("1xtf32", "3xtf32_no_lohi"):
        v = orc.bound_violation(_contract(A, W, rng, wrong), ref, tc)
        assert v > WIDE, (wrong, n, Q, v)


def _graph(rng, N, lens):
    rows, cols = [], []
    for r, L in enumerate(lens):
        rows += [r] * L
        cols += list(rng.choice(N, size=L, replace=False))
    vals = rng.standard_normal(len(rows))
    return sp.csr_matrix((vals, (rows, cols)), shape=(N, N))


def _hop_f32(S, X, rng, drop):
    """float32 hop in a shuffled order per row; drop=True leaves out one neighbour of every non-empty row."""
    out = np.zeros(X.shape, dtype=np.float32)
    S = S.astype(np.float32)
    for r in range(S.shape[0]):
        beg, end = S.indptr[r], S.indptr[r + 1]
        idx = rng.permutation(np.arange(beg, end))
        if drop and len(idx):
            idx = idx[1:]
        acc = np.zeros(X.shape[1], dtype=np.float32)
        for j in idx:
            acc = (acc + S.data[j] * X[S.indices[j]]).astype(np.float32)
        out[r] = acc
    return out


def test_hop_bound_accepts_correct_and_rejects_dropped_neighbour():
    # the row lengths of the dispatch graph around the lane-group boundaries (S*U - 1, S*U, S*U + 1, 31..65) and a hub
    rng = np.random.default_rng(5)
    N = 2500
    lens = [0, 1, 3, 4, 5, 15, 16, 17, 31, 32, 33, 64, 65, 2000] + list(rng.integers(0, 9, N - 14))
    S = _graph(rng, N, lens)
    X = rng.standard_normal((N, 24)).astype(np.float32)
    Sr = S.astype(np.float32).astype(np.float64)
    ref = Sr @ X.astype(np.float64)
    bound = orc.dot_bound(np.diff(S.indptr)[:, None], abs(Sr) @ np.abs(X.astype(np.float64)), np.float32)
    assert orc.bound_violation(_hop_f32(S, X, rng, False), ref, bound) <= 1.0
    v = orc.bound_violation(_hop_f32(S, X, rng, True), ref, bound)
    assert v > 1e3, v


def test_max_normalised_ratio_would_miss_a_small_row():
    """Why the bound is componentwise: one wrong element in a row 1e4 times smaller than the largest passes
    max|a-b| / max|b| < 1e-4 and fails the componentwise bound."""
    ref = np.array([[1e4, 1.0], [1.0, 1.0]])
    out = ref.copy()
    out[1, 1] *= 1.0 + 1e-3
    assert np.abs(out - ref).max() / np.abs(ref).max() < 1e-4
    assert orc.bound_violation(out, ref, orc.dot_bound(8, np.abs(ref), np.float32)) > 100


def test_lsigf_envelope_accepts_fp32_run_and_rejects_perturbation():
    import torch
    c = orc.random_case(3, N=60, B=2, G=5, F=4, K=4, E=2, avg_deg=5, bias="F1")
    rnd = lambda a: np.asarray(a, np.float32).astype(np.float64)          # noqa: E731
    h, S, x, b, dy = (rnd(c[k]) for k in ("h", "S", "x", "b", "dy"))
    env = orc.lsigf_envelope(h, list(S), x, b, dy, np.float32)
    y_ref = orc.lsigf_dense(h, S, x, b)
    y32 = orc.lsigf_dense_torch(*(torch.tensor(a, dtype=torch.float32) for a in (h, S, x, b))).numpy()
    assert orc.bound_violation(y32, y_ref, env["y"]) <= 1.0
    dh_ref, dx_ref, db_ref = orc.lsigf_grads_dense(h, S, x, dy, b.shape)
    for name, ref in (("dh", dh_ref), ("dx", dx_ref), ("db", db_ref)):
        assert orc.bound_violation(ref.astype(np.float32), ref, env[name]) <= 1.0
    bad = y32.copy()
    bad[1, 2, 7] += 1e-3 * abs(y_ref[1, 2, 7]) + 1e-6
    assert orc.bound_violation(bad, y_ref, env["y"]) > WIDE
