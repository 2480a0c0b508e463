"""float64 restatement of the localized activations (MaxLocalActivation / MedianLocalActivation,
alegnn/utils/graphML.py:1535-1810) on ring-ordered K-hop lists (graphtools_sparse.ring_neighborhoods), with the
componentwise error bounds the CUDA kernels are held to.

TEST INFRASTRUCTURE.  Node-major data: x, dy [N, C].  Selection rules, the kernels' as well as the reference's on
index-sorted neighbourhoods:
  max     the largest value; equal values: the smallest node index (the reference's first maximum)
  median  the lower median, the (n - 1) / 2-th smallest of the n values (torch.median); the smallest node index
          holding that value
"""
import numpy as np

import lsigf_oracle as orc

MAX, MEDIAN = 0, 1


def select(x, rowptr, col, ring_end, K, op, rows=None):
    """(agg [K, R, C], arg [K, R, C] int64) for the rows `rows` (default: all), x [N, C] float64."""
    rows = np.arange(len(rowptr) - 1) if rows is None else np.asarray(rows)
    C = x.shape[1]
    agg = np.empty((K, len(rows), C))
    arg = np.empty((K, len(rows), C), dtype=np.int64)
    cidx = np.arange(C)
    for r, i in enumerate(rows):
        for k in range(1, K + 1):
            nb = np.sort(col[rowptr[i]:rowptr[i] + ring_end[i, k]].astype(np.int64))     # index-sorted neighbourhood
            vals = x[nb]                                                                 # [n, C]
            if op == MAX:
                pos = np.argmax(vals, axis=0)                                            # first maximum
            else:
                med = np.sort(vals, axis=0)[(len(nb) - 1) // 2]
                pos = np.argmax(vals == med[None, :], axis=0)                            # first node holding it
            agg[k - 1, r] = vals[pos, cidx]
            arg[k - 1, r] = nb[pos]
    return agg, arg


def forward(x, w, rowptr, col, ring_end, K, op, dtype, rows=None):
    """(y [R, C], its bound, agg, arg): y = w0 x + sum_k w_k agg_k, |dy| <= gamma_{K+1} (|w0 x| + sum_k |w_k agg_k|)."""
    rows = np.arange(len(rowptr) - 1) if rows is None else np.asarray(rows)
    w = np.asarray(w, dtype=np.float64).reshape(-1)
    agg, arg = select(x, rowptr, col, ring_end, K, op, rows)
    y = w[0] * x[rows] + np.einsum("k,krc->rc", w[1:], agg)
    absum = np.abs(w[0] * x[rows]) + np.einsum("k,krc->rc", np.abs(w[1:]), np.abs(agg))
    return y, orc.dot_bound(K + 1, absum, dtype), agg, arg


def backward(x, dy, w, agg, arg, dtype):
    """(dx, its bound, dw, its bound) of the full layer (agg, arg of every row, from select):
    dx = w0 dy + sum_k scatter_{arg_k}(w_k dy), bounded by gamma_m sum |terms| with m the terms of the entry;
    dw_0 = sum x dy, dw_k = sum agg_k dy, bounded by gamma_{NC} sum |.|."""
    w = np.asarray(w, dtype=np.float64).reshape(-1)
    N, C = dy.shape
    K = agg.shape[0]
    cols = np.broadcast_to(np.arange(C), (N, C))
    dx = w[0] * dy
    absdx = np.abs(w[0] * dy)
    cnt = np.ones((N, C))
    for k in range(K):
        np.add.at(dx, (arg[k], cols), w[k + 1] * dy)
        np.add.at(absdx, (arg[k], cols), np.abs(w[k + 1] * dy))
        np.add.at(cnt, (arg[k], cols), 1.0)
    terms = np.concatenate([x[None], agg], axis=0) * dy[None]                          # [K+1, N, C]
    dw = terms.reshape(K + 1, -1).sum(axis=1).reshape(1, K + 1)
    dw_bound = orc.dot_bound(N * C, np.abs(terms).reshape(K + 1, -1).sum(axis=1).reshape(1, K + 1), dtype)
    return dx, orc.dot_bound(cnt, absdx, dtype), dw, dw_bound
