"""CSR-native counterparts of the graph utilities the LSIGF path's callers use to build their GSOs (SURVEY.md §8f-3).

The reference's `alegnn/utils/graphTools.py` works on dense N x N numpy arrays and checks connectivity with a dense
eigendecomposition, which stops at N ~ 1e4; the functions here take and return scipy sparse matrices, keep the
reference's semantics (citations below; verified against the reference itself in tests/test_graphtools_sparse.py) and
scale to the graphs of BASELINE.json's configs.  Host-side numpy/scipy only: this is the data format feeding
`SparseGSO`, not part of the GPU path.

    adjacency_to_laplacian      graphTools.py:203-222
    normalize_adjacency         graphTools.py:224-245
    normalize_laplacian         graphTools.py:247-268
    spectral_normalize          S = W / max(real eig), examples/sourceLocGNN.py:752 (via computeGFT :270-309)
    is_connected                graphTools.py:562-589   (components of the symmetrised pattern instead of Laplacian eig)
    compute_neighborhood        graphTools.py:378-527
    ring_neighborhoods          the K-hop neighbourhoods of compute_neighborhood as one CSR, ordered by hop distance
    perm_degree                 graphTools.py:1020-1052
    edge_fail_sampling          graphTools.py:1163-1190
    sparsify_graph              graphTools.py:591-680
"""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.csgraph as csgraph
import scipy.sparse.linalg as spla

zeroTolerance = 1e-9  # graphTools.py:45


def _csr(W):
    W = sp.csr_matrix(W)
    assert W.shape[0] == W.shape[1]
    return W


def adjacency_to_laplacian(W):
    """L = D - W with d = row sums (graphTools.py:216-222)."""
    W = _csr(W)
    d = np.asarray(W.sum(axis=1)).ravel()
    return (sp.diags(d) - W).tocsr()


def normalize_adjacency(W):
    """D^-1/2 W D^-1/2 with d = row sums (graphTools.py:237-245).  Like the reference, a zero-degree node gives inf."""
    W = _csr(W)
    d = np.asarray(W.sum(axis=1)).ravel()
    with np.errstate(divide="ignore"):
        dinv = 1.0 / np.sqrt(d)
    D = sp.diags(dinv)
    return (D @ W @ D).tocsr()


def normalize_laplacian(L):
    """D^-1/2 L D^-1/2 with d = diag(L) (graphTools.py:260-268)."""
    L = _csr(L)
    with np.errstate(divide="ignore"):
        dinv = 1.0 / np.sqrt(L.diagonal())
    D = sp.diags(dinv)
    return (D @ L @ D).tocsr()


def largest_real_eigenvalue(W, tol=1e-10):
    """max over eigenvalues of Re(lambda) — what `np.max(np.real(G.E))` reads off computeGFT in the examples."""
    W = _csr(W).astype(np.float64)
    N = W.shape[0]
    if N <= 3:
        return float(np.max(np.real(np.linalg.eigvals(W.toarray()))))
    symmetric = abs(W - W.T).max() <= zeroTolerance
    if symmetric:
        vals = spla.eigsh(W, k=1, which="LA", tol=tol, return_eigenvectors=False)
    else:
        vals = spla.eigs(W, k=1, which="LR", tol=tol, return_eigenvectors=False)
    return float(np.max(np.real(vals)))


def spectral_normalize(W):
    """S = W / lambda_max (examples/sourceLocGNN.py:752, movieGNN.py:633): spectral radius 1 for non-negative W."""
    W = _csr(W)
    return (W / largest_real_eigenvalue(W)).tocsr()


def is_connected(W):
    """True iff the graph with all edge directions dropped is connected (graphTools.py:562-589 counts the zero
    eigenvalues of the Laplacian of (W + W^T)/2; the number of weakly connected components is the same number)."""
    W = _csr(W)
    if W.shape[0] == 0:
        return False
    n, _ = csgraph.connected_components(abs(W) + abs(W.T), directed=False)
    return n == 1


def _edge_pattern(S):
    """Boolean CSR pattern of S, or of a list of E matrices (edge features: an edge exists where sum_e |S_e| > 1e-9,
    graphTools.py:424-432)."""
    if isinstance(S, (list, tuple)):
        acc = None
        for Se in S:
            Se = abs(_csr(Se))
            acc = Se if acc is None else acc + Se
        return acc > zeroTolerance
    return _csr(S) > zeroTolerance


def compute_neighborhood(S, K, N="all", nb="all", outputType="list"):
    """K-hop neighbourhoods (graphTools.py:378-527).  S: sparse matrix, or a list of E sparse matrices (edge features:
    an edge exists where sum_e |S_e| > 0, :424-432).  Row i's one-hop neighbours are the columns j with S[i, j] > 0.
    Returns, for the first N nodes, the nodes < nb reachable within K hops (each node is in its own neighbourhood):
    a list of sorted lists, or (outputType 'matrix') an int array padded with the node's own index (:504-525)."""
    A = _edge_pattern(S)
    n = A.shape[0]
    assert K >= 0
    if N == "all":
        N = n
    if nb == "all":
        nb = n
    assert 0 <= N <= n and 0 <= nb <= n
    step = (A.astype(np.int8) + sp.identity(n, dtype=np.int8, format="csr")).tocsr()
    reach = sp.identity(n, dtype=np.int8, format="csr")[:N]
    for _ in range(K):
        reach = (reach @ step)
        reach.data[:] = 1                       # boolean semiring: keep the pattern, drop the path counts
    reach = reach.tocsr()
    reach.sort_indices()
    neighbors = []
    for i in range(N):
        cols = reach.indices[reach.indptr[i]:reach.indptr[i + 1]]
        neighbors.append([int(j) for j in cols if j < nb])
    if outputType == "matrix":
        width = max((len(x) for x in neighbors), default=0)
        out = np.empty((N, width), dtype=np.int64)
        for i, x in enumerate(neighbors):
            out[i, :len(x)] = x
            out[i, len(x):] = i
        return out
    return neighbors


def ring_neighborhoods(S, K):
    """Every node's K-hop neighbourhood (compute_neighborhood's edge rule: row i's neighbours are the columns j with
    sum_e |S_e[i, j]| > 1e-9) as one CSR ordered by hop distance.  S: sparse matrix or list of E of them.

    Returns (rowptr int64 [N+1], col int32, ring_end int32 [N, K+1]): row i lists col[rowptr[i] : rowptr[i+1]], ring 0
    (i itself), then ring 1 (the nodes first reached in one hop), ..., ring K, ascending node index within a ring; its
    k-hop neighbourhood is the prefix of length ring_end[i, k].  This is the list format of the localized activations'
    kernels (b200gf_local_activation_forward): one list per node serves every k, and no row is padded to the widest."""
    A = _edge_pattern(S)
    n = A.shape[0]
    assert K >= 0
    step = (A.astype(np.int32) + sp.identity(n, dtype=np.int32, format="csr")).tocsr()
    reach = sp.identity(n, dtype=np.int32, format="csr")
    rings = [reach]
    for _ in range(K):
        nxt = (reach @ step).tocsr()
        nxt.data[:] = 1                          # boolean semiring; int32 path counts cannot wrap to zero
        ring = (nxt - reach).tocsr()             # reach is a subset of nxt (step holds the identity)
        ring.eliminate_zeros()
        rings.append(ring)
        reach = nxt
    total = int(reach.nnz)
    if total > np.iinfo(np.int32).max:
        raise ValueError("ring_neighborhoods: the %d-hop lists of N = %d nodes hold %d entries, more than the 2^31 - 1 "
                         "that int32 list offsets address" % (K, n, total))
    counts = np.stack([np.diff(r.indptr) for r in rings], axis=1).astype(np.int64)       # [N, K+1]
    ring_end = np.cumsum(counts, axis=1)
    rowptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(ring_end[:, -1], out=rowptr[1:])
    rows = np.concatenate([np.repeat(np.arange(n), np.diff(r.indptr)) for r in rings])
    hops = np.concatenate([np.full(r.nnz, k, dtype=np.int32) for k, r in enumerate(rings)])
    cols = np.concatenate([r.indices for r in rings])
    order = np.lexsort((cols, hops, rows))
    return rowptr, cols[order].astype(np.int32), ring_end.astype(np.int32)


def perm_degree(S):
    """Nodes ordered from highest to lowest degree (graphTools.py:1020-1052).  S: sparse matrix or list of E sparse
    matrices; degree = column sums added over edge features (:1041), order = flip(argsort(d)) (:1043-1045).
    Returns (permuted S in the input's form, order as a list)."""
    many = isinstance(S, (list, tuple))
    mats = [_csr(m) for m in (S if many else [S])]
    d = np.zeros(mats[0].shape[0])
    for m in mats:
        d = d + np.asarray(m.sum(axis=0)).ravel()
    order = np.flip(np.argsort(d), 0)
    perm = [m[order][:, order].tocsr() for m in mats]
    return (perm if many else perm[0]), order.tolist()


def edge_fail_sampling(W, p, rng=None, dense_rng_compat=False):
    """Delete every edge independently with probability p (graphTools.py:1163-1190); for an undirected graph the coin
    is flipped on the upper triangle (diagonal included) and mirrored (:1186-1189).
    dense_rng_compat=True draws np.random.rand(N, N) exactly like the reference (bit-identical result under the same
    numpy seed; O(N^2)); the default draws one number per stored entry (O(nnz))."""
    assert 0 <= p <= 1
    W = _csr(W).astype(np.float64)
    N = W.shape[0]
    undirected = abs(W - W.T).max() <= zeroTolerance if W.nnz else True
    coo = W.tocoo()
    if dense_rng_compat:
        mask = (np.random.rand(N, N) > p)
        keep = mask[coo.row, coo.col]
    else:
        rng = np.random.default_rng() if rng is None else rng
        keep = rng.random(coo.nnz) > p
    if undirected:
        upper = coo.row <= coo.col
        r, c, v = coo.row[upper & keep], coo.col[upper & keep], coo.data[upper & keep]
        U = sp.coo_matrix((v, (r, c)), shape=(N, N)).tocsr()
        return (U + U.T).tocsr()                # the reference adds triu(W) + triu(W)^T: a kept diagonal entry doubles
    return sp.coo_matrix((coo.data[keep], (coo.row[keep], coo.col[keep])), shape=(N, N)).tocsr()


def _threshold(W, p):
    Wn = W.copy()
    Wn.data[np.abs(Wn.data) < p] = 0.0
    Wn.eliminate_zeros()
    return Wn


def _knn_rows(W, k):
    """Keep, in every row, the entries >= the k-th largest value of that row (zeros count, graphTools.py:655-658)."""
    W = W.tocsr()
    N = W.shape[0]
    rows, cols, vals = [], [], []
    for i in range(N):
        lo, hi = W.indptr[i], W.indptr[i + 1]
        data, idx = W.data[lo:hi], W.indices[lo:hi]
        full = np.zeros(N)
        full[idx] = data
        kth = np.sort(full)[-k]
        sel = data >= kth
        # the reference masks the dense row with (W >= kth): zero entries pass the mask when kth <= 0 but stay zero
        rows.extend([i] * int(sel.sum()))
        cols.extend(idx[sel].tolist())
        vals.extend(data[sel].tolist())
    return sp.coo_matrix((vals, (rows, cols)), shape=(N, N)).tocsr()


def sparsify_graph(W, sparsificationType, p):
    """'threshold': drop |w| < p; 'NN': keep each row's p largest entries, then symmetrise by averaging if the input was
    undirected.  If the input is connected and the result is not, the threshold is halved / k is increased until it is
    (graphTools.py:591-680)."""
    assert sparsificationType in ("threshold", "NN")
    W = _csr(W).astype(np.float64)
    connected = is_connected(W)
    undirected = abs(W - W.T).max() <= zeroTolerance if W.nnz else True
    if sparsificationType == "threshold":
        Wn = _threshold(W, p)
        while connected and not is_connected(Wn):
            p = p / 2.0
            Wn = _threshold(W, p)
        return Wn
    Wn = _knn_rows(W, p)
    while connected and not is_connected(Wn):
        p = p + 1
        Wn = _knn_rows(W, p)
    if undirected:
        Wn = (0.5 * (Wn + Wn.T)).tocsr()
    return Wn


def to_sparse_gso(mats, dtype=None):
    """scipy matrices (one per edge feature) -> gnn_b200.SparseGSO, the form GraphFilter.addGSO / LSIGF accept."""
    from .gso import SparseGSO
    return SparseGSO.from_scipy(list(mats) if isinstance(mats, (list, tuple)) else [mats], dtype)
