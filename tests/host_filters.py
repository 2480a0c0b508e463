"""CPU stand-ins for the CUDA filters of gnn_b200.delayed, shared by the host-logic tests (test_widen_grnn_db.py,
test_recurrent_oracle.py): the space-time operator densified, and the delay-line hops applied by torch.sparse."""
import torch


def dense_from_csr(csr, M, dtype):
    """[(rowptr, col, val)] of E operators on M nodes -> dense [E, M, M] tensor."""
    S = torch.zeros(len(csr), M, M, dtype=dtype)
    for e, (rowptr, col, val) in enumerate(csr):
        rows = torch.repeat_interleave(torch.arange(M), rowptr[1:] - rowptr[:-1])
        S[e, rows, col.long()] = val
    return S


class SparseSlabOps:
    """CPU stand-in for delayed._SlabOps: the same per-(t, e) gather operators (slab_csr's `fwd`), applied by torch.sparse
    (differentiable w.r.t. the dense operand, so the recursion's autograd wiring is exercised too)."""

    def __init__(self, S):
        from gnn_b200 import delayed
        fwd, _, R = delayed.slab_csr(S)
        self.hops = 0
        self.A = [torch.sparse_csr_tensor(rp, col.long(), val, size=(R, R)).to_sparse_coo() for (rp, col, val) in fwd]

    def hop(self, o, src):
        self.hops += 1
        return torch.sparse.mm(self.A[o], src)
