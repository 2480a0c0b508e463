"""gnn_b200.MaxPoolLocal vs the reference layer (alegnn/utils/graphML.py:1850-2028) on CPU; the reference's results are
stored in tests/golden (oracle/ref_golden.py)."""
import numpy as np
import pytest
import torch

import lsigf_oracle as orc
from ref_golden import reference


@pytest.mark.parametrize("E,K,Nin,Nout", [(1, 1, 20, 20), (1, 2, 20, 9), (2, 3, 17, 5), (1, 0, 12, 7)])
def test_max_pool_local_matches_reference(E, K, Nin, Nout, monkeypatch):
    import gnn_b200
    from gnn_b200 import pooling
    from gnn_b200.pooling import MaxPoolLocal

    def gather_max(x, nb32, n_out, max_nb):          # torch stand-in for the CUDA gather (csrc/layer.cu); CPU leg only
        B, F, _ = x.shape
        return x.index_select(2, nb32.reshape(-1).long()).reshape(B, F, n_out, max_nb).max(dim=3)[0]

    monkeypatch.setattr(pooling, "_gather_max", gather_max)
    rng = np.random.default_rng(E * 100 + K)
    N = Nin
    S = np.abs(orc.random_sparse_gso(rng, N, 3, E, symmetric=True))     # the reference keeps entries > 1e-9 only
    x0 = rng.standard_normal((3, 4, Nin))
    g0 = rng.standard_normal((3, 4, Nout))
    x = torch.tensor(x0, requires_grad=True)

    def run_reference():
        import ref_import
        gml = ref_import.import_reference()
        ref = gml.MaxPoolLocal(Nin, Nout, K)
        ref.addGSO(torch.tensor(S))
        xr = torch.tensor(x0, requires_grad=True)
        y = ref(xr)
        (gx,) = torch.autograd.grad(y, xr, torch.tensor(g0))
        return dict(max_nb=np.int64(ref.maxNeighborhoodSize), neighborhood=ref.neighborhood.numpy(),
                    y=y.detach().numpy(), gx=gx.numpy())

    r = reference("maxpool_E%d_K%d_Nin%d_Nout%d" % (E, K, Nin, Nout), run_reference)
    mine = MaxPoolLocal(Nin, Nout, K)
    mine.addGSO(torch.tensor(S))
    assert mine.maxNeighborhoodSize == int(r["max_nb"])
    ref_nb = torch.tensor(r["neighborhood"]).to(mine.neighborhood.dtype)
    assert torch.equal(mine.neighborhood.sort(dim=1)[0], ref_nb.sort(dim=1)[0])
    y_ref = torch.tensor(r["y"])
    y = mine(x)
    assert torch.equal(y, y_ref)
    (gx,) = torch.autograd.grad(y, x, torch.tensor(g0))
    assert torch.allclose(gx, torch.tensor(r["gx"]))
    # the sparse description gives the same layer, and it works on a node-major strided view (what LSIGF returns)
    sparse = MaxPoolLocal(Nin, Nout, K)
    sparse.addGSO(gnn_b200.SparseGSO.from_dense(torch.tensor(S)))
    buf = x.detach().permute(2, 0, 1).contiguous()                       # [N, B, F] node-major
    assert torch.equal(sparse(buf.permute(1, 2, 0)), y_ref)
    assert "neighborhood stored" in mine.extra_repr()
