"""Localized activations (graph-neural-networks_b200/activations.py) vs the reference layers
(alegnn/utils/graphML.py:1535-1810) on CPU; the reference's results are stored in tests/golden (oracle/ref_golden.py)."""
import numpy as np
import pytest
import torch

import lsigf_oracle as orc
from ref_golden import reference


@pytest.mark.parametrize("kind", ["Max", "Median"])
@pytest.mark.parametrize("E,K,N", [(1, 1, 14), (1, 2, 18), (2, 3, 11)])
def test_local_activation_matches_reference(kind, E, K, N):
    import gnn_b200
    from gnn_b200 import activations
    rng = np.random.default_rng(10 * E + K + N)
    S = np.abs(orc.random_sparse_gso(rng, N, 3, E, symmetric=True))
    x0 = rng.standard_normal((2, 3, N))
    x = torch.tensor(x0, requires_grad=True)

    def run_reference():
        import ref_import
        gml = ref_import.import_reference()
        torch.manual_seed(K)
        ref = getattr(gml, kind + "LocalActivation")(K).double()
        ref.addGSO(torch.tensor(S))
        xr = torch.tensor(x0, requires_grad=True)
        y = ref(xr)
        g = torch.tensor(np.random.default_rng(10 * E + K + N + 1).standard_normal(tuple(y.shape)))
        gx, gw = torch.autograd.grad(y, [xr, ref.weight], g)
        return dict(weight=ref.weight.detach().numpy(), y=y.detach().numpy(), g=g.numpy(), gx=gx.numpy(), gw=gw.numpy())

    r = reference("activation_%s_E%d_K%d_N%d" % (kind, E, K, N), run_reference)
    y_ref, gx_ref, gw_ref = (torch.tensor(r[k]) for k in ("y", "gx", "gw"))
    mine = getattr(activations, kind + "LocalActivation")(K).double()
    mine.load_state_dict({"weight": torch.tensor(r["weight"])})   # same parameter name / shape as the reference
    mine.addGSO(torch.tensor(S))
    y = mine(x)
    assert torch.allclose(y, y_ref, atol=1e-14)
    gx, gw = torch.autograd.grad(y, [x, mine.weight], torch.tensor(r["g"]))
    assert torch.allclose(gw, gw_ref, atol=1e-13)
    assert torch.allclose(gx, gx_ref, atol=1e-13)
    sparse = getattr(activations, kind + "LocalActivation")(K).double()
    sparse.load_state_dict({"weight": torch.tensor(r["weight"])})
    sparse.addGSO(gnn_b200.SparseGSO.from_dense(torch.tensor(S)))
    assert torch.allclose(sparse(x), y_ref, atol=1e-14)


def test_no_activation():
    from gnn_b200 import activations
    x = torch.randn(2, 3, 4)
    assert activations.NoActivation()(x) is x
