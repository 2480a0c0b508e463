"""Every entry point refuses bad operands before its first launch, with one wording across the layer modules
(graphML.check_operands): x not on CUDA, x in a dtype the kernels do not run in, another operand in the other float
dtype, a tap or bias tensor on the host.  A host tensor must never reach a kernel as a host pointer.

The layers whose parameters meet x in torch operators before the check (MaxPoolLocal, EVGF, the edge-gated and
attention layers) reach only the first two checks: torch itself refuses a host parameter or a mixed dtype there.
Cases with x on the CPU need no GPU and run everywhere."""
import pytest
import torch

import gnn_b200
from gnn_b200 import _cabi, arma, attention, delayed, edgegated, edgevariant, nodevariant, pooling

B, T, G, F, H, K, P, N = 2, 3, 3, 4, 4, 3, 2, 12

FRAGMENT = {"cpu_x": "no CPU fallback", "half_x": "supports float32 and float64", "mixed_dtype": "one dtype",
            "host_taps": "on one device"}


def _gso(diagonal):
    """[1, N, N] ring adjacency, with `diagonal` on its diagonal."""
    i = torch.arange(N)
    S = torch.zeros(1, N, N)
    S[0, i, (i + 1) % N] = 0.5
    S[0, (i + 1) % N, i] = 0.5
    S[0, i, i] = diagonal
    return S


def _operands(case):
    """(t, taps): t(*shape) makes an operand on x's device and dtype, taps(*shape) the tap tensor of `case`."""
    gen = torch.Generator().manual_seed(0)
    dev = "cpu" if case == "cpu_x" else "cuda"
    dt = torch.float16 if case == "half_x" else torch.float32

    def t(*shape):
        return torch.rand(*shape, generator=gen).to(dev, dt)

    def taps(*shape):
        if case == "host_taps":
            return t(*shape).cpu()
        return t(*shape).double() if case == "mixed_dtype" else t(*shape)
    return t, taps


def _lsigf(case):
    t, taps = _operands(case)
    gnn_b200.LSIGF(taps(F, 1, K, G), t(1, N, N), t(B, G, N), t(F, 1))


def _nvgf(case):
    t, taps = _operands(case)
    nodevariant.NVGF(taps(F, 1, K, G, N), t(1, N, N), t(B, G, N), t(F, 1))


def _jarma(diagonal):
    def call(case):
        t, taps = _operands(case)
        S = _gso(diagonal).to(t(1).device, t(1).dtype)
        arma.jARMA(t(F, 1, P, G), t(F, 1, P, G), taps(F, 1, K, G), S, t(B, G, N), t(F, 1), tMax=2)
    return call


def _lsigf_db(case):
    t, taps = _operands(case)
    delayed.LSIGF_DB(taps(F, 1, K, G), t(B, T, 1, N, N), t(B, T, G, N), t(F, 1))


def _maxpool(case):
    t, _ = _operands(case)
    layer = pooling.MaxPoolLocal(N, N // 2, 1)
    layer.addGSO(_gso(0.0))
    layer(t(B, F, N))


def _evgf(case):
    t, _ = _operands(case)
    edgevariant.EVGF(t(F, 1, K, G, N, N), t(B, G, N), t(F, 1))


def _edge_gated(case):
    t, _ = _operands(case)
    pattern = edgegated.EdgeGatePattern(_gso(0.0))
    q = t(B, T, pattern.nnz)
    edgegated.EdgeGatedGRNN(t(H, 1, K, F), t(H, 1, K, H), pattern, t(B, T, F, N), t(B, H, N), torch.tanh, q, q)


def _graph_attention(case):
    t, _ = _operands(case)
    attention.graphAttention(t(B, G, N), t(P, 1, 2 * F), t(P, 1, F, G), _gso(0.0))


ALL_FOUR = ("cpu_x", "half_x", "mixed_dtype", "host_taps")
ENTRY_POINTS = {
    "LSIGF": (_lsigf, ALL_FOUR),
    "NVGF": (_nvgf, ALL_FOUR),
    "jARMA-general": (_jarma(torch.arange(N) * 0.1), ALL_FOUR),
    "jARMA-constant": (_jarma(0.0), ALL_FOUR),
    "LSIGF_DB": (_lsigf_db, ALL_FOUR),
    "MaxPoolLocal": (_maxpool, ALL_FOUR[:2]),
    "EVGF": (_evgf, ALL_FOUR[:2]),
    "EdgeGatedGRNN": (_edge_gated, ALL_FOUR[:2]),
    "graphAttention": (_graph_attention, ALL_FOUR[:2]),
}


@pytest.mark.parametrize("entry,case", [
    pytest.param(entry, case, marks=() if case == "cpu_x" else pytest.mark.gpu)
    for entry, (_, cases) in ENTRY_POINTS.items() for case in cases])
def test_bad_operands_are_rejected_before_any_launch(entry, case):
    lib = _cabi.load()
    call = ENTRY_POINTS[entry][0]
    before = lib.b200gf_launch_count(0)
    with pytest.raises(RuntimeError, match=FRAGMENT[case]):
        call(case)
    assert lib.b200gf_launch_count(0) == before
