"""Static-GSO graph recurrent layers on top of the CUDA LSIGF path (SURVEY.md §8f rank 2).

    GatedGRNN(a, b, S, x, z0, sigma, q_hat, q_check, xBias, zBias)   <- alegnn/utils/graphML.py:1292-1527
    HiddenState(F, H, K, nonlinearity, E, bias)                       <- graphML.py:3540-3681
    TimeGatedHiddenState(...)                                         <- graphML.py:3683-3855
    NodeGatedHiddenState(...)                                         <- graphML.py:3857-4031

    z_t = sigma( q_hat_t * (A(S) x_t) + q_check_t * (B(S) z_{t-1}) ),   t = 1..T

Both filters are LSIGF calls (graphML.py:1403 for all B*T inputs at once, :1461 once per time step).  What changes
here is the data movement between them:

  * the whole recursion lives in node-major memory ([N, B, T, H] / [N, B, H]): A(S)x comes out of LSIGF as a node-major
    view, every state z_t is produced node-major by the element-wise gate/sum/sigma and goes back into LSIGF with
    no transpose (the reference re-lays-out per step through index_select / permute-copies);
  * the T hidden states are stacked once at the end; the reference grows the trajectory with torch.cat inside the loop
    (graphML.py:1522-1525: O(T^2) bytes copied);
  * the returned [B, T, H, N] tensor is a view of the [N, B, T, H] buffer, so `z.reshape(B*T, H, N)` in
    GraphRecurrentNN.splitForward (architectures.py:4551) is again a node-major view the output filter consumes in place.

Edge gating (5-D gates, graphML.py:1410-1451 / :1474-1514) multiplies a dense N x N gate into the GSO per sample and
time step; it runs on per-non-zero gates in edgegated.py (EdgeGatedGRNN / EdgeGatedHiddenState), and GatedGRNN raises.
"""
import math

import torch
import torch.nn as nn

from . import graphML as _gml

# the filter every call below goes through; tests swap in the CPU oracle to check the host logic without a GPU
_lsigf = _gml.LSIGF


def _check_gate(q, B, T, N, name):
    """Shape rules of graphML.py:1378-1391; returns 'none' | 'scalar' | 'time/node'."""
    if q is None:
        return "none"
    assert q.shape[0] == B or q.shape[0] == 1
    if q.dim() <= 1:
        if q.numel() != 1:     # a 1-D gate would broadcast along the node axis in the reference (q*Ax, :1409)
            raise ValueError("b200gf: %s must be a one-element tensor or 4-D [B|1, T, 1, 1|N]" % name)
        return "scalar"
    if q.dim() > 4:
        raise NotImplementedError(
            "b200gf: edge gating (%s of shape %s) needs a per-sample, per-time-step GSO (graphML.py:1410-1451); "
            "only ungated, time-gated and node-gated recursions run on the static-GSO path; edge-gated recursions run on "
            "per-non-zero gates in gnn_b200.EdgeGatedGRNN / EdgeGatedHiddenState" % (name, tuple(q.shape)))
    assert q.dim() == 4
    assert q.shape[1] == T
    assert q.shape[2] == 1
    assert q.shape[3] == 1 or q.shape[3] == N
    return "time/node"


def GatedGRNN(a, b, S, x, z0, sigma, q_hat=None, q_check=None, xBias=None, zBias=None):
    """GatedGRNN(signal_to_hidden_taps, hidden_to_hidden_taps, GSO, input, initial_hidden, nonlinearity,
                 input_gate, forget_gate, signal_bias, hidden_bias)          (graphML.py:1292-1527)

    a [H, E, K, F]; b [H, E, K, H]; S [E, N, N] (dense tensor / SparseGSO / Plan); x [B, T, F, N]; z0 [B, H, N];
    q_hat, q_check: None (the reference's `torch.ones(1)` default), [B|1, T, 1, 1] (time gating) or
    [B|1, T, 1, N] (node gating); xBias, zBias: anything with H elements (the reference passes [H, 1]) or None.
    Returns the hidden-state trajectory z [B, T, H, N].
    """
    H, E, K, F = a.shape
    assert b.shape[0] == H
    assert b.shape[1] == E
    assert b.shape[2] == K
    assert b.shape[3] == H
    assert S.shape[0] == E
    N = S.shape[1]
    assert S.shape[2] == N
    B, T = x.shape[0], x.shape[1]
    assert x.shape[2] == F
    assert x.shape[3] == N
    assert z0.shape[0] == B
    assert z0.shape[1] == H
    assert z0.shape[2] == N
    hat_kind = _check_gate(q_hat, B, T, N, "q_hat")
    check_kind = _check_gate(q_check, B, T, N, "q_check")
    if xBias is not None:
        xBias = xBias.reshape(H, 1)
    if zBias is not None:
        zBias = zBias.reshape(H, 1)

    # A(S) x_t for every (b, t) in one filter call (graphML.py:1403); node-major [N, B, T, H] from here on
    Ax = _lsigf(a, S, x.reshape(B * T, F, N), xBias)                   # [B*T, H, N]
    Ax = Ax.permute(2, 0, 1).reshape(N, B, T, H)
    if hat_kind == "scalar":
        Ax = q_hat.to(Ax.device).reshape(()) * Ax
    elif hat_kind == "time/node":
        Ax = q_hat.permute(3, 0, 1, 2) * Ax                             # [1|N, B|1, T, 1] against [N, B, T, H]
    gate = None
    if check_kind == "scalar":
        gate = [q_check.to(Ax.device).reshape(())] * T
    elif check_kind == "time/node":
        qn = q_check.permute(3, 0, 1, 2)                                # [1|N, B|1, T, 1]
        gate = qn.unbind(2)                                             # T x [1|N, B|1, 1] against [N, B, H]

    # unbind, not Ax[:, :, t]: its backward is one stack instead of T zero-filled [N, B, T, H] buffers
    Ax_t = Ax.unbind(2)
    zt = z0
    states = []
    for t in range(T):
        Bz = _lsigf(b, S, zt, zBias).permute(2, 0, 1)                   # B(S) z_{t-1} (graphML.py:1461), [N, B, H]
        if gate is not None:
            Bz = gate[t] * Bz
        zn = sigma(Ax_t[t] + Bz).contiguous()                            # graphML.py:1516-1521, kept node-major
        states.append(zn)
        zt = zn.permute(1, 2, 0)                                        # [B, H, N] view with ld = B*H
    z = torch.stack(states, dim=2)                                      # [N, B, T, H], one copy for the trajectory
    return z.permute(1, 2, 3, 0)


class HiddenState(nn.Module):
    """HiddenState(signal_features, hidden_features, filter_taps, nonlinearity=torch.tanh, edge_features=1, bias=True)

    Same surface as graphML.py:3540-3681: parameters aWeights [H,E,K,F], bWeights [H,E,K,H], xBias/zBias [H,1];
    forward(x [B,T,F,N], z0 [B,H,N]) -> (z [B,T,H,N], z_T [B,1,1,H,N])."""

    def __init__(self, F, H, K, nonlinearity=torch.tanh, E=1, bias=True):
        super().__init__()
        self.F = F
        self.H = H
        self.K = K
        self.E = E
        self.S = None
        self.bias = bias
        self.sigma = nonlinearity
        self.aWeights = nn.parameter.Parameter(torch.Tensor(H, E, K, F))
        self.bWeights = nn.parameter.Parameter(torch.Tensor(H, E, K, H))
        if self.bias:
            self.xBias = nn.parameter.Parameter(torch.Tensor(H, 1))
            self.zBias = nn.parameter.Parameter(torch.Tensor(H, 1))
        else:
            self.register_parameter("xBias", None)
            self.register_parameter("zBias", None)
        self.reset_parameters()

    def reset_parameters(self):
        stdv = 1. / math.sqrt(self.F * self.K)      # graphML.py:3620-3627
        self.aWeights.data.uniform_(-stdv, stdv)
        self.bWeights.data.uniform_(-stdv, stdv)
        if self.bias:
            self.xBias.data.uniform_(-stdv, stdv)
            self.zBias.data.uniform_(-stdv, stdv)

    def _gates(self, x, z0):
        return None, None

    def forward(self, x, z0):
        assert self.S is not None
        assert len(x.shape) == 4
        B = x.shape[0]
        T = x.shape[1]
        assert x.shape[2] == self.F
        N = x.shape[3]
        assert len(z0.shape) == 3
        assert z0.shape[0] == B
        assert z0.shape[1] == self.H
        assert z0.shape[2] == N
        qHat, qCheck = self._gates(x, z0)
        z = GatedGRNN(self.aWeights, self.bWeights, self.S, x, z0, self.sigma, qHat, qCheck,
                      xBias=self.xBias, zBias=self.zBias)
        zT = z[:, T - 1:T]                          # the last state, to chain calls (graphML.py:3656-3660)
        return z, zT.unsqueeze(1)

    def addGSO(self, S):
        assert len(S.shape) == 3
        assert S.shape[0] == self.E
        self.N = S.shape[1]
        assert S.shape[2] == self.N
        self.S = S
        if torch.cuda.is_available() and (isinstance(S, (_gml.SparseGSO, _gml.Plan)) or
                                          (isinstance(S, torch.Tensor) and S.device.type == "cuda")):
            _gml.plan_for(S)

    def extra_repr(self):
        reprString = "in_features=%d, hidden_features=%d, " % (self.F, self.H) + "filter_taps=%d, " % (self.K) + \
                     "edge_features=%d, " % (self.E) + "bias=%s, " % (self.bias) + "nonlinearity=%s" % (self.sigma)
        if self.S is not None:
            reprString += "GSO stored"
        else:
            reprString += "no GSO stored"
        return reprString


class _GatedHiddenState(HiddenState):
    """Shared part of the time- and node-gated layers: two auxiliary ungated GRNNs (tanh, E = 1 as in
    graphML.py:3757-3760 / :3931-3934) whose trajectories are mapped to the input and forget gates."""

    def __init__(self, F, H, K, nonlinearity=torch.tanh, E=1, bias=True):
        nn.Module.__init__(self)
        self.F = F
        self.H = H
        self.K = K
        self.E = E
        self.S = None
        self.bias = bias
        self.sigma = nonlinearity
        self.aWeights = nn.parameter.Parameter(torch.Tensor(H, E, K, F))
        self.bWeights = nn.parameter.Parameter(torch.Tensor(H, E, K, H))
        self.inputGateGRNN = HiddenState(F, H, K, bias=bias)
        self.forgetGateGRNN = HiddenState(F, H, K, bias=bias)
        if self.bias:
            self.xBias = nn.parameter.Parameter(torch.Tensor(H, 1))
            self.zBias = nn.parameter.Parameter(torch.Tensor(H, 1))
        else:
            self.register_parameter("xBias", None)
            self.register_parameter("zBias", None)
        self.reset_parameters()

    def addGSO(self, S):
        HiddenState.addGSO(self, S)
        # fresh gate maps on every addGSO, as in the reference; initialised as the reference does, then placed on the
        # layer's device (a layer moved to the GPU before addGSO keeps its gates there too)
        self._make_gate_maps()
        self.inputGateGRNN.addGSO(S)
        self.forgetGateGRNN.addGSO(S)


class TimeGatedHiddenState(_GatedHiddenState):
    """graphML.py:3683-3855: one scalar gate per (sample, time step): q = sigmoid(Linear(H*N -> 1)(z_gate[b, t]))."""

    def _make_gate_maps(self):
        dev = self.aWeights.device
        self.inputGateFC = nn.Linear(self.H * self.N, 1, self.bias).to(dev)       # graphML.py:3838-3839
        self.forgetGateFC = nn.Linear(self.H * self.N, 1, self.bias).to(dev)

    def _gates(self, x, z0):
        B, T = x.shape[0], x.shape[1]
        N = x.shape[3]
        zHat, _ = self.inputGateGRNN(x, z0)
        qHat = torch.sigmoid(self.inputGateFC(zHat.reshape((B, T, self.H * N)))).unsqueeze(2)      # [B, T, 1, 1]
        zCheck, _ = self.forgetGateGRNN(x, z0)
        qCheck = torch.sigmoid(self.forgetGateFC(zCheck.reshape((B, T, self.H * N)))).unsqueeze(2)
        return qHat, qCheck


class NodeGatedHiddenState(_GatedHiddenState):
    """graphML.py:3857-4031: one gate per (sample, time step, node): q = sigmoid(GraphFilter(H -> 1)(z_gate))."""

    def _make_gate_maps(self):
        dev = self.aWeights.device
        self.inputGateGraphFilter = _gml.GraphFilter(self.H, 1, self.K, bias=self.bias).to(dev)   # graphML.py:4008-4009
        self.forgetGateGraphFilter = _gml.GraphFilter(self.H, 1, self.K, bias=self.bias).to(dev)
        self.inputGateGraphFilter.addGSO(self.S)
        self.forgetGateGraphFilter.addGSO(self.S)

    def _gates(self, x, z0):
        B, T = x.shape[0], x.shape[1]
        N = x.shape[3]
        zHat, _ = self.inputGateGRNN(x, z0)
        qHat = torch.sigmoid(self.inputGateGraphFilter(zHat.reshape((B * T, self.H, N)))).reshape((B, T, 1, N))
        zCheck, _ = self.forgetGateGRNN(x, z0)
        qCheck = torch.sigmoid(self.forgetGateGraphFilter(zCheck.reshape((B * T, self.H, N)))).reshape((B, T, 1, N))
        return qHat, qCheck
