"""fp64 restatement of the recurrent and time-varying graph layers, with componentwise error bounds.
TEST INFRASTRUCTURE — NOT PRODUCT CODE.

Layers (gnn_b200.recurrent / gnn_b200.delayed; the reference's alegnn/utils/graphML.py):
  * `grnn_forward` / `grnn_backward`  – GatedGRNN (:1292-1527): ungated, scalar, time or node gates given;
  * `hidden_state`                    – HiddenState and the gated TimeGatedHiddenState / NodeGatedHiddenState
                                        (:3540-4031): gate GRNNs, Linear(H*N -> 1) / GraphFilter(H -> 1), sigmoid;
  * `lsigf_db`                        – LSIGF_DB (:977-1094) as LSIGF on the block-delay operator S_big (scipy);
  * `grnn_db`                         – GRNN_DB (:1096-1290) with its delay line of K-1 shifted states.
The reverse passes are the adjoint recursions written out by hand (no autograd), in the order autograd runs them.

Every quantity is a pair (v, beta): v the fp64 value computed from the inputs rounded to the layer's dtype, beta >= 0 a
componentwise first-order bound on how far an implementation in that dtype may lie from v.  The rules, with
u = lsigf_oracle.unit_roundoff(dtype) and gamma_n = n u / (1 - n u):
  LSIGF call        beta_y  = env_y(h, S, |x| + beta_x, b) + LSIGF(|h|, |S|, beta_x)     (3xTF32 term for fp32)
  LSIGF gradients   beta_dx = env_dx + LSIGF-adjoint(|h|, |S|, beta_dy)
                    beta_dh = env_dh + tapgrad(|x|, beta_dy) + tapgrad(beta_x, |dy| + beta_dy)
                    beta_db = env_db + sum beta_dy
  a + b             beta_a + beta_b + u |a + b|
  a * b             |a| beta_b + |b| beta_a + beta_a beta_b + u |a b|
  sigma(a)          L beta_a + c u |sigma(a)| + tiny          L = 1, 1/4, 1, 1 and c = 4, 4, 0, 0 for tanh, sigmoid, ReLU,
                                                              identity.  c = 4: CUDA documents <= 2 ulp for tanhf / expf.
  tanh' = 1 - z^2   2 |z| beta_z + 3 u;  sigmoid' = s (1 - s): |1 - 2 s| beta_s + 3 u s (1 - s);  ReLU: where
                    |pre| <= beta_pre the derivative is undetermined and |upstream| + beta_upstream is added.
  matmul (n terms)  gamma_n |W| |a| + |W| beta_a (+ |a| beta_W for a computed W)
  sums of n terms   sum beta + gamma_n sum |terms|   (parameter gradients over time steps, broadcast reductions)
(env_*: lsigf_oracle.lsigf_envelope.)  `tiny` is the underflow floor 4 * finfo(dtype).tiny.

Keyword `bug` plants one defect (tests/test_recurrent_oracle.py checks that the bound rejects each); None is the layer.
"""
import numpy as np
import scipy.sparse as sp

import lsigf_oracle as orc

F32, F64 = np.float32, np.float64


def rounded(a, dtype):
    """a rounded to dtype, held as float64."""
    return np.asarray(np.asarray(a, dtype=np.float64).astype(dtype), dtype=np.float64)


def exact(v):
    v = np.asarray(v, dtype=np.float64)
    return v, np.zeros_like(v)


def _u(dt):
    return orc.unit_roundoff(dt)


def _tiny(dt):
    return 4.0 * np.finfo(np.dtype(dt)).tiny


# ------------------------------------------------------------------------------------------------ element-wise rules
def add(a, b, dt):
    v = a[0] + b[0]
    return v, a[1] + b[1] + _u(dt) * np.abs(v) + _tiny(dt)


def mul(a, b, dt):
    v = a[0] * b[0]
    return v, np.abs(a[0]) * b[1] + np.abs(b[0]) * a[1] + a[1] * b[1] + _u(dt) * np.abs(v) + _tiny(dt)


def _sigmoid(v):
    return 0.5 * (1.0 + np.tanh(0.5 * v))


ACT = {"tanh": (np.tanh, 1.0, 4.0), "sigmoid": (_sigmoid, 0.25, 4.0),
       "relu": (lambda v: np.maximum(v, 0.0), 1.0, 0.0), "identity": (lambda v: v, 1.0, 0.0)}


def act(name, a, dt):
    f, L, c = ACT[name]
    v = f(a[0])
    return v, L * a[1] + c * _u(dt) * np.abs(v) + _tiny(dt)


def act_bwd(name, g, pre, z, dt):
    """upstream g times sigma'(pre), with sigma' written in the output z = sigma(pre) as autograd does."""
    u = _u(dt)
    if name == "tanh":
        return mul(g, (1.0 - z[0] ** 2, 2.0 * np.abs(z[0]) * z[1] + 3.0 * u), dt)
    if name == "sigmoid":
        s = z[0]
        return mul(g, (s * (1.0 - s), np.abs(1.0 - 2.0 * s) * z[1] + 3.0 * u * s * (1.0 - s)), dt)
    if name == "relu":
        on = (pre[0] > 0).astype(np.float64)
        kink = np.abs(pre[0]) <= pre[1]
        return g[0] * on, g[1] * on + np.where(kink, np.abs(g[0]) + g[1], 0.0)
    assert name == "identity"
    return g


def _sum_to(v, shape):
    """v summed over the axes where `shape` (same rank) has extent 1 and v has more."""
    axes = tuple(i for i, (n, m) in enumerate(zip(v.shape, shape)) if m == 1 and n != 1)
    return v.sum(axis=axes, keepdims=True) if axes else v


def reduce_mul(a, b, shape, dt):
    """sum of a * b down to `shape` (the gradient of a broadcast factor): one product, then an n-term sum."""
    p = a[0] * b[0]
    bp = np.abs(a[0]) * b[1] + np.abs(b[0]) * a[1] + a[1] * b[1]
    v = _sum_to(p, shape)
    n = p.size // max(v.size, 1)
    return v, _sum_to(bp, shape) + orc.gamma(n + 1, dt) * _sum_to(np.abs(p), shape) + _tiny(dt) * (n + 1)


def reduce_sum(a, shape, dt):
    v = _sum_to(a[0], shape)
    n = a[0].size // max(v.size, 1)
    return v, _sum_to(a[1], shape) + orc.gamma(max(n, 1), dt) * _sum_to(np.abs(a[0]), shape) + _tiny(dt) * (n + 1)


def time_sum(terms, dt):
    """sum over time steps of (v, beta) parameter-gradient terms: sum beta_t + gamma_T sum |g_t|."""
    v = sum(t[0] for t in terms)
    return v, sum(t[1] for t in terms) + orc.gamma(len(terms), dt) * sum(np.abs(t[0]) for t in terms) + \
        _tiny(dt) * (len(terms) + 1)


def matmul(a, W, dt):
    """a [.., n] @ W [n, m], W = (v, beta_W)."""
    n = a[0].shape[-1]
    aa, aW = np.abs(a[0]), np.abs(W[0])
    v = a[0] @ W[0]
    return v, orc.gamma(max(n, 1), dt) * (aa @ aW) + a[1] @ aW + aa @ W[1] + a[1] @ W[1] + _tiny(dt) * (n + 1)


# ------------------------------------------------------------------------------------------------ LSIGF calls
def _abs_ops(S_list):
    return [abs(sp.csr_matrix(S_e)).astype(np.float64) for S_e in S_list]


def lsigf(h, S_list, x, b, dt):
    """y = LSIGF(h, S, x, b) for x = (v, beta) [B, G, N]; h, b exact in dt."""
    xv, xb = x
    B, _, N = xv.shape
    F = h.shape[0]
    y = orc.lsigf_sparse_stream(h, S_list, xv, b)
    env = orc.lsigf_envelope(h, S_list, np.abs(xv) + xb, b, np.zeros((B, F, N)), dt, tf32x3=dt == F32, stream=True)
    beta = env["y"]
    if np.any(xb):
        beta = beta + orc.lsigf_sparse_stream(np.abs(h), _abs_ops(S_list), xb)
    return y, beta


def lsigf_grads(h, S_list, x, dy, bshape, dt, drop_hop=None):
    """(dh, dx, db) of LSIGF(h, S, x, b) for x, dy = (v, beta) pairs; db None without a bias.  drop_hop=k: the dx of
    a defective kernel that leaves out the k-th hop (a planted bug)."""
    xv, xb = x
    dyv, dyb = dy
    dh, dx, db = orc.lsigf_grads_sparse_stream(h, S_list, xv, dyv, bshape)
    if drop_hop is not None:
        hk = h.copy()
        hk[:, :, drop_hop, :] = 0.0
        dx = orc.lsigf_grads_sparse_stream(hk, S_list, xv, dyv, None)[1]
    bz = None if bshape is None else np.zeros(bshape)
    env = orc.lsigf_envelope(h, S_list, np.abs(xv) + xb, bz, np.abs(dyv) + dyb, dt, tf32x3=dt == F32, stream=True)
    ah, aS = np.abs(h), _abs_ops(S_list)
    dh1, dx1, db1 = orc.lsigf_grads_sparse_stream(ah, aS, np.abs(xv), dyb, bshape)
    bdh = env["dh"] + dh1
    if np.any(xb):
        bdh = bdh + orc.lsigf_grads_sparse_stream(ah, aS, xb, np.abs(dyv) + dyb, None)[0]
    out_db = None if bshape is None else (db, env["db"] + db1)
    return (dh, bdh), (dx, env["dx"] + dx1), out_db


# ------------------------------------------------------------------------------------------------ GatedGRNN
def _gate(q, T):
    """None, a scalar or [B|1, T, 1, 1|N] (v, beta) -> None or a [B|1, T, 1, 1|N] pair."""
    if q is None:
        return None
    v, b = np.asarray(q[0], np.float64), np.asarray(q[1], np.float64)
    if v.size == 1:
        v, b = np.full((1, T, 1, 1), float(v.reshape(()))), np.full((1, T, 1, 1), float(b.reshape(())))
    return v, b


def grnn_forward(p, S_list, x, z0, sigma, dt, q_hat=None, q_check=None, bug=None):
    """GatedGRNN forward.  p: a [H, E, K, F], b [H, E, K, H], xb / zb [H, 1] or None (exact in dt); x [B, T, F, N],
    z0 [B, H, N] (v, beta) pairs or plain arrays; gates (v, beta) pairs or None.  Returns ctx; ctx["z"] = (v, beta) of
    the trajectory [B, T, H, N].  bug: "S^T" (the transposed GSO for the hidden hop of step 1), "z_t-2" (z_{t-2} in
    place of z_{t-1}), "gate_t+1" (the forget gate of step t+1 applied at step t), "no_zBias"."""
    x = x if isinstance(x, tuple) else exact(x)
    z0 = z0 if isinstance(z0, tuple) else exact(z0)
    a, b = p["a"], p["b"]
    H, E, K, F = a.shape
    B, T, _, N = x[0].shape
    qh, qc = _gate(q_hat, T), _gate(q_check, T)
    xr = (x[0].reshape(B * T, F, N), x[1].reshape(B * T, F, N))
    Ax = lsigf(a, S_list, xr, p.get("xb"), dt)
    Ax = (Ax[0].reshape(B, T, H, N), Ax[1].reshape(B, T, H, N))
    Axg = mul(qh, Ax, dt) if qh is not None else Ax
    S_T = [sp.csr_matrix(S_e).T.tocsr() for S_e in S_list] if bug == "S^T" else None
    zb = None if bug == "no_zBias" else p.get("zb")
    states, steps = [z0], []
    for t in range(T):
        zin = states[max(t - 1, 0)] if (bug == "z_t-2" and t >= 1) else states[t]
        Bz = lsigf(b, S_T if (bug == "S^T" and t == 1) else S_list, zin, zb, dt)
        q = None
        if qc is not None:
            tq = min(t + 1, T - 1) if bug == "gate_t+1" else t
            q = (qc[0][:, tq], qc[1][:, tq])
        Bzg = mul(q, Bz, dt) if q is not None else Bz
        pre = add((Axg[0][:, t], Axg[1][:, t]), Bzg, dt)
        z = act(sigma, pre, dt)
        steps.append(dict(zin=zin, Bz=Bz, q=q, pre=pre, z=z))
        states.append(z)
    zv = np.stack([s["z"][0] for s in steps], 1)
    zbeta = np.stack([s["z"][1] for s in steps], 1)
    return dict(p=p, S=S_list, x=x, xr=xr, z0=z0, sigma=sigma, dt=dt, qh=qh, qc=qc, Ax=Ax, steps=steps, z=(zv, zbeta),
                shape=(B, T, F, H, K, E, N))


def grnn_backward(ctx, dz, bug=None):
    """Reverse pass for upstream dz = (v, beta) [B, T, H, N].  Returns dict of (v, beta): dx, dz0, a, b, xb, zb (the
    parameter gradients, the biases when present) and dq_hat / dq_check for given gates.  bug: "dW_last" (the hidden taps'
    gradient without the last time step), "dz0_hop1" (dz0 without the first hop of step 0)."""
    dz = dz if isinstance(dz, tuple) else exact(dz)
    p, S_list, dt, sigma = ctx["p"], ctx["S"], ctx["dt"], ctx["sigma"]
    B, T, F, H, K, E, N = ctx["shape"]
    steps = ctx["steps"]
    zbs = None if p.get("zb") is None else (H, 1)
    dAxg = [None] * T
    db_t, dzb_t, dqc = [], [], [None] * T
    g_next = None
    for t in reversed(range(T)):
        s = steps[t]
        g = (dz[0][:, t], dz[1][:, t])
        if g_next is not None:
            g = add(g, g_next, dt)
        dpre = act_bwd(sigma, g, s["pre"], s["z"], dt)
        dAxg[t] = dpre
        dBz = dpre
        if s["q"] is not None:
            dqc[t] = reduce_mul(dpre, s["Bz"], s["q"][0].shape, dt)
            dBz = mul(s["q"], dpre, dt)
        dh, dx, dbias = lsigf_grads(p["b"], S_list, s["zin"], dBz, zbs, dt,
                                    drop_hop=1 if (bug == "dz0_hop1" and t == 0 and K > 1) else None)
        if not (bug == "dW_last" and t == T - 1):
            db_t.append(dh)
        if dbias is not None:
            dzb_t.append(dbias)
        g_next = dx
    out = dict(dz0=g_next, b=time_sum(db_t, dt))
    if dzb_t:
        out["zb"] = time_sum(dzb_t, dt)
    dAxg = (np.stack([d[0] for d in dAxg], 1), np.stack([d[1] for d in dAxg], 1))
    dAx = dAxg
    if ctx["qh"] is not None:
        out["dq_hat"] = reduce_mul(dAxg, ctx["Ax"], ctx["qh"][0].shape, dt)
        dAx = mul(ctx["qh"], dAxg, dt)
    if ctx["qc"] is not None:
        out["dq_check"] = (np.stack([d[0] for d in dqc], 1), np.stack([d[1] for d in dqc], 1))
    dAx = (dAx[0].reshape(B * T, H, N), dAx[1].reshape(B * T, H, N))
    xbs = None if p.get("xb") is None else (H, 1)
    da, dx, dxb = lsigf_grads(p["a"], S_list, ctx["xr"], dAx, xbs, dt)
    out["a"] = da
    out["dx"] = (dx[0].reshape(B, T, F, N), dx[1].reshape(B, T, F, N))
    if dxb is not None:
        out["xb"] = dxb
    return out


def grnn(p, S_list, x, z0, sigma, dt, q_hat=None, q_check=None, dz=None, bug=None):
    """GatedGRNN forward (and reverse pass when dz is given): dict with "z" and the gradients of grnn_backward."""
    ctx = grnn_forward(p, S_list, x, z0, sigma, dt, q_hat, q_check, bug)
    out = dict(z=ctx["z"])
    if dz is not None:
        out.update(grnn_backward(ctx, dz, bug))
    return out


# ------------------------------------------------------------------------------------------------ gated hidden states
def _sub(p, pre):
    """the GRNN parameters of p under the prefix `pre` (reference state_dict names) as grnn's dict."""
    out = dict(a=p[pre + "aWeights"], b=p[pre + "bWeights"])
    if pre + "xBias" in p:
        out["xb"], out["zb"] = p[pre + "xBias"], p[pre + "zBias"]
    return out


def _to_state(g, pre):
    names = dict(a="aWeights", b="bWeights", xb="xBias", zb="zBias")
    return {pre + names[k]: v for k, v in g.items() if k in names}


def _gate_map_forward(kind, p, which, zg, S_list, dt):
    """q = sigmoid(Linear(H*N -> 1)(z_gate[b, t])) (time) or sigmoid(GraphFilter(H -> 1)(z_gate)) (node)."""
    B, T, H, N = zg[0].shape
    if kind == "time":
        W = p[which + "FC.weight"]                                    # [1, H*N]
        c = p.get(which + "FC.bias")
        zr = (zg[0].reshape(B, T, H * N), zg[1].reshape(B, T, H * N))
        lin = matmul(zr, exact(W.T), dt)                              # [B, T, 1]
        if c is not None:
            lin = add(lin, exact(c.reshape(1, 1, 1)), dt)
        s = act("sigmoid", lin, dt)
        return (s[0][:, :, :, None], s[1][:, :, :, None]), dict(lin=lin, s=s, zr=zr)
    w = p[which + "GraphFilter.weight"]                               # [1, 1, K, H]
    c = p.get(which + "GraphFilter.bias")                             # [1, 1]
    zr = (zg[0].reshape(B * T, H, N), zg[1].reshape(B * T, H, N))
    lin = lsigf(w, S_list, zr, c, dt)                                 # [B*T, 1, N]
    s = act("sigmoid", lin, dt)
    return (s[0].reshape(B, T, 1, N), s[1].reshape(B, T, 1, N)), dict(lin=lin, s=s, zr=zr)


def _gate_map_backward(kind, p, which, st, dq, S_list, dt):
    """-> (d z_gate (v, beta) [B, T, H, N], {parameter name: gradient})."""
    out = {}
    if kind == "time":
        B, T, HN = st["zr"][0].shape
        dqs = (dq[0].reshape(B, T, 1), dq[1].reshape(B, T, 1))
        dlin = act_bwd("sigmoid", dqs, st["lin"], st["s"], dt)
        W = p[which + "FC.weight"]
        out[which + "FC.weight"] = reduce_mul(dlin, st["zr"], (1, 1, HN), dt)
        out[which + "FC.weight"] = (out[which + "FC.weight"][0].reshape(1, HN), out[which + "FC.weight"][1].reshape(1, HN))
        if which + "FC.bias" in p:
            db = reduce_sum(dlin, (1, 1, 1), dt)
            out[which + "FC.bias"] = (db[0].reshape(1), db[1].reshape(1))
        dzr = mul(dlin, exact(W.reshape(1, 1, HN)), dt)
        H = p["aWeights"].shape[0]
        return (dzr[0].reshape(B, T, H, HN // H), dzr[1].reshape(B, T, H, HN // H)), out
    BT, H, N = st["zr"][0].shape
    dqs = (dq[0].reshape(BT, 1, N), dq[1].reshape(BT, 1, N))
    dlin = act_bwd("sigmoid", dqs, st["lin"], st["s"], dt)
    c = p.get(which + "GraphFilter.bias")
    dw, dzr, dc = lsigf_grads(p[which + "GraphFilter.weight"], S_list, st["zr"], dlin, None if c is None else (1, 1), dt)
    out[which + "GraphFilter.weight"] = dw
    if dc is not None:
        out[which + "GraphFilter.bias"] = dc
    B = dq[0].shape[0]
    return (dzr[0].reshape(B, BT // B, H, N), dzr[1].reshape(B, BT // B, H, N)), out


def hidden_state(kind, p, S_list, x, z0, sigma, dt, dz=None, bug=None):
    """HiddenState (kind "plain"), TimeGatedHiddenState ("time") or NodeGatedHiddenState ("node") forward and, with dz,
    reverse pass.  p: the layer's state_dict as fp64 arrays (reference names).  Returns {"z", "zT", "dx", "dz0", and
    "g_<parameter name>" for every parameter}, each (v, beta)."""
    x, z0 = exact(x), exact(z0)
    gates = {}
    q = dict(inputGate=None, forgetGate=None)
    if kind != "plain":
        for which, pre in (("inputGate", "inputGateGRNN."), ("forgetGate", "forgetGateGRNN.")):
            gctx = grnn_forward(_sub(p, pre), S_list, x, z0, "tanh", dt)
            q[which], st = _gate_map_forward(kind, p, which, gctx["z"], S_list, dt)
            gates[which] = (gctx, st)
    main = grnn_forward(_sub(p, ""), S_list, x, z0, sigma, dt, q["inputGate"], q["forgetGate"], bug)
    z = main["z"]
    out = dict(z=z, zT=(z[0][:, -1:][:, None], z[1][:, -1:][:, None]))
    if dz is None:
        return out
    g = grnn_backward(main, dz, bug)
    dx, dz0 = g["dx"], g["dz0"]
    grads = _to_state(g, "")
    for which, pre, dq in (("inputGate", "inputGateGRNN.", "dq_hat"), ("forgetGate", "forgetGateGRNN.", "dq_check")):
        if which not in gates:
            continue
        gctx, st = gates[which]
        dzg, pg = _gate_map_backward(kind, p, which, st, g[dq], S_list, dt)
        grads.update(pg)
        gg = grnn_backward(gctx, dzg)
        grads.update(_to_state(gg, pre))
        dx, dz0 = add(dx, gg["dx"], dt), add(dz0, gg["dz0"], dt)
    out.update(dx=dx, dz0=dz0)
    out.update({"g_" + k: v for k, v in grads.items()})
    return out


# ------------------------------------------------------------------------------------------------ LSIGF_DB
def block_delay_ops(S, bug=None):
    """S [B, T, E, N, N] -> [S_big_e as scipy CSR, M x M], M = B*T*N:  S_big_e[(b, t-1, i), (b, t, j)] = S[b, t, e, i, j]
    (nothing enters t = 0).  bug: "S_t" (S(b, t-1) on the block that belongs to S(b, t)), "history" (the block of t = 0
    fed from (b, T-1) with S(b, 0))."""
    S = np.asarray(S, np.float64)
    B, T, E, N, _ = S.shape
    M = B * T * N
    out = []
    for e in range(E):
        rows, cols, vals = [], [], []
        for b in range(B):
            for t in range(T):
                if t == 0 and bug != "history":
                    continue
                src = (b * T + (t - 1) % T) * N
                blk = S[b, t - 1 if (bug == "S_t" and t >= 1) else t, e]
                i, j = np.nonzero(blk)
                rows.append(src + i)
                cols.append((b * T + t) * N + j)
                vals.append(blk[i, j])
        cat = lambda v, d: np.concatenate(v).astype(d) if v else np.zeros(0, d)  # noqa: E731
        out.append(sp.csr_matrix((cat(vals, np.float64), (cat(rows, np.int64), cat(cols, np.int64))), shape=(M, M)))
    return out


def lsigf_db(h, S, x, b, dt, dy=None, bug=None):
    """LSIGF_DB(h, S, x, b): h [F, E, K, G], S [B, T, E, N, N], x [B, T, G, N] (v, beta) or array, b None / [F, 1] /
    [F, N].  Returns {"y": (v, beta) [B, T, F, N]} and, with dy, "dh", "dx" and "db".  bug: those of block_delay_ops, or
    "bias_interleaved" (a per-node bias spread over the M space-time nodes by repeat_interleave instead of repeat)."""
    x = x if isinstance(x, tuple) else exact(x)
    F, E, K, G = h.shape
    B, T, _, N = x[0].shape
    M = B * T * N
    ops = block_delay_ops(S, bug)
    big = lambda v: v.transpose(0, 1, 3, 2).reshape(M, G).T[None]     # noqa: E731   [1, G, M]
    xb = (big(x[0]), big(x[1]))
    b_big = b
    if b is not None and b.shape[1] == N and M != N:
        b_big = np.repeat(b, B * T, axis=1) if bug == "bias_interleaved" else np.tile(b, (1, B * T))
    y = lsigf(h, ops, xb, b_big, dt)
    unbig = lambda v, C: v[0].reshape(C, B, T, N).transpose(1, 2, 0, 3)   # noqa: E731
    out = dict(y=(unbig(y[0], F), unbig(y[1], F)))
    if dy is None:
        return out
    dy = dy if isinstance(dy, tuple) else exact(dy)
    dyb = (dy[0].transpose(2, 0, 1, 3).reshape(1, F, M), dy[1].transpose(2, 0, 1, 3).reshape(1, F, M))
    dh, dx, db = lsigf_grads(h, ops, xb, dyb, None if b_big is None else b_big.shape, dt)
    out.update(dh=dh, dx=(unbig(dx[0], G), unbig(dx[1], G)))
    if db is not None:
        if b_big is not b:       # the per-node bias was repeated over the B*T copies: its gradient sums them
            db = reduce_sum((db[0].reshape(F, B * T, N), db[1].reshape(F, B * T, N)), (F, 1, N), dt)
            db = (db[0].reshape(F, N), db[1].reshape(F, N))
        out["db"] = db
    return out


# ------------------------------------------------------------------------------------------------ GRNN_DB
def slab_ops(S):
    """A_o for o = (t-1)*E + e, t = 1 .. T-1 (scipy CSR on R = B*N rows (b, n)): the block-diagonal S[b, t, e]."""
    S = np.asarray(S, np.float64)
    B, T, E, N, _ = S.shape
    out = []
    for t in range(1, T):
        for e in range(E):
            A = sp.block_diag([sp.csr_matrix(S[b, t, e]) for b in range(B)], format="csr")
            A.eliminate_zeros()                                           # the pattern is S != 0, as in slab_csr
            A.sort_indices()
            out.append(A)
    return out


def hop(A, src, dt):
    """dst = A src (the hop kernel over the rows of A, src = (v, beta))."""
    A = sp.csr_matrix(A)
    aA = abs(A)
    n = np.maximum(np.diff(A.indptr), 1)[:, None]
    return A @ src[0], orc.dot_bound(n, aA @ np.abs(src[0]), dt) + aA @ src[1]


def grnn_db(a, b, S, x, z0, sigma, dt, xb=None, zb=None, dz=None, bug=None):
    """GRNN_DB(a, b, S, x, z0, sigma, xBias, zBias) forward and, with dz, reverse pass; all arrays exact in dt.  Returns
    {"z"} and, with dz, {"dx", "dz0", "da", "db", "dxb", "dzb"} (biases when present), each (v, beta).  bug: "op+1" (the
    delay line advanced with operator o+1), "slot" (the last delay slot hopped from itself instead of from the slot
    before it), "swap_e" (the operators of e = 0 and e = 1 swapped), "dW_last", "dz0_hop1" (dz0 without the hop of step 1)."""
    H, E, K, F = a.shape
    B, T, _, N, _ = S.shape
    R = B * N
    A = slab_ops(S)
    n_ops = len(A)
    xbb = None if xb is None else xb.reshape(H, 1)
    Ax = lsigf_db(a, S, x, xbb, dt)["y"]                                 # [B, T, H, N]
    Ax_t = [(Ax[0][:, t].transpose(0, 2, 1), Ax[1][:, t].transpose(0, 2, 1)) for t in range(T)]   # [B, N, H]
    W0v = b[:, :, 0, :].sum(1).T                                         # [H, H']
    W0 = (W0v, orc.gamma(max(E - 1, 1), dt) * np.abs(b[:, :, 0, :]).sum(1).T if E > 1 else np.zeros_like(W0v))
    We = [exact(b[:, e, 1:, :].transpose(1, 2, 0).reshape((K - 1) * H, H)) for e in range(E)] if K > 1 else []
    rows = lambda v: v.transpose(0, 2, 1).reshape(R, H)                 # noqa: E731   [B, H, N] -> [R, H]
    Z = [exact(rows(z0))]                                                # Z[s] = z_{s-1} as rows
    D = []                                                               # D[t][e], delay lines of step t
    ops_of = {}
    steps = []
    for t in range(T):
        Bz = matmul(Z[t], W0, dt)
        Dt = [None] * E
        if t >= 1 and K > 1:
            for e in range(E):
                prev = D[t - 1][e]
                zp2 = Z[t - 1]
                if K > 2:
                    if prev is None:
                        tail = (np.zeros((R, (K - 2) * H)), np.zeros((R, (K - 2) * H)))
                    elif bug == "slot":
                        tail = (prev[0][:, H:], prev[1][:, H:])
                    else:
                        tail = (prev[0][:, :(K - 2) * H], prev[1][:, :(K - 2) * H])
                    src = (np.concatenate([zp2[0], tail[0]], 1), np.concatenate([zp2[1], tail[1]], 1))
                else:
                    src = zp2
                o = (t - 1) * E + (E - 1 - e if bug == "swap_e" else e)
                if bug == "op+1":
                    o = min(o + 1, n_ops - 1)
                ops_of[t, e] = (o, src)
                Dt[e] = hop(A[o].T.tocsr(), src, dt)
                Bz = add(Bz, matmul(Dt[e], We[e], dt), dt)
        D.append(Dt)
        pre = add((Ax_t[t][0], Ax_t[t][1]), (Bz[0].reshape(B, N, H), Bz[1].reshape(B, N, H)), dt)
        if zb is not None:
            pre = add(pre, exact(zb.reshape(1, 1, H)), dt)
        pre = (pre[0].transpose(0, 2, 1), pre[1].transpose(0, 2, 1))    # [B, H, N]
        z = act(sigma, pre, dt)
        steps.append(dict(pre=pre, z=z))
        Z.append((rows(z[0]), rows(z[1])))
    out = dict(z=(np.stack([s["z"][0] for s in steps], 1), np.stack([s["z"][1] for s in steps], 1)))
    if dz is None:
        return out
    dz = dz if isinstance(dz, tuple) else exact(dz)
    gZ = [None] * (T + 1)                       # gradient of Z[s] from later steps
    gD = [[None] * E for _ in range(T + 1)]     # gradient of D[t][e] from the source of step t+1
    dW0_t, dWe_t = [], [[] for _ in range(E)]
    dzb_t = []
    dAx = [None] * T

    def acc(cur, new):
        return new if cur is None else add(cur, new, dt)
    for t in reversed(range(T)):
        g = (dz[0][:, t], dz[1][:, t])
        if gZ[t + 1] is not None:
            gr = gZ[t + 1]
            g = add(g, (gr[0].reshape(B, N, H).transpose(0, 2, 1), gr[1].reshape(B, N, H).transpose(0, 2, 1)), dt)
        dpre = act_bwd(sigma, g, steps[t]["pre"], steps[t]["z"], dt)   # [B, H, N]
        dAx[t] = dpre
        dBz = (rows(dpre[0]), rows(dpre[1]))
        if zb is not None:
            dzb_t.append(reduce_sum(dBz, (1, H), dt))
        if not (bug == "dW_last" and t == T - 1):
            dW0_t.append(matmul((Z[t][0].T, Z[t][1].T), dBz, dt))
        gZ[t] = acc(gZ[t], matmul(dBz, (W0[0].T, W0[1].T), dt))
        if t >= 1 and K > 1:
            for e in range(E):
                gd = matmul(dBz, (We[e][0].T, We[e][1].T), dt)
                if gD[t][e] is not None:
                    gd = add(gd, gD[t][e], dt)
                Dv = D[t][e]
                if not (bug == "dW_last" and t == T - 1):
                    dWe_t[e].append(matmul((Dv[0].T, Dv[1].T), dBz, dt))
                o, _ = ops_of[t, e]
                gs = hop(A[o], gd, dt)
                if not (bug == "dz0_hop1" and t == 1):
                    gZ[t - 1] = acc(gZ[t - 1], (gs[0][:, :H], gs[1][:, :H]))
                if K > 2 and D[t - 1][e] is not None:
                    pad = np.zeros((R, H))
                    gD[t - 1][e] = (np.concatenate([gs[0][:, H:], pad], 1), np.concatenate([gs[1][:, H:], pad], 1))
    res = dict(out)
    g0 = gZ[0]
    res["dz0"] = (g0[0].reshape(B, N, H).transpose(0, 2, 1), g0[1].reshape(B, N, H).transpose(0, 2, 1))
    dW0 = time_sum(dW0_t, dt)                                            # [H, H']
    dbv, dbb = np.zeros_like(b), np.full_like(b, _tiny(dt))      # taps no step reaches (T = 1) stay exactly 0
    for e in range(E):
        dbv[:, e, 0, :], dbb[:, e, 0, :] = dW0[0].T, dW0[1].T
        if K > 1 and dWe_t[e]:
            dWe = time_sum(dWe_t[e], dt)                                 # [(K-1)*H, H']
            dbv[:, e, 1:, :] = dWe[0].reshape(K - 1, H, H).transpose(2, 0, 1)
            dbb[:, e, 1:, :] = dWe[1].reshape(K - 1, H, H).transpose(2, 0, 1)
    res["db"] = (dbv, dbb)
    if zb is not None:
        res["dzb"] = time_sum(dzb_t, dt)
        res["dzb"] = (res["dzb"][0].reshape(H, 1), res["dzb"][1].reshape(H, 1))
    dAx = (np.stack([d[0] for d in dAx], 1), np.stack([d[1] for d in dAx], 1))
    g = lsigf_db(a, S, x, xbb, dt, dy=dAx)
    res.update(da=g["dh"], dx=g["dx"])
    if xb is not None:
        res["dxb"] = g["db"]
    return res
