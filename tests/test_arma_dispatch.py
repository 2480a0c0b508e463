"""One case per launch branch of the ARMA filter's kernels (csrc/arma/arma.cu), each held to oracle/arma_oracle.py's
componentwise fp64 bound by tests/dispatch_harness.py's check_case.  This table owns the kernels of csrc/arma/
(tests/test_dispatch_tables.py).

Every row calls b200gf_arma_forward (with saved states, and without: the inference ping-pong) and b200gf_arma_backward
through the C ABI and names the kernels its branch must launch.  The rows' launches are traced in a child process
(dispatch_harness.child_traced), so this table's profiling leaves the pytest process's profiler untouched.  Outputs
are checked against their bound; memory outside the contract must keep its canary pattern; NaN in input pad columns
must reach no output; a rerun must be bit-identical; and the inference forward must equal the training forward bit for
bit.
"""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import lsigf_oracle as orc
from dispatch_harness import (F32, F64, NPD, SENT, Result, _check, _from_node_major, _graph, _lib, _st, check_case,
                              child_traced)


def _arma_case(dtype, N, B, G, F, P, E, tMax, graph="rand", x_pad=3, diag="vary"):
    """b200gf_arma_forward (states kept, and the inference ping-pong) + b200gf_arma_backward against the oracle.  x and
    dU carry NaN in x_pad pad columns; out and dx start from seeded values (the ABI adds to them) and are followed by
    SENT canaries, as are dpsi, dvarphi and the states; the workspaces are followed by 4 KB of 0x5A."""
    memo = {}

    def run():
        import arma_oracle as ao
        import gnn_b200
        cabi, lib = _lib()
        npd = NPD[dtype]
        if not memo:
            m = _graph(graph, N)
            rng = np.random.default_rng(N + 7 * B + 31 * G + F + 5 * P + tMax)
            mats = []
            for e in range(E):
                a = m if e == 0 else sp.csr_matrix(m.T)
                a = sp.csr_matrix(a - sp.diags(a.diagonal()))
                dv = rng.uniform(-1, 1, N) if diag == "vary" else np.zeros(N)
                a = sp.csr_matrix((a + sp.diags(dv)).astype(npd).astype(np.float64))
                a.sort_indices()
                mats.append(a)
            stdv = 1. / np.sqrt(G * P)
            r = lambda a: np.asarray(a).astype(npd).astype(np.float64)      # noqa: E731
            psi, varphi = r(rng.uniform(1 + 1 / stdv, 1 + 2 / stdv, (F, E, P, G))), r(rng.uniform(-stdv, stdv, (F, E, P, G)))
            x, dU = r(orc.biased_uniform(rng, (B, G, N))), r(orc.biased_uniform(rng, (B, F, N)))
            base_u, base_dx = r(rng.uniform(-1, 1, (B, F, N))), r(rng.uniform(-1, 1, (B, G, N)))
            St, dd = ao.split_gso(mats)
            dx_ref, dpsi_ref, dvar_ref = ao._adjoints(psi, varphi, St, dd, x, dU, tMax)
            u_ref = ao.arma_chain_terms(psi, varphi, St, dd, x, tMax)
            phi0 = np.zeros((F, E, 1, G))
            env = ao.arma_envelope(psi, varphi, phi0, mats, x, None, dU, tMax, npd)
            uu = orc.unit_roundoff(npd)
            memo.update(psi=psi, varphi=varphi, x=x, dU=dU, base_u=base_u, base_dx=base_dx,
                        ref=dict(u=base_u + u_ref, dx=base_dx + dx_ref, dpsi=dpsi_ref, dvarphi=dvar_ref),
                        env=dict(u=env["y"] + 2 * uu * np.abs(base_u), dx=env["dx"] + 2 * uu * np.abs(base_dx),
                                 dpsi=env["dpsi"], dvarphi=env["dvarphi"]),
                        op=gnn_b200.ArmaOperator(gnn_b200.SparseGSO.from_scipy(mats, dtype=dtype)))
        op = memo["op"]
        plan = op.plan(list(range(E)), "cuda")
        d = op.diag(list(range(E)), "cuda")
        pad = 4096 // torch.empty(0, dtype=dtype).element_size()
        dev = lambda a: torch.tensor(a, dtype=dtype, device="cuda")            # noqa: E731

        def node_major(t_bcn, ld, fill=float("nan"), rows=N):
            out = torch.full((rows, ld), fill, dtype=dtype, device="cuda")
            out[:N, :t_bcn.shape[0] * t_bcn.shape[1]] = dev(np.transpose(t_bcn, (2, 0, 1)).reshape(N, -1))
            return out

        xl, ul = B * G + x_pad, B * F + x_pad
        x, dU = node_major(memo["x"], xl), node_major(memo["dU"], ul)
        psi, varphi = dev(memo["psi"]), dev(memo["varphi"])
        res = Result()
        nst = lib.b200gf_arma_workspace_bytes(plan.handle, B, G, F, P, tMax, 3)
        states = torch.full((nst // torch.empty(0, dtype=dtype).element_size() + pad,), SENT, dtype=dtype, device="cuda")
        ws = {}
        for what in (0, 1, 2):
            nb = lib.b200gf_arma_workspace_bytes(plan.handle, B, G, F, P, tMax, what)
            ws[what] = (torch.full((nb + 4096,), 0x5A, dtype=torch.uint8, device="cuda"), nb)
        outs = []
        for keep in (1, 0):
            out = node_major(memo["base_u"], ul, SENT, N + 1)
            w, nb = ws[keep]
            _check(lib.b200gf_arma_forward(plan.handle, d.data_ptr(), psi.data_ptr(), varphi.data_ptr(), tMax, B, G, F,
                                           P, x.data_ptr(), xl, out.data_ptr(), ul,
                                           states.data_ptr() if keep else None, w.data_ptr(), nb, _st()))
            res.canaries += [("fwd ws tail (keep=%d)" % keep, w[nb:]), ("out pad", out[:N, B * F:]), ("out row N", out[N:])]
            outs.append(out)
        res.canaries.append(("states tail", states[nst // states.element_size():]))
        dx = node_major(memo["base_dx"], xl, SENT, N + 1)
        ng = F * E * P * G
        dpsi = torch.full((ng + pad,), SENT, dtype=dtype, device="cuda")
        dvar = torch.full((ng + pad,), SENT, dtype=dtype, device="cuda")
        dpsi[:ng] = float("nan")
        dvar[:ng] = float("nan")
        w, nb = ws[2]
        _check(lib.b200gf_arma_backward(plan.handle, d.data_ptr(), psi.data_ptr(), varphi.data_ptr(), tMax, B, G, F, P,
                                        dU.data_ptr(), ul, states.data_ptr(), dx.data_ptr(), xl, dpsi.data_ptr(),
                                        dvar.data_ptr(), w.data_ptr(), nb, _st()))
        res.canaries += [("bwd ws tail", w[nb:]), ("dx pad", dx[:N, B * G:]), ("dx row N", dx[N:]),
                         ("dpsi tail", dpsi[ng:]), ("dvarphi tail", dvar[ng:])]
        uv, uv_inf, dxv = _from_node_major(outs[0], B, F, N), _from_node_major(outs[1], B, F, N), _from_node_major(dx, B, G, N)
        dpsiv, dvarv = dpsi[:ng].view(F, E, P, G), dvar[:ng].view(F, E, P, G)
        ref, env = memo["ref"], memo["env"]
        res.checks += [("u", uv, ref["u"], env["u"]), ("dx", dxv, ref["dx"], env["dx"]),
                       ("dpsi", dpsiv, ref["dpsi"], env["dpsi"]), ("dvarphi", dvarv, ref["dvarphi"], env["dvarphi"])]
        res.outputs += [uv, uv_inf, dxv, dpsiv, dvarv]
        res.finite += [("u", uv), ("dx", dxv), ("dpsi (every element written)", dpsiv), ("dvarphi", dvarv)]
        res.same = [("inference forward == training forward", uv_inf, uv)]
        return res
    return run


def _arma_rows():
    def ks(t, tMax, E=1):
        fwd = ([r"arma_scale_acc_kernel<%s,1>" % t] + ([r"arma_scale_acc_kernel<%s,0>" % t] if tMax else [])) * E * 2
        bwd = ([r"arma_bwd_step_kernel<%s,1>" % t] + ([r"arma_bwd_step_kernel<%s,0>" % t] if tMax else [])
               + [r"arma_fold_kernel<%s>" % t] * 2 + [r"arma_colsum_partial_kernel<%s>" % t,
                                                      r"arma_colsum_reduce_kernel<%s>" % t]) * E
        return fwd + bwd
    rows = [
        # odd ld (pad 3), P G = 6: no alignment of the (b, f) column blocks; tMax odd
        ("arma-f32-B2-G3-F2-P2-t3", _arma_case(F32, 3000, 2, 3, 2, 2, 1, 3), ks("float", 3)),
        # E = 2 (the second edge feature the transpose), P G = 5, tMax even >= 4
        ("arma-f32-B1-G5-F3-P1-E2-t4", _arma_case(F32, 3000, 1, 5, 3, 1, 2, 4), ks("float", 4, 2)),
        # tMax = 0: the seed alone, no wide hop; the backward's first step is also its last
        ("arma-f32-B3-G2-F4-P2-t0", _arma_case(F32, 3000, 3, 2, 4, 2, 1, 0), ks("float", 0)),
        # zero diagonal through the general kernels; aligned ld (pad 0)
        ("arma-f32-zero-diag-ld-aligned", _arma_case(F32, 3000, 2, 4, 2, 2, 1, 2, x_pad=0, diag="zero"), ks("float", 2)),
        ("arma-f64-B3-G2-F2-P3-E2-t1", _arma_case(F64, 3000, 3, 2, 2, 3, 2, 1), ks("double", 1, 2)),
        # the 20 000-entry hub row and column; more than 1024 row pieces in the column sums
        ("arma-f64-hub-t5", _arma_case(F64, 24000, 2, 4, 1, 2, 1, 5, x_pad=1), ks("double", 5)),
        ("arma-f32-hub-wide", _arma_case(F32, 24000, 4, 8, 4, 2, 1, 2), ks("float", 2)),
    ]
    for N in (1, 3, 7):
        rows.append(("arma-tinyN%d-f32" % N, _arma_case(F32, N, 2, 3, 2, 2, 1, 2, graph="tiny"), ks("float", 2)))
        rows.append(("arma-tinyN%d-f64-t0" % N, _arma_case(F64, N, 1, 2, 3, 1, 1, 0, graph="tiny"), ks("double", 0)))
    return rows


ARMA_CASES = _arma_rows()


# ------------------------------------------------------------------------------------------------------------ CPU
def test_the_abi_rejects_bad_arguments_before_any_cuda_call():
    """Null pointers, negative sizes, short leading dimensions and misaligned workspaces are EINVAL; a null plan sizes
    nothing."""
    _, lib = _lib()
    assert lib.b200gf_arma_workspace_bytes(None, 1, 1, 1, 1, 0, 0) == 0
    assert lib.b200gf_arma_forward(None, None, None, None, 0, 1, 1, 1, 1, None, 1, None, 1, None, None, 0, None) == -1
    assert lib.b200gf_arma_backward(None, None, None, None, 0, 1, 1, 1, 1, None, 1, None, None, 1, None, None, None, 0,
                                    None) == -1


# ------------------------------------------------------------------------------------------------------------ GPU
traced = child_traced("test_arma_dispatch", "ARMA_CASES")


@pytest.mark.gpu
@pytest.mark.parametrize("cid,fn,kernels", ARMA_CASES, ids=[c[0] for c in ARMA_CASES])
def test_arma_dispatch(cid, fn, kernels, traced):
    check_case(cid, fn, kernels, traced[cid])
