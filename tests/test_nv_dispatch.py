"""One case per dispatch branch of the node-variant filter's kernels (csrc/nv/nv.cu), each held to oracle/nv_oracle.py's
componentwise fp64 bound.

Every row names the kernels its branch must launch (regexes on the demangled name).  The GPU test runs the case once under
torch.profiler in the pytest process and holds it to tests/dispatch_harness.py's check_case: those kernels ran, every
output is within its bound, memory outside the kernels' contract kept its canary pattern, NaN in input pad columns
reached no output, and a second run is bit-identical.  This table owns the kernels of csrc/nv/
(tests/test_dispatch_tables.py).
"""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import lsigf_oracle as orc
from dispatch_harness import (F32, F64, NPD, SENT, Result, _check, _from_node_major, _graph, _launched, _lib, _st,
                              check_case)


def _nv_case(dtype, N, B, G, F, K, E, M, bias="F1", graph="rand", x_pad=3):
    """b200gf_nv_pack_taps + b200gf_nv_forward + b200gf_nv_backward through the C ABI against oracle/nv_oracle.py.
    x and dy carry NaN in x_pad pad columns; y, dx, W, dh and db start as SENT / NaN and are followed by canaries, the
    workspaces by 4 KB of 0x5A.  M < N: random node taps; M >= N: node n reads tap n (taps past N get exactly 0)."""
    memo = {}

    def run():
        import nv_oracle as nvo
        from gnn_b200 import nodevariant as nvm
        import gnn_b200
        cabi, lib = _lib()
        enum = cabi.F32 if dtype == F32 else cabi.F64
        npd = NPD[dtype]
        if not memo:
            m = _graph(graph, N)
            mats = [m] if E == 1 else [m, sp.csr_matrix(m.T)]
            mats = [sp.csr_matrix((a.data.astype(npd).astype(np.float64), a.indices, a.indptr), shape=a.shape) for a in mats]
            rng = np.random.default_rng(N + 7 * B + 31 * G + F + K + M)
            r = lambda shape: orc.biased_uniform(rng, shape).astype(npd).astype(np.float64)   # noqa: E731
            copy = rng.integers(0, M, N) if M < N else np.arange(N)
            h, x, dy = r((F, E, K, G, M)), r((B, G, N)), r((B, F, N))
            b = None if bias is None else r((F, 1) if bias == "F1" else (F, N))
            bshape = None if b is None else b.shape
            dxr, dhr, dbr = nvo.nv_backward(h, copy, mats, x, dy, bshape)
            memo.update(mats=mats, copy=copy, h=h, x=x, dy=dy, b=b, taps=nvm.TapMap(copy, M),
                        ref=dict(y=nvo.nv_forward(h, copy, mats, x, b), dx=dxr, dh=dhr, db=dbr),
                        env=nvo.nv_envelope(h, copy, mats, x, b, dy, npd),
                        gso=gnn_b200.SparseGSO.from_scipy(mats, dtype=dtype))
        plan = memo["gso"].plan("cuda")
        node_tap, tap_rowptr, tap_nodes = memo["taps"].on("cuda")
        T = 1 + E * (K - 1)
        pad = 4096 // torch.empty(0, dtype=dtype).element_size()
        dev = lambda a: torch.tensor(a, dtype=dtype, device="cuda")          # noqa: E731

        def node_major(t_bcn, ld):
            out = torch.full((N, ld), float("nan"), dtype=dtype, device="cuda")
            out[:, :t_bcn.shape[0] * t_bcn.shape[1]] = dev(np.transpose(t_bcn, (2, 0, 1)).reshape(N, -1))
            return out

        xl, yl = B * G + x_pad, B * F + x_pad
        x, dy = node_major(memo["x"], xl), node_major(memo["dy"], yl)
        hd = dev(memo["h"])
        bd = None if memo["b"] is None else dev(memo["b"])
        res = Result()
        Wb = torch.full((M * T * G * F + pad,), SENT, dtype=dtype, device="cuda")
        _check(lib.b200gf_nv_pack_taps(enum, hd.data_ptr(), Wb.data_ptr(), F, E, K, G, M, _st()))
        res.canaries.append(("W tail", Wb[M * T * G * F:]))
        wsb = lib.b200gf_nv_workspace_bytes(plan.handle, B, G, F, K, M, 0)
        ws = torch.full((wsb + 4096,), 0x5A, dtype=torch.uint8, device="cuda")
        y = torch.full((N + 1, yl), SENT, dtype=dtype, device="cuda")
        _check(lib.b200gf_nv_forward(plan.handle, x.data_ptr(), xl, Wb.data_ptr(), node_tap.data_ptr(), M,
                                     None if bd is None else bd.data_ptr(), 1 if bias == "FN" else 0, y.data_ptr(), yl,
                                     ws.data_ptr(), wsb, B, G, F, K, _st()))
        res.canaries += [("fwd ws tail", ws[wsb:]), ("y pad", y[:N, B * F:]), ("y row N", y[N:])]
        wsb2 = lib.b200gf_nv_workspace_bytes(plan.handle, B, G, F, K, M, 1)
        ws2 = torch.full((wsb2 + 4096,), 0x5A, dtype=torch.uint8, device="cuda")
        dx = torch.full((N + 1, xl), SENT, dtype=dtype, device="cuda")
        nh = F * E * K * G * M
        dhb = torch.full((nh + pad,), SENT, dtype=dtype, device="cuda")
        dhb[:nh] = float("nan")
        nb = 0 if bd is None else bd.numel()
        dbb = torch.full((nb + pad,), SENT, dtype=dtype, device="cuda")
        _check(lib.b200gf_nv_backward(plan.handle, dy.data_ptr(), yl, x.data_ptr(), xl, Wb.data_ptr(), node_tap.data_ptr(),
                                      M, tap_rowptr.data_ptr(), tap_nodes.data_ptr(), dx.data_ptr(), xl, dhb.data_ptr(),
                                      None if bd is None else dbb.data_ptr(), 1 if bias == "FN" else 0, ws2.data_ptr(),
                                      wsb2, B, G, F, K, _st()))
        res.canaries += [("bwd ws tail", ws2[wsb2:]), ("dx pad", dx[:N, B * G:]), ("dx row N", dx[N:]),
                         ("dh tail", dhb[nh:]), ("db tail", dbb[nb:])]
        yv, dxv = _from_node_major(y, B, F, N), _from_node_major(dx, B, G, N)
        dh = dhb[:nh].view(F, E, K, G, M)
        ref, env = memo["ref"], memo["env"]
        res.checks += [("y", yv, ref["y"], env["y"]), ("dx", dxv, ref["dx"], env["dx"]), ("dh", dh, ref["dh"], env["dh"])]
        res.outputs += [yv, dxv, dh]
        res.finite += [("y", yv), ("dx", dxv), ("dh (every element written)", dh)]
        if bd is not None:
            db = dbb[:nb].view(bd.shape)
            res.checks.append(("db", db, ref["db"], env["db"]))
            res.outputs.append(db)
        if M > N:                                  # taps no node reads: exactly 0
            assert bool((dh[..., N:] == 0).all()), "unused taps must get exactly 0"
        return res
    return run


def _nv_rows():
    def ks(t, stream=0, hops=True, add=False, stream_t=None):
        out = [r"nv_pack_taps_kernel<%s>" % t, r"nv_contract_kernel<%s,%d>" % (t, stream), r"nv_piece_scan_kernel",
               r"nv_tap_grad_partial_kernel<%s>" % t, r"nv_tap_grad_reduce_kernel<%s>" % t,
               r"nv_contract_kernel<%s,%d>" % (t, stream if stream_t is None else stream_t)]
        return out + ([r"nv_add_kernel<%s>" % t] if add else [])
    rows = [
        # F, G not multiples of 8 or 32; B = 8 (one batch tile), random node taps (M < N)
        ("nv-f32-B8-G9-F11-M300", _nv_case(F32, 3000, 8, 9, 11, 3, 1, 300), ks("float")),
        # B = 33: a partial batch tile; E = 2: the Horner chains summed; M = N and a per-node bias
        ("nv-f32-B33-G17-F5-E2-MeqN-biasFN", _nv_case(F32, 3000, 33, 17, 5, 3, 2, 3000, bias="FN"), ks("float", add=True)),
        ("nv-f32-B1-G13-F7-K4-E2", _nv_case(F32, 3000, 1, 13, 7, 4, 2, 700), ks("float", add=True)),
        # K = 1: no hops; M > N: taps past N read by no node
        ("nv-f64-B4-G6-F10-K1-MgtN", _nv_case(F64, 2000, 4, 6, 10, 1, 2, 2050, bias=None), ks("double")),
        ("nv-f64-B3-G5-F4-K3-E2", _nv_case(F64, 3000, 3, 5, 4, 3, 2, 90, bias="FN"), ks("double", add=True)),
        # tap blocks larger than shared memory: forward (T G F) and transposed (G F) both stream the taps
        ("nv-f32-oversized-G128-F128", _nv_case(F32, 2000, 2, 128, 128, 3, 1, 50), ks("float", stream=1)),
        ("nv-f64-oversized-fwd-only", _nv_case(F64, 2000, 2, 40, 40, 3, 2, 50), ks("double", stream=1, stream_t=0,
                                                                                    add=True)),
        # M = 1 at N > 20 000: the tap gradient takes many pieces; the 20 000-entry hub row and column
        ("nv-f64-M1-hub", _nv_case(F64, 24000, 2, 3, 5, 3, 1, 1), ks("double")),
        ("nv-f32-hub-M2400", _nv_case(F32, 24000, 4, 8, 8, 3, 1, 2400), ks("float")),
    ]
    for N in (1, 3, 7):
        rows.append(("nv-tinyN%d-f32" % N, _nv_case(F32, N, 2, 3, 2, 3, 1, N, graph="tiny"), ks("float")))
        rows.append(("nv-tinyN%d-f64-M1" % N, _nv_case(F64, N, 1, 2, 3, 2, 1, 1, graph="tiny"), ks("double")))
    return rows


NV_CASES = _nv_rows()


# ------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("cid,fn,kernels", NV_CASES, ids=[c[0] for c in NV_CASES])
def test_nv_dispatch(cid, fn, kernels):
    res1, names = _launched(fn)
    check_case(cid, fn, kernels, names, res1)
