"""One case per kernel variant the host dispatch code can choose, each held to a componentwise fp64 bound.

Every row of CASES names an entry point, the shape / layout / alignment that selects a branch, and the kernels that
branch must launch (regexes on the demangled name, template arguments included).  The GPU test runs the case once under
torch.profiler in the pytest process and holds it to tests/dispatch_harness.py's check_case: those kernels ran, every
output is within oracle/lsigf_oracle.py's componentwise bound (oracle/ev_oracle.py's for the edge-variant filter),
memory outside the kernel's contract kept its canary pattern, and a second run is bit-identical.  This table owns the
kernels of csrc/*.cu and csrc/*.cuh except egate.cu: tests/test_dispatch_tables.py requires each of them to have a
case here or an entry in EXCLUDED.

Determinism exemption: maxpool_backward scatters with atomicAdd, so the order of its additions (and its last bits) may
change from run to run; its case checks only the bound.
"""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import ev_oracle as evo
import lsigf_oracle as orc
from dispatch_harness import (F32, F64, NPD, SENT, Result, _bits, _check, _from_node_major, _graph, _launched, _lib,
                              _padded, _st, check_case)


# ---------------------------------------------------------------------------------------------------------------- hop
def _hop_case(dtype, C, ld, N=3000, graph="rand", src_off=0, dst_off=0, plan_kind="full"):
    """b200gf_hop, both directions: src [n_cols, ld] with NaN in its pad columns, dst [n_rows + 3, ld] of SENT."""
    def run():
        import gnn_b200
        cabi, lib = _lib()
        m = _graph(graph, N)
        npd = NPD[dtype]
        mr = sp.csr_matrix((m.data.astype(npd).astype(np.float64), m.indices, m.indptr), shape=m.shape)
        if plan_kind == "full":
            gso = gnn_b200.SparseGSO.from_scipy([m], dtype=dtype)
            plan = gso.plan("cuda")
            ops = {cabi.HOP_FWD: mr.T.tocsr(), cabi.HOP_BWD: mr}
            n_rows = N
        else:   # partitioned: rows [r0, r1) of S^T and of S, global columns (the node-sharded path's plan)
            r0, r1 = N // 3, N // 3 + N // 2
            fwd, bwd = mr.T.tocsr()[r0:r1], mr[r0:r1]
            plan = gnn_b200.gso.Plan.from_ops([(fwd.indptr, fwd.indices, fwd.data)], [(bwd.indptr, bwd.indices, bwd.data)],
                                              r1 - r0, N, dtype, "cuda")
            assert plan.info(0) == r1 - r0 and plan.info(1) == N
            ops = {cabi.HOP_FWD: fwd, cabi.HOP_BWD: bwd}
            n_rows = r1 - r0
        if graph == "sym":
            assert plan.info(6) == 1
        g = torch.Generator(device="cpu").manual_seed(C * 7 + ld)
        X = torch.randn(N, C, generator=g, dtype=torch.float64).to(dtype)
        srcbuf = torch.full((N * ld + src_off + 8,), float("nan"), dtype=dtype, device="cuda")
        src = srcbuf[src_off:src_off + N * ld].view(N, ld)
        src[:, :C] = X.cuda()
        res = Result()
        Xd = X.double().numpy()
        for direction, op in ops.items():
            dstbuf = torch.full(((n_rows + 3) * ld + dst_off,), SENT, dtype=dtype, device="cuda")
            dst = dstbuf[dst_off:].view(n_rows + 3, ld)
            _check(lib.b200gf_hop(plan.handle, 0, direction, src.data_ptr(), ld, dst.data_ptr(), ld, C, _st()))
            ref = op @ Xd
            lens = np.diff(op.indptr)[:, None]
            res.checks.append(("dir%d" % direction, dst[:n_rows, :C], ref,
                               orc.dot_bound(np.maximum(lens, 1), abs(op) @ np.abs(Xd), npd)))
            # contract: columns [C, padded_ld(C)) may be written (whole tail vector), nothing at or past that
            res.canaries.append(("cols>=padded", dst[:, min(ld, _padded(C, dtype)):]))
            res.canaries.append(("rows>=n_rows", dst[n_rows:]))
            res.canaries.append(("before", dstbuf[:dst_off]))
            res.outputs.append(dst[:n_rows, :C])
            res.finite.append(("valid", dst[:n_rows, :C]))
        if graph == "sym":
            assert torch.equal(res.outputs[0], res.outputs[1]), "symmetric S: FWD and BWD must be bit-identical"
        return res
    return run


def _hop_rows():
    rows = []
    # (dtype, C, ld, kernel, extra)
    table = [
        (F32, 3, 3, r"spmm_hop_kernel<float,1,32,", {}),
        (F32, 4, 4, r"spmm_hop_multirow_kernel<float,4,1,8,", {}),
        (F32, 7, 8, r"spmm_hop_multirow_kernel<float,4,2,8,", {}),
        (F32, 13, 16, r"spmm_hop_multirow_v2_kernel<float,int,8,", {}),
        (F32, 13, 20, r"spmm_hop_multirow_kernel<float,4,4,16,", {}),
        (F32, 29, 32, r"spmm_hop_multirow_kernel<float,4,8,32,", {}),
        (F32, 61, 64, r"spmm_hop_v2_kernel<float,int,8,8,", {}),
        (F32, 100, 104, r"spmm_hop_v2_kernel<float,int,8,16,", {}),
        (F32, 1100, 1104, r"spmm_hop_v2_kernel<float,int,8,32,", {}),
        (F32, 61, 68, r"spmm_hop_kernel<float,4,16,", {}),
        (F32, 300, 308, r"spmm_hop_kernel<float,4,32,", {}),
        (F32, 61, 64, r"spmm_hop_kernel<float,4,16,", dict(src_off=4, dst_off=4)),   # 16- but not 32-byte aligned
        (F64, 3, 3, r"spmm_hop_kernel<double,1,32,", {}),
        (F64, 2, 2, r"spmm_hop_multirow_kernel<double,2,1,8,", {}),
        (F64, 3, 4, r"spmm_hop_multirow_kernel<double,2,2,8,", {}),
        (F64, 7, 8, r"spmm_hop_multirow_v2_kernel<double,int,4,", {}),
        (F64, 7, 10, r"spmm_hop_multirow_kernel<double,2,4,16,", {}),
        (F64, 15, 16, r"spmm_hop_multirow_kernel<double,2,8,32,", {}),
        (F64, 29, 32, r"spmm_hop_v2_kernel<double,int,4,8,", {}),
        (F64, 50, 52, r"spmm_hop_v2_kernel<double,int,4,16,", {}),
        (F64, 600, 600, r"spmm_hop_v2_kernel<double,int,4,32,", {}),
        (F64, 29, 34, r"spmm_hop_kernel<double,2,16,", {}),
        (F64, 150, 154, r"spmm_hop_kernel<double,2,32,", {}),
        (F64, 29, 32, r"spmm_hop_kernel<double,2,16,", dict(src_off=2, dst_off=2)),
    ]
    for dt, C, ld, k, extra in table:
        tag = "hop-%s-C%d-ld%d%s" % ("f32" if dt == F32 else "f64", C, ld, "-off" if extra else "")
        rows.append((tag, _hop_case(dt, C, ld, **extra), [k]))
    # the hub graph (20 000-entry row and column) on one kernel of every family
    for dt, C, ld, k in ((F32, 1100, 1104, r"spmm_hop_v2_kernel<float,int,8,32,"),
                         (F32, 13, 16, r"spmm_hop_multirow_v2_kernel<float,"),
                         (F32, 29, 32, r"spmm_hop_multirow_kernel<float,4,8,32,"),
                         (F32, 300, 308, r"spmm_hop_kernel<float,4,32,"),
                         (F64, 3, 3, r"spmm_hop_kernel<double,1,32,"),
                         (F64, 50, 52, r"spmm_hop_v2_kernel<double,int,4,16,")):
        rows.append(("hop-hub-%s-C%d" % ("f32" if dt == F32 else "f64", C), _hop_case(dt, C, ld, N=24000), [k]))
    # fewer rows than a warp handles
    for N in (1, 3, 7):
        rows.append(("hop-tinyN%d-f32" % N, _hop_case(F32, 7, 8, N=N, graph="tiny"), [r"spmm_hop_multirow_kernel<float,4,2,8,"]))
        rows.append(("hop-tinyN%d-f64-v2" % N, _hop_case(F64, 7, 8, N=N, graph="tiny"), [r"spmm_hop_multirow_v2_kernel<double,"]))
    rows.append(("hop-symmetric-f32", _hop_case(F32, 100, 104, graph="sym"), [r"spmm_hop_v2_kernel<float,int,8,16,"]))
    rows.append(("hop-symmetric-f64", _hop_case(F64, 15, 16, graph="sym"), [r"spmm_hop_multirow_kernel<double,2,8,32,"]))
    rows.append(("hop-partitioned-f32", _hop_case(F32, 61, 64, plan_kind="ops"), [r"spmm_hop_v2_kernel<float,int,8,8,"]))
    rows.append(("hop-partitioned-f64", _hop_case(F64, 3, 3, plan_kind="ops"), [r"spmm_hop_kernel<double,1,32,"]))
    return rows


# ------------------------------------------------------------------------------------------------ tap contraction
def _contract_case(dtype, n_rows, B, P, Q, T, bias="none", accumulate=0, out_pad=4, out_off=0, z_pad=0, tc=False,
                   scratch=True):
    """b200gf_tap_contract: Z_t [n_rows, B*P + z_pad] (NaN in the pad), out [n_rows + 2, B*Q + out_pad] of SENT."""
    def run():
        cabi, lib = _lib()
        rng = np.random.default_rng(n_rows * 131 + P * 7 + Q + T)
        enum = cabi.F32 if dtype == F32 else cabi.F64
        zl = B * P + z_pad
        Zs = [torch.full((n_rows, zl), float("nan"), dtype=dtype, device="cuda") for _ in range(T)]
        for Z in Zs:
            Z[:, :B * P] = torch.tensor(orc.biased_uniform(rng, (n_rows, B * P)), dtype=dtype)
        W = torch.tensor(orc.biased_uniform(rng, (T, P, Q)), dtype=dtype, device="cuda")
        bt = {"none": None, "q": (Q,), "qn": (Q, n_rows)}[bias]
        bvec = None if bt is None else torch.tensor(orc.biased_uniform(rng, bt), dtype=dtype, device="cuda")
        ol = B * Q + out_pad
        obuf = torch.full(((n_rows + 2) * ol + out_off,), SENT, dtype=dtype, device="cuda")
        out = obuf[out_off:].view(n_rows + 2, ol)
        y0 = None
        if accumulate:
            y0 = torch.tensor(orc.biased_uniform(rng, (n_rows, B * Q)), dtype=dtype, device="cuda")
            out[:n_rows, :B * Q] = y0
        sb = lib.b200gf_tap_contract_scratch_bytes(T, P, Q)
        scr = torch.empty(sb, dtype=torch.uint8, device="cuda") if scratch else None
        _check(lib.b200gf_tap_contract(enum, n_rows, B, P, Q, T, cabi.ptr_array([z.data_ptr() for z in Zs]),
                                       cabi.i64_array([zl] * T), W.data_ptr(), 0 if bvec is None else bvec.data_ptr(),
                                       1 if bias == "qn" else 0, out.data_ptr(), ol, accumulate,
                                       scr.data_ptr() if scratch else None, sb if scratch else 0, _st()))
        # fp64 reference on the GPU: rows (n, b) -> [n_rows * B, P]
        ref = torch.zeros(n_rows * B, Q, dtype=F64, device="cuda")
        absr = torch.zeros_like(ref)
        for t in range(T):
            Zt = Zs[t][:, :B * P].double().reshape(n_rows * B, P)
            ref += Zt @ W[t].double()
            absr += Zt.abs() @ W[t].double().abs()
        if bvec is not None:
            bb = bvec.double()
            badd = bb[None, :] if bias == "q" else bb.t().repeat_interleave(B, dim=0)
            ref += badd
            absr += badd.abs()
        ref = ref.reshape(n_rows, B * Q)
        absr = absr.reshape(n_rows, B * Q)
        if y0 is not None:
            ref += y0.double()
            absr += y0.double().abs()
        res = Result()
        n = T * P + 1 + (1 if accumulate else 0)
        res.checks.append(("out", out[:n_rows, :B * Q], ref.cpu().numpy(),
                           orc.dot_bound(n, absr.cpu().numpy(), NPD[dtype], tf32x3=tc)))
        res.canaries += [("cols>=B*Q", out[:, B * Q:]), ("rows>=n_rows", out[n_rows:]), ("before", obuf[:out_off])]
        res.outputs.append(out[:n_rows, :B * Q])
        res.finite.append(("valid", out[:n_rows, :B * Q]))
        return res
    return run


def _contract_rows():
    tcr = lambda np_: [r"tc_contract_kernel<%d>" % np_, r"split_w_kernel"]   # noqa: E731
    fma32 = [r"tap_contract_kernel<float>"]
    fma64 = [r"tap_contract_kernel<double>"]
    rows = [
        # wgmma: every N (NP = Q rounded up to a power of two), Q not a power of two (B-tile rows the TMA never writes),
        # T = 1 and 16 (MAX_T), R = 128 / 129 / > 132 tiles, B > 1, bias none / [Q] / [Q, N]
        ("tc-Q16-P32-T1-R129", _contract_case(F32, 129, 1, 32, 16, 1, tc=True), tcr(16)),
        ("tc-Q48-P96-T16-B2-biasq", _contract_case(F32, 300, 2, 96, 48, 16, bias="q", tc=True), tcr(64)),
        ("tc-Q80-P32-T16-R128-biasqn", _contract_case(F32, 128, 1, 32, 80, 16, bias="qn", tc=True), tcr(128)),
        ("tc-Q96-P288-T1-B2-multitile", _contract_case(F32, 20000, 2, 288, 96, 1, bias="q", tc=True), tcr(128)),
        ("tc-Q128-P32-T16-B2-141tiles", _contract_case(F32, 9000, 2, 32, 128, 16, bias="qn", tc=True), tcr(128)),
        ("tc-Q144-P96-T1-B3", _contract_case(F32, 129, 3, 96, 144, 1, tc=True), tcr(256)),
        ("tc-Q240-P32-T16-biasqn", _contract_case(F32, 200, 1, 32, 240, 16, bias="qn", tc=True), tcr(256)),
        ("tc-Q256-P96-T16-biasq", _contract_case(F32, 1000, 1, 96, 256, 16, bias="q", tc=True), tcr(256)),
        ("tc-Q32-P288-T1-B4", _contract_case(F32, 700, 4, 288, 32, 1, tc=True), tcr(32)),
        # fallbacks to the FMA kernel, still correct
        ("fma-f32-T17", _contract_case(F32, 300, 1, 32, 64, 17), fma32),
        ("fma-f32-Q272", _contract_case(F32, 300, 1, 32, 272, 1, bias="q"), fma32),
        ("fma-f32-R127", _contract_case(F32, 127, 1, 32, 64, 2), fma32),
        ("fma-f32-misaligned-out", _contract_case(F32, 300, 1, 32, 64, 2, out_off=1), fma32),
        ("fma-f32-no-scratch", _contract_case(F32, 300, 1, 32, 64, 2, scratch=False), fma32),
        ("fma-f32-padded-z", _contract_case(F32, 300, 2, 32, 64, 2, z_pad=4), fma32),
        # FMA with T > 48 (TermList::MAX_TERMS): bias only in chunk 0, accumulate into later chunks
        ("fma-f32-T49-acc0-biasq", _contract_case(F32, 150, 2, 20, 70, 49, bias="q"), fma32),
        ("fma-f32-T53-acc1-biasqn", _contract_case(F32, 150, 1, 20, 70, 53, bias="qn", accumulate=1), fma32),
        ("fma-f64-T49-acc1", _contract_case(F64, 150, 2, 20, 70, 49, bias="q", accumulate=1), fma64),
        ("fma-f64-T53-acc0-biasqn", _contract_case(F64, 150, 1, 20, 70, 53, bias="qn"), fma64),
        ("fma-f64-P13-Q5", _contract_case(F64, 77, 3, 13, 5, 3, bias="q"), fma64),
        # DMMA (fp64): QB = 32, two and three 64-column blocks, P = 16 / 48, T = 16, the shared-memory limit
        ("dmma-Q32-P16-T16", _contract_case(F64, 300, 1, 16, 32, 16, bias="q"), [r"contract_f64_kernel<4>"]),
        ("dmma-Q128-P16-T16-B2", _contract_case(F64, 400, 2, 16, 128, 16, bias="qn"), [r"contract_f64_kernel<8>"]),
        ("dmma-Q192-P48-T5", _contract_case(F64, 500, 1, 48, 192, 5, bias="q"), [r"contract_f64_kernel<8>"]),
        # the taps of one 64-column block stay in shared memory: T P (64 + 4) 8 + 40 KB <= 227 KB, i.e. T P <= 352
        ("dmma-Q128-P48-T16-over-limit", _contract_case(F64, 400, 2, 48, 128, 16, bias="qn"), fma64),
        ("dmma-Q64-P32-T11-smem-limit", _contract_case(F64, 300, 1, 32, 64, 11), [r"contract_f64_kernel<8>"]),
        ("dmma-Q64-P32-T12-over-limit", _contract_case(F64, 300, 1, 32, 64, 12), fma64),
        ("dmma-Q64-T17-fma", _contract_case(F64, 300, 1, 16, 64, 17), fma64),
    ]
    return rows


# ----------------------------------------------------------------------------------------------------- tap gradient
def _tap_grad_case(dtype, n_rows, B, P, Q, T, a_pad=0, v_pad=0):
    """b200gf_tap_grad: dW[t] = A^T V_t over rows (n, b); A [n_rows, B*P + a_pad], V_t [n_rows, B*Q + v_pad] (NaN pads)."""
    def run():
        cabi, lib = _lib()
        rng = np.random.default_rng(n_rows + P * 3 + Q * 5 + T)
        enum = cabi.F32 if dtype == F32 else cabi.F64
        al, vl = B * P + a_pad, B * Q + v_pad
        A = torch.full((n_rows, al), float("nan"), dtype=dtype, device="cuda")
        A[:, :B * P] = torch.tensor(orc.biased_uniform(rng, (n_rows, B * P)), dtype=dtype)
        Vs = [torch.full((n_rows, vl), float("nan"), dtype=dtype, device="cuda") for _ in range(T)]
        for V in Vs:
            V[:, :B * Q] = torch.tensor(orc.biased_uniform(rng, (n_rows, B * Q)), dtype=dtype)
        sb = lib.b200gf_tap_grad_scratch_bytes(enum, n_rows, B, P, Q, T)
        scr = torch.empty(sb, dtype=torch.uint8, device="cuda")
        dWbuf = torch.full((T * P * Q + 64,), SENT, dtype=dtype, device="cuda")
        _check(lib.b200gf_tap_grad(enum, n_rows, B, P, Q, T, A.data_ptr(), al, cabi.ptr_array([v.data_ptr() for v in Vs]),
                                   cabi.i64_array([vl] * T), dWbuf.data_ptr(), scr.data_ptr(), sb, _st()))
        Ad = A[:, :B * P].double().reshape(n_rows * B, P)
        ref = torch.stack([Ad.t() @ V[:, :B * Q].double().reshape(n_rows * B, Q) for V in Vs])
        absr = torch.stack([Ad.abs().t() @ V[:, :B * Q].double().abs().reshape(n_rows * B, Q) for V in Vs])
        res = Result()
        dW = dWbuf[:T * P * Q].view(T, P, Q)
        res.checks.append(("dW", dW, ref.cpu().numpy(), orc.dot_bound(n_rows * B, absr.cpu().numpy(), NPD[dtype])))
        res.canaries.append(("past dW", dWbuf[T * P * Q:]))
        res.outputs.append(dW)
        return res
    return run


def _tap_grad_rows():
    red = [r"tap_grad_reduce_kernel<float>"]
    mk = lambda *tpb: [r"tap_grad_multi_kernel<%d>" % t for t in tpb] + red   # noqa: E731
    rows = []
    for T in (1, 2, 3, 4, 5):
        rows.append(("tapgrad-f32-T%d-P64-Q64-R200" % T, _tap_grad_case(F32, 100, 2, 64, 64, T), mk(T)))
    rows += [
        ("tapgrad-f32-T9-P60-Q68", _tap_grad_case(F32, 2000, 2, 60, 68, 9), mk(5, 4)),
        ("tapgrad-f32-T48-P4-Q4", _tap_grad_case(F32, 3000, 1, 4, 4, 48), mk(3)),
        ("tapgrad-f32-T49-P4-Q60-split", _tap_grad_case(F32, 3000, 1, 4, 60, 49), mk(1, 3)),
        ("tapgrad-f32-T3-P68-Q60-chunks", _tap_grad_case(F32, 60000, 2, 68, 60, 3, a_pad=4, v_pad=8), mk(3)),
        ("tapgrad-f32-T2-P64-Q4-one-chunk", _tap_grad_case(F32, 100, 1, 64, 4, 2), mk(2)),
        ("tapgrad-f32-generic-P6", _tap_grad_case(F32, 3000, 2, 6, 64, 3), [r"tap_grad_partial_kernel<float>"]),
        ("tapgrad-f32-generic-vld", _tap_grad_case(F32, 3000, 1, 64, 64, 2, v_pad=1), [r"tap_grad_partial_kernel<float>"]),
        ("tapgrad-f64-T49-P60-Q4", _tap_grad_case(F64, 3000, 2, 60, 4, 49),
         [r"tap_grad_partial_kernel<double>", r"tap_grad_reduce_kernel<double>"]),
        ("tapgrad-f64-chunks", _tap_grad_case(F64, 60000, 1, 68, 64, 2, a_pad=2), [r"tap_grad_partial_kernel<double>"]),
    ]
    return rows


# ------------------------------------------------------------------------------ LSIGF through the C ABI (and dbias)
def _eye_plan(dtype, N):
    import gnn_b200
    rng = np.random.default_rng(N)
    m = sp.diags(rng.uniform(0.5, 1.5, N)).tocsr()
    return gnn_b200.SparseGSO.from_scipy([m], dtype=dtype).plan("cuda")


def _bias_grad_case(dtype, N, B, F, dy_pad=0, per_node=False):
    """dbias of b200gf_backward (K = 1, G = 1): db[f] = sum_{n,b} dy[n, b*F + f] or per node db[f, n] = sum_b dy."""
    def run():
        cabi, lib = _lib()
        rng = np.random.default_rng(N + F + dy_pad)
        plan = _eye_plan(dtype, N)
        G, K = 1, 1
        ld = B * F + dy_pad
        dy = torch.full((N, ld), float("nan"), dtype=dtype, device="cuda")
        dy[:, :B * F] = torch.tensor(orc.biased_uniform(rng, (N, B * F)), dtype=dtype)
        x = torch.tensor(rng.standard_normal((N, B * G)), dtype=dtype, device="cuda")
        h = torch.tensor(rng.standard_normal((F, 1, K, G)), dtype=dtype, device="cuda")
        dh = torch.empty(F, 1, K, G, dtype=dtype, device="cuda")
        nb = F * N if per_node else F
        dbb = torch.full((nb + 64,), SENT, dtype=dtype, device="cuda")
        wsb = lib.b200gf_workspace_bytes(plan.handle, B, G, F, K, cabi.NODE_MAJOR, 1)
        ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
        _check(lib.b200gf_backward(plan.handle, dy.data_ptr(), cabi.NODE_MAJOR, ld, x.data_ptr(), cabi.NODE_MAJOR, B * G,
                                   h.data_ptr(), None, 0, 0, dh.data_ptr(), dbb.data_ptr(), 1 if per_node else 0,
                                   ws.data_ptr(), wsb, B, G, F, K, _st()))
        dyv = dy[:, :B * F].double().reshape(N, B, F)
        if per_node:
            ref, absr, n = dyv.sum(1).t(), dyv.abs().sum(1).t(), B
        else:
            ref, absr, n = dyv.sum((0, 1)), dyv.abs().sum((0, 1)), N * B
        res = Result()
        db = dbb[:nb].view(ref.shape)
        res.checks.append(("db", db, ref.cpu().numpy(), orc.dot_bound(n, absr.cpu().numpy(), NPD[dtype])))
        res.canaries.append(("past db", dbb[nb:]))
        res.outputs.append(db)
        return res
    return run


def _bias_grad_rows():
    vec = [r"bias_grad_partial_vec_kernel", r"bias_grad_reduce_kernel<float>"]
    gen32 = [r"bias_grad_partial_kernel<float>", r"bias_grad_reduce_kernel<float>"]
    rows = []
    for F in (4, 64, 1024):
        rows.append(("biasgrad-vec-F%d-N2049" % F, _bias_grad_case(F32, 2049, 2, F), vec))
    for N in (2047, 2048, 2049):
        rows.append(("biasgrad-vec-F64-B1-N%d" % N, _bias_grad_case(F32, N, 1, 64), vec))
        rows.append(("biasgrad-generic-F12-N%d" % N, _bias_grad_case(F32, N, 2, 12), gen32))
    rows += [
        ("biasgrad-generic-F1028", _bias_grad_case(F32, 2049, 1, 1028), gen32),
        ("biasgrad-generic-F64-padded-ld", _bias_grad_case(F32, 2049, 2, 64, dy_pad=4), gen32),
        ("biasgrad-f64-F64", _bias_grad_case(F64, 2049, 2, 64), [r"bias_grad_partial_kernel<double>",
                                                                 r"bias_grad_reduce_kernel<double>"]),
        ("biasgrad-node-f32", _bias_grad_case(F32, 2049, 3, 12, per_node=True), [r"bias_grad_node_kernel<float>"]),
        ("biasgrad-node-f64", _bias_grad_case(F64, 2049, 3, 12, dy_pad=2, per_node=True), [r"bias_grad_node_kernel<double>"]),
    ]
    return rows


def _random_gso(N, E, seed, dtype, avg_deg=6):
    import gnn_b200
    rng = np.random.default_rng(seed)
    mats = []
    for _ in range(E):
        m = sp.random(N, N, density=avg_deg / N, format="csr", random_state=rng, data_rvs=rng.standard_normal)
        m = m / max(abs(m).sum(axis=1).max(), 1.0)
        mats.append(sp.csr_matrix(m))
    gso = gnn_b200.SparseGSO.from_scipy(mats, dtype=dtype)
    rounded = [sp.csr_matrix((c[2].astype(np.float64), c[1], c[0]), shape=(N, N)) for c in gso.csr]
    return gso, rounded


def _lsigf_abi_case(dtype, N, B, G, F, K, E, layout, act=0, bias="F1"):
    """b200gf_forward_act + b200gf_backward through the C ABI in one layout, with 4 KB of SENT past each workspace."""
    def run():
        cabi, lib = _lib()
        gso, S = _random_gso(N, E, N + G + F + K, dtype)
        plan = gso.plan("cuda")
        rng = np.random.default_rng(K)
        rnd = lambda a: torch.tensor(a, dtype=dtype)                                    # noqa: E731
        h = rnd(rng.uniform(-1, 1, (F, E, K, G)) / np.sqrt(G * K))
        x = rnd(rng.standard_normal((B, G, N)))
        b = rnd(rng.uniform(-0.5, 0.5, (F, 1) if bias == "F1" else (F, N)))
        dy = rnd(rng.standard_normal((B, F, N)))
        H, Xd, Bd, DY = (t.double().numpy() for t in (h, x, b, dy))
        fm = layout == cabi.FEATURE_MAJOR
        to_dev = lambda t_bfn, ld: (t_bfn.cuda().contiguous() if fm else _node_major(t_bfn, ld))  # noqa: E731
        xl, yl = _padded(B * G, dtype), _padded(B * F, dtype)
        xd, dyd = to_dev(x, xl), to_dev(dy, yl)
        hd, bd = h.cuda(), b.cuda().contiguous()
        res = Result()
        # forward
        wsb = lib.b200gf_workspace_bytes(plan.handle, B, G, F, K, layout, 0)
        ws = torch.full((wsb + 4096,), 0x5A, dtype=torch.uint8, device="cuda")
        y = torch.full((B, F, N) if fm else (N + 1, yl), SENT, dtype=dtype, device="cuda")
        _check(lib.b200gf_forward_act(plan.handle, xd.data_ptr(), layout, 0 if fm else xl, hd.data_ptr(), bd.data_ptr(),
                                      0 if bias == "F1" else 1, y.data_ptr(), layout, 0 if fm else yl, ws.data_ptr(), wsb,
                                      B, G, F, K, act, _st()))
        res.canaries.append(("fwd ws tail", ws[wsb:]))
        # backward
        wsb2 = lib.b200gf_workspace_bytes(plan.handle, B, G, F, K, layout, 1)
        ws2 = torch.full((wsb2 + 4096,), 0x5A, dtype=torch.uint8, device="cuda")
        dx = torch.full((B, G, N) if fm else (N + 1, xl), SENT, dtype=dtype, device="cuda")
        dh = torch.empty(F, E, K, G, dtype=dtype, device="cuda")
        db = torch.empty_like(bd)
        _check(lib.b200gf_backward(plan.handle, dyd.data_ptr(), layout, 0 if fm else yl, xd.data_ptr(), layout,
                                   0 if fm else xl, hd.data_ptr(), dx.data_ptr(), layout, 0 if fm else xl, dh.data_ptr(),
                                   db.data_ptr(), 0 if bias == "F1" else 1, ws2.data_ptr(), wsb2, B, G, F, K, _st()))
        res.canaries.append(("bwd ws tail", ws2[wsb2:]))
        y_ref = orc.lsigf_sparse(H, S, Xd, Bd)
        dh_ref, dx_ref, db_ref = orc.lsigf_grads_sparse(H, S, Xd, DY, Bd.shape)
        env = orc.lsigf_envelope(H, S, Xd, Bd, DY, NPD[dtype], tf32x3=dtype == F32)
        if act:
            y_ref = np.maximum(y_ref, 0.0)
        yv = y if fm else _from_node_major(y, B, F, N)
        dxv = dx if fm else _from_node_major(dx, B, G, N)
        res.checks += [("y", yv, y_ref, env["y"]), ("dx", dxv, dx_ref, env["dx"]), ("dh", dh, dh_ref, env["dh"]),
                       ("db", db, db_ref, env["db"])]
        if not fm:
            res.canaries += [("y pad", y[:N, B * F:]), ("y row N", y[N:]), ("dx pad", dx[:N, B * G:]), ("dx row N", dx[N:])]
        res.outputs += [yv, dxv, dh, db]
        res.finite += [("y", yv), ("dx", dxv)]
        return res
    return run


def _node_major(t_bfn, ld):
    """[B, C, N] host tensor -> node-major [N, ld] on the GPU with NaN in the pad columns."""
    B, C, N = t_bfn.shape
    out = torch.full((N, ld), float("nan"), dtype=t_bfn.dtype, device="cuda")
    out[:, :B * C] = t_bfn.permute(2, 0, 1).reshape(N, B * C).cuda()
    return out


def _lsigf_autograd_case(dtype, N, B, G, F, K, E, bias="F1"):
    """gnn_b200.LSIGF forward + autograd backward against the sparse oracle and its envelope."""
    def run():
        import gnn_b200
        gso, S = _random_gso(N, E, 3 * N + G + F + K, dtype)
        rng = np.random.default_rng(G * F + K)
        dev = lambda a: torch.tensor(a, dtype=dtype, device="cuda").requires_grad_(True)   # noqa: E731
        h = dev(rng.uniform(-1, 1, (F, E, K, G)) / np.sqrt(G * K))
        x = dev(rng.standard_normal((B, G, N)))
        b = dev(rng.uniform(-0.5, 0.5, (F, 1) if bias == "F1" else (F, N)))
        dy = torch.tensor(rng.standard_normal((B, F, N)), dtype=dtype, device="cuda")
        y = gnn_b200.LSIGF(h, gso, x, b)
        y.backward(dy)
        H, Xd, Bd, DY = (t.detach().double().cpu().numpy() for t in (h, x, b, dy))
        y_ref = orc.lsigf_sparse(H, S, Xd, Bd)
        dh_ref, dx_ref, db_ref = orc.lsigf_grads_sparse(H, S, Xd, DY, Bd.shape)
        env = orc.lsigf_envelope(H, S, Xd, Bd, DY, NPD[dtype], tf32x3=dtype == F32)
        res = Result()
        res.checks += [("y", y.detach(), y_ref, env["y"]), ("dx", x.grad, dx_ref, env["dx"]),
                       ("dh", h.grad, dh_ref, env["dh"]), ("db", b.grad, db_ref, env["db"])]
        res.outputs += [y.detach(), x.grad, h.grad, b.grad]
        return res
    return run


def _lsigf_rows():
    return [
        # (G, F) = (48, 64): forward FMA (P = 48), dx on the tensor cores with Q = 48; (64, 48) the reverse
        ("lsigf-f32-G48-F64", _lsigf_autograd_case(F32, 600, 2, 48, 64, 3, 2),
         [r"tap_contract_kernel<float>", r"tc_contract_kernel<64>", r"pack_taps_split_kernel", r"pack_taps_kernel<float>",
          r"tap_grad_multi_kernel<5>", r"tap_grad_reduce_kernel<float>"]),
        ("lsigf-f32-G64-F48", _lsigf_autograd_case(F32, 600, 2, 64, 48, 3, 2),
         [r"tc_contract_kernel<64>", r"tap_contract_kernel<float>"]),
        ("lsigf-f32-T16", _lsigf_autograd_case(F32, 500, 1, 32, 32, 6, 3), [r"tc_contract_kernel<32>"]),
        ("lsigf-f32-T17", _lsigf_autograd_case(F32, 500, 1, 32, 32, 9, 2), [r"tap_contract_kernel<float>"]),
        ("lsigf-f64-dmma-2-blocks", _lsigf_autograd_case(F64, 700, 1, 16, 128, 3, 2, bias="FN"),
         [r"contract_f64_kernel<8>", r"tap_grad_partial_kernel<double>", r"pack_taps_kernel<double>"]),
        # C ABI in both layouts, workspace canaries; forward_act ReLU on wgmma (Q = 48) and on FMA with T = 53 (fp64)
        ("abi-f32-node-major-relu-tc", _lsigf_abi_case(F32, 700, 2, 32, 48, 3, 2, 1, act=1),
         [r"tc_contract_kernel<64>"]),
        ("abi-f32-feature-major", _lsigf_abi_case(F32, 700, 2, 32, 48, 3, 2, 0, bias="FN"),
         [r"transpose_kernel<float>", r"tc_contract_kernel<64>"]),
        ("abi-f64-node-major-relu-T53", _lsigf_abi_case(F64, 300, 1, 3, 5, 14, 4, 1, act=1),
         [r"tap_contract_kernel<double>", r"tap_grad_partial_kernel<double>"]),
        ("abi-f64-feature-major", _lsigf_abi_case(F64, 300, 2, 5, 7, 3, 2, 0), [r"transpose_kernel<double>"]),
    ]


# --------------------------------------------------------------------------------------------------------- layout
def _layout_case(dtype, N, C, direction):
    """to_node_major: pad columns [C, ld) zero-filled, rows past N untouched; to_feature_major: nothing past N*C."""
    def run():
        cabi, lib = _lib()
        enum = cabi.F32 if dtype == F32 else cabi.F64
        g = torch.Generator(device="cuda").manual_seed(N + C)
        res = Result()
        ld = _padded(C, dtype) + (0 if dtype == F64 else 8)
        if direction == "to_node":
            src = torch.randn(C, N, generator=g, device="cuda", dtype=F64).to(dtype)
            dst = torch.full((N + 2, ld), SENT, dtype=dtype, device="cuda")
            _check(lib.b200gf_to_node_major(enum, src.data_ptr(), dst.data_ptr(), ld, N, C, _st()))
            assert torch.equal(dst[:N, :C], src.t()), "transpose must be exact"
            res.checks.append(("out", dst[:N, :C], None, None))
            assert torch.count_nonzero(dst[:N, C:]) == 0, "pad columns must be zero-filled"
            res.canaries.append(("rows>=N", dst[N:]))
            res.outputs.append(dst)
        else:
            src = torch.full((N, ld), float("nan"), dtype=dtype, device="cuda")
            src[:, :C] = torch.randn(N, C, generator=g, device="cuda", dtype=F64).to(dtype)
            dst = torch.full((C * N + 64,), SENT, dtype=dtype, device="cuda")
            _check(lib.b200gf_to_feature_major(enum, src.data_ptr(), ld, dst.data_ptr(), N, C, _st()))
            ref = src[:, :C].t()
            out = dst[:C * N].view(C, N)
            res.checks.append(("out", out, None, None))
            assert torch.equal(out, ref), "transpose must be exact"
            res.canaries.append(("past C*N", dst[C * N:]))
            res.outputs.append(out)
        return res
    return run


def _layout_rows():
    rows = []
    for dt, name in ((F32, "float"), (F64, "double")):
        for d in ("to_node", "to_feature"):
            rows.append(("layout-%s-%s-N1000-C37" % (d, name), _layout_case(dt, 1000, 37, d), [r"transpose_kernel<%s>" % name]))
    # N > 65535 * 32 nodes: the feature-major output needs more than 65535 grid rows -> slab loop (two launches)
    rows.append(("layout-to_feature-slab-N2200000-C3", _layout_case(F32, 2200000, 3, "to_feature"),
                 [r"transpose_kernel<float>", r"transpose_kernel<float>"]))
    return rows


# -------------------------------------------------------------------------------------------- relu / maxpool
def _relu_bwd_case(dtype, n, C, ld):
    def run():
        cabi, lib = _lib()
        enum = cabi.F32 if dtype == F32 else cabi.F64
        g = torch.Generator(device="cuda").manual_seed(n)
        y = torch.full((n, ld), float("nan"), dtype=dtype, device="cuda")
        y[:, :C] = torch.randn(n, C, generator=g, device="cuda", dtype=F64).to(dtype)
        y[0, :C] = 0.0                                          # y == 0 is not > 0
        y[1, :C] = -0.0
        dy = torch.full((n, ld + 1), float("nan"), dtype=dtype, device="cuda")
        dy[:, :C] = torch.randn(n, C, generator=g, device="cuda", dtype=F64).to(dtype)
        out = torch.full((n + 1, ld + 3), SENT, dtype=dtype, device="cuda")
        _check(lib.b200gf_relu_backward(enum, y.data_ptr(), ld, dy.data_ptr(), ld + 1, out.data_ptr(), ld + 3, n, C, _st()))
        ref = torch.where(y[:, :C] > 0, dy[:, :C], torch.zeros_like(dy[:, :C]))
        res = Result()
        assert torch.equal(out[:n, :C], ref)
        res.checks.append(("out", out[:n, :C], None, None))
        res.canaries += [("cols>=C", out[:, C:]), ("rows>=n", out[n:])]
        res.outputs.append(out[:n, :C])
        return res
    return run


def _maxpool_case(dtype, n_in, n_out, C, max_nb, backward):
    """MaxPoolLocal: ties (first maximum in the list wins), -inf entries, repeated padding members, padded ld."""
    def run():
        cabi, lib = _lib()
        enum = cabi.F32 if dtype == F32 else cabi.F64
        rng = np.random.default_rng(n_in + max_nb)
        ld = C + 3
        xh = np.round(rng.standard_normal((n_in, C)) * 2) / 2         # coarse values: many ties
        xh[rng.random((n_in, C)) < 0.05] = -np.inf
        xh[0, :] = -np.inf
        x = torch.full((n_in, ld), float("nan"), dtype=dtype, device="cuda")
        x[:, :C] = torch.tensor(xh, dtype=dtype)
        nbh = rng.integers(0, n_in, (n_out, max_nb)).astype(np.int32)
        nbh[:, -1] = nbh[:, 0]                                         # padding repeats a member
        nbh[0, :] = 0                                                  # an all -inf neighbourhood
        nb = torch.tensor(nbh, device="cuda")
        out = torch.full((n_out + 1, ld), SENT, dtype=dtype, device="cuda")
        arg = torch.full((n_out, C), -1, dtype=torch.int32, device="cuda")
        _check(lib.b200gf_maxpool_forward(enum, x.data_ptr(), ld, n_in, C, nb.data_ptr(), n_out, max_nb, out.data_ptr(), ld,
                                          arg.data_ptr(), _st()))
        vals = xh[nbh]                                                 # [n_out, max_nb, C]
        first = vals.argmax(axis=1)                                    # numpy argmax: the first maximum
        ref_arg = np.take_along_axis(nbh[:, :, None].repeat(C, 2), first[:, None, :], 1)[:, 0, :]
        ref = vals.max(axis=1)
        res = Result()
        assert torch.equal(out[:n_out, :C].cpu(), torch.tensor(ref, dtype=dtype))
        assert np.array_equal(arg.cpu().numpy(), ref_arg), "the first maximum of the list must win"
        res.canaries += [("out cols>=C", out[:, C:]), ("out rows>=n_out", out[n_out:])]
        if not backward:
            res.outputs += [out[:n_out, :C], arg]
            res.checks.append(("out", out[:n_out, :C], None, None))
            return res
        dy = torch.full((n_out, ld), float("nan"), dtype=dtype, device="cuda")
        dyh = rng.standard_normal((n_out, C))
        dy[:, :C] = torch.tensor(dyh, dtype=dtype)
        dx = torch.full((n_in, ld + 1), SENT, dtype=dtype, device="cuda")
        _check(lib.b200gf_maxpool_backward(enum, dy.data_ptr(), ld, arg.data_ptr(), n_out, C, dx.data_ptr(), ld + 1, n_in,
                                           _st()))
        dyr = dy[:, :C].double().cpu().numpy()
        ref_dx = np.zeros((n_in, C))
        abs_dx = np.zeros((n_in, C))
        cnt = np.zeros((n_in, C))
        cols = np.broadcast_to(np.arange(C), (n_out, C))
        np.add.at(ref_dx, (ref_arg, cols), dyr)
        np.add.at(abs_dx, (ref_arg, cols), np.abs(dyr))
        np.add.at(cnt, (ref_arg, cols), 1.0)
        res.checks.append(("dx", dx[:, :C], ref_dx, orc.dot_bound(np.maximum(cnt, 1), abs_dx, NPD[dtype])))
        res.nondeterministic = True   # atomicAdd: addition order varies between runs
        return res
    return run


def _layer_rows():
    rows = []
    for dt, name in ((F32, "float"), (F64, "double")):
        rows.append(("relu-bwd-%s" % name, _relu_bwd_case(dt, 1001, 37, 40), [r"relu_bwd_kernel<%s>" % name]))
        rows.append(("maxpool-fwd-%s" % name, _maxpool_case(dt, 500, 300, 21, 7, False), [r"maxpool_fwd_kernel<%s>" % name]))
        rows.append(("maxpool-fwd-nb1-%s" % name, _maxpool_case(dt, 500, 300, 21, 1, False), [r"maxpool_fwd_kernel<%s>" % name]))
        rows.append(("maxpool-bwd-%s" % name, _maxpool_case(dt, 200, 900, 21, 5, True), [r"maxpool_bwd_kernel<%s>" % name]))
    return rows


# ------------------------------------------------------------------------------------------------ edge-variant filter
def _ev_pattern(graph, N, diag):
    """The edge-variant structure (gnn_b200.edgevariant.EVStructure, so the transposed pattern and perm come from the
    product code) of _graph(graph, N)'s pattern.  diag adds the diagonal on every row i % 4 != 1: the other rows have
    diag[i] = -1 unless the graph has a self-loop there."""
    from gnn_b200 import edgevariant as evm
    m = _graph(graph, N)
    pat = sp.csr_matrix((np.ones(m.nnz), m.indices, m.indptr), shape=m.shape)
    if diag:
        d = np.nonzero(np.arange(N) % 4 != 1)[0]
        pat = sp.csr_matrix(pat + sp.csr_matrix((np.ones(len(d)), (d, d)), shape=(N, N)))
    pat.sum_duplicates()
    pat.sort_indices()
    rows = np.repeat(np.arange(N), np.diff(pat.indptr))
    st = evm.EVStructure.from_coo(N, [(torch.from_numpy(rows), torch.from_numpy(pat.indices.astype(np.int64)))], "cuda")
    return st.per_e[0], st.NA


def _ev_case(dtype, B, G, K, F=3, diag=True, N=3000, graph="rand", misaligned=False, pingpong=False):
    """b200gf_ev_forward + b200gf_ev_backward through the C ABI against oracle/ev_oracle.py.  Y, states, lam, dw and dxT
    start as NaN and are followed by 4 KB of SENT; the k = 0 weights are non-zero on every slot, so a diag step that read
    the whole row would show.  misaligned: Y and dY one element past a 16-byte boundary, which selects the VB = 1
    kernels; their per-element operation order is the vector kernels', so Y, dw and dxT must equal the aligned run bit
    for bit.  pingpong: a forward with n_states = 2 (inference) must give the Y of n_states = K - 1."""
    memo = {}

    def run():
        cabi, lib = _lib()
        enum = cabi.F32 if dtype == F32 else cabi.F64
        if not memo:
            pe, NA = _ev_pattern(graph, N, diag)
            rng = np.random.default_rng(NA + 7 * B + 31 * G + K)
            r = lambda shape: orc.biased_uniform(rng, shape).astype(NPD[dtype]).astype(np.float64)   # noqa: E731
            w, xT, dY = r((F, K, G, pe["nnz"])), r((G, NA, B)), r((F, NA, B))
            host = [pe[k].cpu().numpy() for k in ("rowptr", "col")] + [pe["diag"].cpu().numpy() if diag else None]
            Yr, _ = evo.ev_forward(*host, w, xT)
            dwr, dxr, _ = evo.ev_backward(*host, w, xT, dY)
            memo.update(pe=pe, NA=NA, w=w, xT=xT, dY=dY, ref=(Yr, dwr, dxr),
                        env=evo.ev_envelope(*host, w, xT, dY, dtype=NPD[dtype]))
        pe, NA = memo["pe"], memo["NA"]
        nnz = pe["nnz"]
        dev = lambda a: torch.tensor(a, dtype=dtype, device="cuda")          # noqa: E731
        w, xT = dev(memo["w"]), dev(memo["xT"])
        pad = 4096 // w.element_size()
        chain, ny, nw, nx = F * G * NA * B, F * NA * B, F * K * G * nnz, G * NA * B
        diag_p = pe["diag"].data_ptr() if diag else None

        def buf(n, off=0):
            t = torch.full((off + n + pad,), SENT, dtype=dtype, device="cuda")
            t[off:off + n] = float("nan")
            return t

        def fwd_bwd(n_states, off, backward=True):
            Yb, Sb = buf(ny, off), buf(n_states * chain)
            _check(lib.b200gf_ev_forward(enum, NA, B, G, F, K, pe["rowptr"].data_ptr(), pe["col"].data_ptr(), diag_p, nnz,
                                         w.data_ptr(), xT.data_ptr(), Sb.data_ptr(), n_states, Yb[off:].data_ptr(), _st()))
            bufs = dict(Y=(Yb, off, ny), states=(Sb, 0, n_states * chain))
            if backward:
                dYb = torch.full((off + ny,), float("nan"), dtype=dtype, device="cuda")
                dYb[off:] = dev(memo["dY"]).flatten()
                lam, dw, dx = buf(2 * chain), buf(nw), buf(nx)
                _check(lib.b200gf_ev_backward(enum, NA, B, G, F, K, pe["rowptr"].data_ptr(), pe["col"].data_ptr(),
                                              pe["rowptrT"].data_ptr(), pe["colT"].data_ptr(), pe["perm"].data_ptr(), diag_p,
                                              nnz, w.data_ptr(), xT.data_ptr(), Sb.data_ptr(), dYb[off:].data_ptr(),
                                              lam.data_ptr(), dw.data_ptr(), dx.data_ptr(), _st()))
                bufs.update(lam=(lam, 0, 2 * chain), dw=(dw, 0, nw), dxT=(dx, 0, nx))
            return bufs

        res = Result()

        def fence(bufs, tag=""):
            for name, (t, off, n) in bufs.items():
                res.canaries += [(tag + name + " before", t[:off]), (tag + name + " tail", t[off + n:])]
            return bufs

        bufs = fence(fwd_bwd(max(K - 1, 1), 1 if misaligned else 0))
        Y =bufs["Y"][0][bufs["Y"][1]:][:ny].view(F, NA, B)
        dw = bufs["dw"][0][:nw].view(F, K, G, nnz)
        dx = bufs["dxT"][0][:nx].view(G, NA, B)
        env = memo["env"]
        res.checks += [(n, t, ref, env[n]) for n, t, ref in zip(("Y", "dw", "dxT"), (Y, dw, dx), memo["ref"])]
        res.finite += [("Y", Y), ("dw (every slot written)", dw), ("dxT", dx)]
        res.outputs += [Y, dw, dx]
        if diag:                                 # the k = 0 off-diagonal slots are written, with exactly 0
            off_diag = torch.ones(nnz, dtype=torch.bool, device="cuda")
            d = pe["diag"]
            off_diag[d[d >= 0].long()] = False
            assert bool((dw[:, 0][..., off_diag] == 0).all()), "k = 0 off-diagonal dw slots must be exactly 0"
        if misaligned:
            al = fence(fwd_bwd(max(K - 1, 1), 0), "aligned ")
            for n, t in (("Y", Y), ("dw", dw), ("dxT", dx)):
                assert torch.equal(_bits(t.flatten()), _bits(al[n][0][:t.numel()])), "%s: VB = 1 and VB = 4 differ" % n
        if pingpong:
            pp = fence(fwd_bwd(2, 0, backward=False), "ping-pong ")
            assert torch.equal(_bits(Y.flatten()), _bits(pp["Y"][0][:ny])), "n_states = 2 and n_states = K-1 differ"
        return res
    return run


def _ev_rows():
    fwd_bwd = lambda t, vb: [r"step_kernel<%s,%d,8>" % (t, vb), r"adjoint_step_kernel<%s,%d>" % (t, vb),   # noqa: E731
                             r"adjoint_init_kernel<%s>" % t, r"wgrad_kernel<%s>" % t, r"xgrad_kernel<%s>" % t]
    rows = [
        # 16-byte batch vectors, the G-tail of the GB = 8 loop (G = 9), diag with k = 0 off-diagonal weights
        ("ev-f32-B8-G9-K3-diag", _ev_case(F32, 8, 9, 3), fwd_bwd("float", 4)),
        ("ev-f32-B7-G17-K3", _ev_case(F32, 7, 17, 3, diag=False), fwd_bwd("float", 1)),
        # Y / dY misaligned: the VB = 1 kernels, bit-identical to the aligned (VB = 4) run made in the same case
        ("ev-f32-B8-G8-K2-misaligned", _ev_case(F32, 8, 8, 2, diag=False, misaligned=True),
         fwd_bwd("float", 1) + [r"step_kernel<float,4,8>", r"adjoint_step_kernel<float,4>"]),
        # B > 32: wgrad's lane loop
        ("ev-f64-B33-G1-K4-diag", _ev_case(F64, 33, 1, 4), fwd_bwd("double", 1)),
        # K = 1: no adjoint step, xgrad on the diag branch
        ("ev-f64-B64-G20-K1-diag", _ev_case(F64, 64, 20, 1),
         [r"step_kernel<double,1,8>", r"adjoint_init_kernel<double>", r"wgrad_kernel<double>", r"xgrad_kernel<double>"]),
        ("ev-f32-B16-G4-K5-diag-pingpong", _ev_case(F32, 16, 4, 5, pingpong=True), fwd_bwd("float", 4)),
        # the 20 000-entry hub row and column, F NA B / VB > 132 * 16 * 256: every grid-stride loop takes several passes
        ("ev-hub-f32", _ev_case(F32, 16, 2, 3, F=8, diag=False, N=24000), fwd_bwd("float", 4)),
        ("ev-hub-f64", _ev_case(F64, 16, 2, 3, F=8, diag=False, N=24000), fwd_bwd("double", 1)),
    ]
    for N in (1, 3, 7):
        rows.append(("ev-tinyN%d-f64" % N, _ev_case(F64, 1, 1, 2, N=N, graph="tiny"), fwd_bwd("double", 1)))
    return rows


CASES = (_hop_rows() + _contract_rows() + _tap_grad_rows() + _bias_grad_rows() + _lsigf_rows() + _layout_rows()
         + _layer_rows() + _ev_rows())

# __global__ functions of this table's sources without a case here, and where they are tested
EXCLUDED = {
    "peer_signal_kernel": "peer fence: tests/test_peer_epilogues.py (one participant), tests/test_distributed.py",
    "peer_wait_kernel": "peer fence: tests/test_peer_epilogues.py (one participant), tests/test_distributed.py",
    "bcast_rows_kernel": "all-gather of the node-sharded path's k = 0 rows: tests/test_peer_epilogues.py",
    "scatter_rows_kernel": "scatter of the feature-sharded path's k = 0 slices: tests/test_peer_epilogues.py",
    "narrow_rowptr_kernel": "device plan build (b200gf_plan_create_device): tests/test_widen_*",
}


@pytest.mark.gpu
@pytest.mark.parametrize("cid,fn,kernels", CASES, ids=[c[0] for c in CASES])
def test_dispatch(cid, fn, kernels):
    res1, names = _launched(fn)
    check_case(cid, fn, kernels, names, res1)
