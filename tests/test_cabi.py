"""C-ABI boundary tests.  CPU part: the library loads and exports exactly what include/b200gf.h declares.
GPU part (-m gpu): raw ctypes calls with the reference's feature-major [B,G,N] buffers and the building blocks."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import lsigf_oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_functions():
    txt = open(os.path.join(ROOT, "include", "b200gf.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(b200gf_[a-z_0-9]+)\s*\(", txt)))


def test_library_exports_every_declared_symbol():
    import gnn_b200
    lib = gnn_b200._cabi.load()
    declared = _header_functions()
    assert len(declared) >= 15
    for name in declared:
        assert hasattr(lib, name), "libb200gf.so does not export %s" % name
    assert sorted(gnn_b200._cabi.EXPORTED_SYMBOLS) == declared, "ctypes binding and header disagree"
    assert lib.b200gf_version() >= 100
    assert b"invalid argument" in lib.b200gf_strerror(-1)
    assert b"workspace" in lib.b200gf_strerror(-4)


def test_invalid_arguments_return_codes_without_gpu():
    import gnn_b200
    lib = gnn_b200._cabi.load()
    out = ctypes.c_void_p()
    # null arrays -> EINVAL before any CUDA call
    assert lib.b200gf_plan_create(ctypes.byref(out), 0, 4, 1, None, None, None, 0) == -1
    assert lib.b200gf_plan_create(ctypes.byref(out), 0, 4, 1, gnn_b200._cabi.ptr_array([0]),
                                  gnn_b200._cabi.ptr_array([0]), gnn_b200._cabi.ptr_array([0]), 7) == -2
    assert lib.b200gf_plan_info(None, 0) == -1
    assert lib.b200gf_workspace_bytes(None, 1, 1, 1, 1, 0, 0) == 0
    lib.b200gf_plan_destroy(None)  # no-op
    if not torch.cuda.is_available():
        rp = np.array([0, 1, 2], dtype=np.int64); ci = np.array([1, 0], dtype=np.int32); va = np.ones(2, np.float32)
        rc = lib.b200gf_plan_create(ctypes.byref(out), 0, 2, 1, gnn_b200._cabi.ptr_array([rp.ctypes.data]),
                                    gnn_b200._cabi.ptr_array([ci.ctypes.data]), gnn_b200._cabi.ptr_array([va.ctypes.data]), 0)
        assert rc == -5  # B200GF_ENODEVICE: loud, no fallback
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            gnn_b200.LSIGF(torch.zeros(1, 1, 1, 1), torch.zeros(1, 2, 2), torch.zeros(1, 1, 2))


# ------------------------------------------------------------------------------------------------ GPU
def _rel(a, b):
    return np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-300)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_forward_backward_feature_major_raw(dtype):
    """Calls b200gf_forward / b200gf_backward exactly as a C caller holding the reference's [B,G,N] buffers would."""
    import gnn_b200
    cabi = gnn_b200._cabi
    lib = cabi.load()
    c = orc.random_case(77, N=300, B=3, G=5, F=6, K=4, E=2, avg_deg=7, bias="F1")
    enum = cabi.F32 if dtype == torch.float32 else cabi.F64
    tol = 1e-4 if dtype == torch.float32 else 1e-11
    gso = gnn_b200.SparseGSO.from_dense(torch.tensor(c["S"], dtype=dtype))
    plan = gso.plan("cuda")
    assert plan.info(0) == 300 and plan.info(2) == 2 and plan.info(5) == gso.nnz() and plan.info(6) == 0
    dev = lambda a: torch.tensor(a, dtype=dtype, device="cuda").contiguous()
    h, x, b, dy = dev(c["h"]), dev(c["x"]), dev(c["b"]), dev(c["dy"])
    B, G, N = x.shape
    F, E, K, _ = h.shape
    y = torch.empty(B, F, N, dtype=dtype, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    wsb = lib.b200gf_workspace_bytes(plan.handle, B, G, F, K, cabi.FEATURE_MAJOR, 0)
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    rc = lib.b200gf_forward(plan.handle, x.data_ptr(), cabi.FEATURE_MAJOR, 0, h.data_ptr(), b.data_ptr(), 0,
                            y.data_ptr(), cabi.FEATURE_MAJOR, 0, ws.data_ptr(), wsb, B, G, F, K, st)
    assert rc == 0, lib.b200gf_strerror(rc)
    rnd = lambda a: torch.tensor(a, dtype=dtype).double().numpy()
    y_ref = orc.lsigf_dense(rnd(c["h"]), rnd(c["S"]), rnd(c["x"]), rnd(c["b"]))
    assert _rel(y.cpu().numpy(), y_ref) < tol
    # too-small workspace is reported, not overrun
    assert lib.b200gf_forward(plan.handle, x.data_ptr(), 0, 0, h.data_ptr(), b.data_ptr(), 0, y.data_ptr(), 0, 0,
                              ws.data_ptr(), 256, B, G, F, K, st) == -4
    dx = torch.empty_like(x); dh = torch.empty_like(h); db = torch.empty_like(b)
    wsb = lib.b200gf_workspace_bytes(plan.handle, B, G, F, K, cabi.FEATURE_MAJOR, 1)
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    rc = lib.b200gf_backward(plan.handle, dy.data_ptr(), 0, 0, x.data_ptr(), 0, 0, h.data_ptr(), dx.data_ptr(), 0, 0,
                             dh.data_ptr(), db.data_ptr(), 0, ws.data_ptr(), wsb, B, G, F, K, st)
    assert rc == 0, lib.b200gf_strerror(rc)
    dh_ref, dx_ref, db_ref = orc.lsigf_grads_dense(rnd(c["h"]), rnd(c["S"]), rnd(c["x"]), rnd(c["dy"]), (F, 1))
    assert _rel(dh.cpu().numpy(), dh_ref) < tol
    assert _rel(dx.cpu().numpy(), dx_ref) < tol
    assert _rel(db.cpu().numpy(), db_ref) < tol


@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 3, 4, 17, 32, 64, 100, 128, 130, 320, 2048])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_hop_building_block(C, dtype):
    """One shift for every lane-mapping variant of spmm.cu (C selects L / chunks / scalar fallback), both directions,
    empty rows and rows longer than 32 and 64 entries included."""
    import scipy.sparse as sp
    import gnn_b200
    cabi = gnn_b200._cabi
    lib = cabi.load()
    N = 777
    rs = np.random.RandomState(C)
    m = sp.random(N, N, density=0.02, format="lil", random_state=rs)
    m[5, :] = 0                                  # empty row
    m[:, 9] = 0                                  # empty column
    m[11, rs.choice(N, 100, replace=False)] = rs.randn(100)   # long row
    m[rs.choice(N, 70, replace=False), 13] = rs.randn(70)[:, None]  # long column (long row of the transpose)
    m = sp.csr_matrix(m)
    gso = gnn_b200.SparseGSO.from_scipy([m], dtype=dtype)
    plan = gso.plan("cuda")
    npd = np.float32 if dtype == torch.float32 else np.float64
    mr = sp.csr_matrix((m.data.astype(npd).astype(np.float64), m.indices, m.indptr), shape=m.shape)
    X = torch.randn(N, C, dtype=dtype, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    tol = 1e-5 if dtype == torch.float32 else 1e-13
    for direction, op in ((cabi.HOP_FWD, mr.T), (cabi.HOP_BWD, mr)):
        for ld_pad in (0, 8):                   # ld == C (possibly unaligned -> scalar path) and padded ld
            ld = gnn_b200.padded_ld(C, dtype) + ld_pad if ld_pad else C
            src = torch.zeros(N, ld, dtype=dtype, device="cuda"); src[:, :C] = X
            dst = torch.full((N, ld), float("nan"), dtype=dtype, device="cuda")
            rc = lib.b200gf_hop(plan.handle, 0, direction, src.data_ptr(), ld, dst.data_ptr(), ld, C, st)
            assert rc == 0, lib.b200gf_strerror(rc)
            ref = op @ X.double().cpu().numpy()
            assert _rel(dst[:, :C].cpu().numpy(), ref) < tol, (C, direction, ld)


@pytest.mark.gpu
def test_layout_and_tap_blocks():
    import gnn_b200
    cabi = gnn_b200._cabi
    lib = cabi.load()
    st = torch.cuda.current_stream().cuda_stream
    for dtype, enum in ((torch.float32, cabi.F32), (torch.float64, cabi.F64)):
        N, B, G, F, T = 1000, 3, 5, 7, 4
        C = B * G
        x = torch.randn(B, G, N, dtype=dtype, device="cuda")
        ld = gnn_b200.padded_ld(C, dtype)
        xn = torch.full((N, ld), float("nan"), dtype=dtype, device="cuda")
        assert lib.b200gf_to_node_major(enum, x.data_ptr(), xn.data_ptr(), ld, N, C, st) == 0
        assert torch.equal(xn[:, :C], x.reshape(C, N).t())
        assert torch.all(xn[:, C:] == 0)
        back = torch.empty_like(x)
        assert lib.b200gf_to_feature_major(enum, xn.data_ptr(), ld, back.data_ptr(), N, C, st) == 0
        assert torch.equal(back, x)
        # tap contraction and tap gradient against einsum
        zs = [torch.randn(N, ld, dtype=dtype, device="cuda") for _ in range(T)]
        W = torch.randn(T, G, F, dtype=dtype, device="cuda")
        bias = torch.randn(F, dtype=dtype, device="cuda")
        ldo = gnn_b200.padded_ld(B * F, dtype)
        out = torch.zeros(N, ldo, dtype=dtype, device="cuda")
        rc = lib.b200gf_tap_contract(enum, N, B, G, F, T, cabi.ptr_array([z.data_ptr() for z in zs]),
                                     cabi.i64_array([ld] * T), W.data_ptr(), bias.data_ptr(), 0, out.data_ptr(), ldo, 0, None, 0, st)
        assert rc == 0
        Z = torch.stack([z[:, :C].reshape(N, B, G) for z in zs]).double()
        ref = torch.einsum("tnbg,tgf->nbf", Z, W.double()) + bias.double()
        tol = 1e-5 if dtype == torch.float32 else 1e-12
        assert _rel(out[:, :B * F].reshape(N, B, F).cpu().numpy(), ref.cpu().numpy()) < tol
        vs = [torch.randn(N, ldo, dtype=dtype, device="cuda") for _ in range(T)]
        dW = torch.empty(T, G, F, dtype=dtype, device="cuda")
        sb = lib.b200gf_tap_grad_scratch_bytes(enum, N, B, G, F, T)
        scratch = torch.empty(sb, dtype=torch.uint8, device="cuda")
        rc = lib.b200gf_tap_grad(enum, N, B, G, F, T, zs[0].data_ptr(), ld, cabi.ptr_array([v.data_ptr() for v in vs]),
                                 cabi.i64_array([ldo] * T), dW.data_ptr(), scratch.data_ptr(), sb, st)
        assert rc == 0
        V = torch.stack([v[:, :B * F].reshape(N, B, F) for v in vs]).double()
        refg = torch.einsum("nbg,tnbf->tgf", Z[0], V)
        assert _rel(dW.cpu().numpy(), refg.cpu().numpy()) < tol
        # pack_taps
        E, K = 2, 3
        h = torch.randn(F, E, K, G, dtype=dtype, device="cuda")
        Wp = torch.empty(1 + E * (K - 1), G, F, dtype=dtype, device="cuda")
        assert lib.b200gf_pack_taps(enum, h.data_ptr(), Wp.data_ptr(), F, E, K, G, 0, st) == 0
        assert torch.allclose(Wp[0], h[:, :, 0, :].sum(1).t())
        assert torch.equal(Wp[1 + 1 * (K - 1) + 1], h[:, 1, 2, :].t())


@pytest.mark.gpu
@pytest.mark.parametrize("N,B,P,Q,T,bias_mode", [
    (1000, 1, 64, 64, 5, "q"),        # headline layer shape, ragged last tile
    (128, 1, 32, 16, 1, None),        # one tile, one chunk
    (777, 3, 32, 32, 9, "q"),         # B > 1 (cfg4 shape: E=4, K=3 -> T=9)
    (2500, 2, 64, 128, 3, "node"),    # wide output, per-node bias
    (4096, 1, 96, 256, 2, "q"),       # P = 3 chunks, Q = 256 (2 pipeline stages)
    (50000, 1, 64, 64, 5, "q"),       # several tiles per CTA: accumulator double-buffering and ring wrap-around
])
def test_tensor_core_tap_contract(N, B, P, Q, T, bias_mode):
    """wgmma 3xTF32 contraction (tc_contract.cu) vs an fp64 einsum; must sit at FP32 accuracy, far inside 1e-4."""
    import gnn_b200
    cabi = gnn_b200._cabi
    lib = cabi.load()
    st = torch.cuda.current_stream().cuda_stream
    g = torch.Generator(device="cuda").manual_seed(N + P + Q)
    ld = B * P
    zs = [torch.randn(N, ld, device="cuda", generator=g) * (1.0 + t) for t in range(T)]
    W = (torch.rand(T, P, Q, device="cuda", generator=g) * 2 - 1) / np.sqrt(P * T)
    bias = None
    if bias_mode == "q":
        bias = torch.randn(Q, device="cuda", generator=g)
    elif bias_mode == "node":
        bias = torch.randn(Q, N, device="cuda", generator=g)
    ldo = B * Q
    out = torch.full((N, ldo), float("nan"), device="cuda")
    sb = lib.b200gf_tap_contract_scratch_bytes(T, P, Q)
    scratch = torch.empty(sb, dtype=torch.uint8, device="cuda")
    rc = lib.b200gf_tap_contract(cabi.F32, N, B, P, Q, T, cabi.ptr_array([z.data_ptr() for z in zs]),
                                 cabi.i64_array([ld] * T), W.data_ptr(), None if bias is None else bias.data_ptr(),
                                 1 if bias_mode == "node" else 0, out.data_ptr(), ldo, 0, scratch.data_ptr(), sb, st)
    assert rc == 0, lib.b200gf_strerror(rc)
    torch.cuda.synchronize()
    Z = torch.stack([z.view(N, B, P) for z in zs]).double()
    ref = torch.einsum("tnbp,tpq->nbq", Z, W.double())
    if bias_mode == "q":
        ref = ref + bias.double()
    elif bias_mode == "node":
        ref = ref + bias.double().t()[:, None, :]
    err = _rel(out.view(N, B, Q).cpu().numpy(), ref.cpu().numpy())
    # same problem through the FMA kernel (no scratch): the two paths must agree to FP32 rounding
    out2 = torch.empty_like(out)
    rc = lib.b200gf_tap_contract(cabi.F32, N, B, P, Q, T, cabi.ptr_array([z.data_ptr() for z in zs]),
                                 cabi.i64_array([ld] * T), W.data_ptr(), None if bias is None else bias.data_ptr(),
                                 1 if bias_mode == "node" else 0, out2.data_ptr(), ldo, 0, None, 0, st)
    assert rc == 0
    err_fma = _rel(out2.view(N, B, Q).cpu().numpy(), ref.cpu().numpy())
    print("tc err %.2e  fma err %.2e" % (err, err_fma))
    assert err < 5e-6, err
    assert err_fma < 5e-6, err_fma


def test_header_is_plain_c(tmp_path):
    """include/b200gf.h must be consumable from C (the boundary is a C ABI, not a C++ one): compile a C99 translation
    unit that includes it and takes the address of every declared function, then link it against the library."""
    import shutil
    import subprocess
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    import gnn_b200
    names = _header_functions()
    src = tmp_path / "abi.c"
    body = "\n".join("    p[%d] = (fn_t)&%s;" % (i, n) for i, n in enumerate(names))
    src.write_text('#include "b200gf.h"\n#include <stdio.h>\ntypedef void (*fn_t)(void);\nint main(void) {\n'
                   '    fn_t p[%d];\n%s\n    printf("%%d %%d\\n", b200gf_version(), (int)(p[0] != 0));\n    return 0;\n}\n'
                   % (len(names), body))
    exe = tmp_path / "abi"
    libdir = os.path.dirname(gnn_b200._cabi.LIB_PATH)
    cmd = [gcc, "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe),
           "-L", libdir, "-lb200gf", "-Wl,-rpath," + libdir]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    run = subprocess.run([str(exe)], capture_output=True, text=True)
    assert run.returncode == 0 and run.stdout.split()[0] == str(gnn_b200._cabi.load().b200gf_version())


@pytest.mark.gpu
def test_launch_counter_counts_library_kernels():
    import gnn_b200
    from gnn_b200 import graphs
    lib = gnn_b200._cabi.load()
    gso = graphs.er_gso(5000, 8, seed=1)
    h = torch.randn(64, 1, 4, 64, device="cuda") * 0.1
    x = torch.randn(1, 64, 5000, device="cuda")
    gnn_b200.LSIGF(h, gso, x, None)                               # plan + warm-up
    lib.b200gf_launch_count(1)
    gnn_b200.LSIGF(h, gso, x, None)
    # transpose to node-major, 3 hops, tap packing, contraction
    assert lib.b200gf_launch_count(0) == 6 and lib.b200gf_launch_count(1) == 6 and lib.b200gf_launch_count(0) == 0
