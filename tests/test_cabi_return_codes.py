"""Return codes of the C entry points for bad arguments, and the order their checks run in (CPU only).

Each entry point is called with placeholder device pointers: first with arguments that pass every check, then with one
or two faults at a time.  A call that passes every check would launch a kernel; without a CUDA device that launch
fails, so it comes back as a CUDA error code (rc <= B200GF_ECUDA).  For the same reason the whole module skips itself
when a CUDA device is visible: placeholder pointers must never reach a kernel.

The plan-based entry points need a plan, and b200gf_plan_create needs a device.  A small helper compiled against
csrc/common.cuh builds host-only plans (no CSR on the device) that get exactly as far as the argument checks need; a
plan with v2=1 also carries a placeholder for the 32-bit row offsets, which the fused all-gather and grid epilogues
require before they launch."""
import ctypes
import os
import shutil
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "graph-neural-networks_b200", "csrc")

pytestmark = pytest.mark.skipif(torch.cuda.is_available(),
                                reason="placeholder pointers must not reach a kernel on a real device")

OK, EINVAL, EUNSUPPORTED, EWORKSPACE, ECUDA = 0, -1, -2, -4, -1000
PASS = "passes every check"     # expected rc <= B200GF_ECUDA: the first launch or CUDA call fails without a device
F32, F64, FM, NM = 0, 1, 0, 1
P = 0x10000                     # placeholder device pointer (256-byte aligned)
WS = 0x20000                    # placeholder workspace
MISALIGNED = 0x101
RP32 = 0x30000                  # placeholder 32-bit row offsets of a host-only plan
BIG = 1 << 31                   # > INT32_MAX

_HELPER = r"""
#include "common.cuh"
extern "C" b200gf_plan* rc_test_plan(int64_t n_rows, int64_t n_cols, int E, int dtype, int has_bwd, void* rowptr32) {
  b200gf_plan* p = new b200gf_plan();
  p->dtype = dtype; p->n_rows = n_rows; p->n_cols = n_cols; p->E = E; p->has_bwd = has_bwd != 0;
  p->fwd.resize(E); p->bwd.resize(E);
  for (int e = 0; e < E; ++e) p->fwd[e].rowptr32 = p->bwd[e].rowptr32 = (int32_t*)rowptr32;
  return p;
}
extern "C" void rc_test_plan_free(b200gf_plan* p) { delete p; }
"""


@pytest.fixture(scope="module")
def lib():
    import gnn_b200
    return gnn_b200._cabi.load()


@pytest.fixture(scope="module")
def plans(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    d = tmp_path_factory.mktemp("rc_plan")
    src, so = d / "rc_plan.cu", d / "rc_plan.so"
    src.write_text(_HELPER)
    out = subprocess.run([nvcc, "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-I", CSRC, str(src), "-o", str(so)],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    h = ctypes.CDLL(str(so))
    h.rc_test_plan.restype = ctypes.c_void_p
    h.rc_test_plan.argtypes = [ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    h.rc_test_plan_free.argtypes = [ctypes.c_void_p]
    made = {}

    def plan(N=64, E=2, dtype=F32, has_bwd=1, n_cols=None, v2=0):
        key = (N, E, dtype, has_bwd, n_cols, v2)
        if key not in made:
            made[key] = h.rc_test_plan(N, N if n_cols is None else n_cols, E, dtype, has_bwd, RP32 if v2 else None)
        return made[key]

    yield plan
    for p in made.values():
        h.rc_test_plan_free(p)


def _check(fn, defaults, cases):
    """fn(*defaults) with each case's overrides; returns the cases whose return code differs from the expected one."""
    bad = []
    for over, want in cases:
        args = dict(defaults, **over)
        rc = fn(*args.values())
        if (rc > ECUDA) if want == PASS else (rc != want):
            bad.append((over, want, rc))
    return bad


def _ptrs(n, null_at=None, shift_at=None, by=0):
    """n placeholder device pointers, 256-byte aligned; the one at null_at null, the one at shift_at moved by `by` bytes."""
    import gnn_b200
    return gnn_b200._cabi.ptr_array([0 if i == null_at else P + 0x1000 * i + (by if i == shift_at else 0) for i in range(n)])


def _lds(n, ld):
    import gnn_b200
    return gnn_b200._cabi.i64_array([ld] * n)


# ------------------------------------------------------------------------------------------------ plan-based
B, G, F, K = 2, 3, 5, 3
C, CF = B * G, B * F


def _lsigf_forward(lib, plans):
    plan = plans()
    need = lib.b200gf_workspace_bytes(plan, B, G, F, K, NM, 0) - 256
    need_fm = lib.b200gf_workspace_bytes(plan, B, G, F, K, FM, 0) - 256
    d = dict(plan=plan, x=P, x_layout=NM, x_ld=C, h=P, bias=None, bpn=0, y=P, y_layout=NM, y_ld=CF, ws=WS, wsb=need,
             B=B, G=G, F=F, K=K, stream=None)
    cases = [
        ({}, PASS), (dict(K=1), PASS), (dict(x_layout=FM, y_layout=FM, wsb=need_fm), PASS),
        (dict(plan=None), EINVAL), (dict(x=None), EINVAL), (dict(y=None), EINVAL), (dict(B=0), EINVAL),
        (dict(K=-1), EINVAL), (dict(x_layout=7), EINVAL), (dict(y_layout=7), EINVAL), (dict(x_ld=C - 1), EINVAL),
        (dict(y_ld=CF - 1), EINVAL), (dict(plan=plans(n_cols=65)), EINVAL),
        (dict(ws=MISALIGNED), EINVAL), (dict(ws=None), EWORKSPACE), (dict(wsb=need - 1), EWORKSPACE),
        (dict(x_layout=FM, y_layout=FM, wsb=need_fm - 1), EWORKSPACE),
        # order
        (dict(ws=MISALIGNED, wsb=need - 1), EINVAL), (dict(ws=None, wsb=0), EWORKSPACE),
        (dict(x_ld=C - 1, ws=None), EINVAL), (dict(plan=None, x_layout=7), EINVAL),
        (dict(plan=plans(N=0), ws=None), OK), (dict(plan=plans(N=0), ws=MISALIGNED), OK),
        (dict(plan=plans(N=0), x_ld=C - 1), EINVAL),
    ]
    return lib.b200gf_forward, d, cases


def _lsigf_forward_act(lib, plans):
    fn, d, cases = _lsigf_forward(lib, plans)
    d = dict(list(d.items())[:-1] + [("act", 1), ("stream", None)])
    cases = cases + [(dict(act=7), EINVAL), (dict(act=7, plan=None), EINVAL), (dict(act=7, ws=None), EINVAL)]
    return lib.b200gf_forward_act, d, cases


def _lsigf_backward(lib, plans):
    plan = plans()
    need = lib.b200gf_workspace_bytes(plan, B, G, F, K, NM, 1) - 256
    need_fm = lib.b200gf_workspace_bytes(plan, B, G, F, K, FM, 1) - 256
    d = dict(plan=plan, dy=P, dy_layout=NM, dy_ld=CF, x=P, x_layout=NM, x_ld=C, h=P, dx=P, dx_layout=NM, dx_ld=C, dh=P,
             dbias=P, bpn=0, ws=WS, wsb=need, B=B, G=G, F=F, K=K, stream=None)
    cases = [
        ({}, PASS), (dict(K=1), PASS), (dict(dx=None, dx_ld=0, dx_layout=7), PASS),
        (dict(dy_layout=FM, wsb=need_fm), PASS), (dict(plan=plans(N=0)), PASS),
        (dict(plan=None), EINVAL), (dict(dy=None), EINVAL), (dict(x=None), EINVAL), (dict(h=None), EINVAL),
        (dict(dh=None), EINVAL), (dict(G=0), EINVAL), (dict(dy_layout=7), EINVAL), (dict(dx_layout=7), EINVAL),
        (dict(dy_ld=CF - 1), EINVAL), (dict(x_ld=C - 1), EINVAL), (dict(dx_ld=C - 1), EINVAL),
        (dict(plan=plans(has_bwd=0)), EINVAL), (dict(plan=plans(n_cols=65)), EINVAL),
        (dict(ws=MISALIGNED), EINVAL), (dict(ws=None), EWORKSPACE), (dict(wsb=need - 1), EWORKSPACE),
        (dict(dy_layout=FM, wsb=need_fm - 1), EWORKSPACE),
        # order
        (dict(ws=MISALIGNED, wsb=need - 1), EINVAL), (dict(dy_ld=CF - 1, ws=None), EINVAL),
        (dict(plan=plans(N=0), ws=None), EWORKSPACE), (dict(plan=plans(N=0), ws=MISALIGNED), EINVAL),
        (dict(plan=plans(N=0), wsb=0), EWORKSPACE),
    ]
    return lib.b200gf_backward, d, cases


def _hop(lib, plans):
    d = dict(plan=plans(), e=1, direction=1, src=P, src_ld=C, dst=P, dst_ld=C, C=C, stream=None)
    cases = [
        ({}, PASS), (dict(direction=0), PASS),
        (dict(plan=None), EINVAL), (dict(src=None), EINVAL), (dict(e=2), EINVAL), (dict(e=-1), EINVAL),
        (dict(direction=2), EINVAL), (dict(plan=plans(has_bwd=0)), EINVAL), (dict(C=0), EINVAL),
        (dict(src_ld=C - 1), EINVAL), (dict(dst_ld=C - 1), EINVAL),
        (dict(plan=plans(has_bwd=0), direction=0), PASS),
    ]
    return lib.b200gf_hop, d, cases


# ------------------------------------------------------------------------------------------------ peer epilogues
# The fused multi-GPU hops and row copies: ScatterArgs (peer r // rows_per_peer, column b*stride_b + out_col + g of
# b*gl + g) and BcastArgs (full-height peer buffers, rows from row0).  Scatter peers must be 16-byte aligned (EINVAL);
# the all-gather and grid epilogues need 32-byte lanes, so their misaligned buffers are EUNSUPPORTED, as is a 16-byte
# row copy whose source or peer is not 16-byte aligned.
def _hop_scatter(lib, plans):
    d = dict(plan=plans(), e=1, direction=1, src=P, src_ld=16, dst=P, dst_ld=16, C=16, peers=_ptrs(2), n_peers=2,
             rows_per_peer=32, out_ld=96, out_col=8, gl=8, stride_b=48, stream=None)
    cases = [
        ({}, PASS), (dict(direction=0), PASS), (dict(plan=plans(v2=1)), PASS), (dict(C=48, src_ld=48, dst_ld=48), PASS),
        (dict(peers=_ptrs(16), n_peers=16, rows_per_peer=4), PASS), (dict(gl=4, out_col=4), PASS),
        (dict(plan=None), EINVAL), (dict(src=None), EINVAL), (dict(dst=None), EINVAL), (dict(e=2), EINVAL),
        (dict(direction=2), EINVAL), (dict(plan=plans(has_bwd=0)), EINVAL),
        (dict(peers=None), EINVAL), (dict(n_peers=0), EINVAL), (dict(peers=_ptrs(17), n_peers=17), EINVAL),
        (dict(peers=_ptrs(2, null_at=1)), EINVAL), (dict(rows_per_peer=0), EINVAL), (dict(gl=0), EINVAL),
        (dict(rows_per_peer=31), EINVAL),                               # 2 x 31 < 64 rows
        (dict(C=12, src_ld=12, dst_ld=12), EINVAL),                     # C % gl
        (dict(peers=_ptrs(2, shift_at=1, by=8)), EINVAL),               # peer not 16-byte aligned
        (dict(C=0), EINVAL), (dict(src_ld=15), EINVAL), (dict(dst_ld=15), EINVAL),
        (dict(src=P + 8), EUNSUPPORTED), (dict(src_ld=18), EUNSUPPORTED), (dict(out_col=2), EUNSUPPORTED),
        (dict(stride_b=50), EUNSUPPORTED), (dict(out_ld=98), EUNSUPPORTED),
        # order: the peers, then rows and C % gl, then the hop's own checks
        (dict(plan=None, peers=None), EINVAL), (dict(peers=_ptrs(17), n_peers=17, src=P + 8), EINVAL),
        (dict(rows_per_peer=31, src=P + 8), EINVAL), (dict(C=12, out_col=2), EINVAL),
    ]
    return lib.b200gf_hop_scatter, d, cases


def _hop_bcast(lib, plans):
    d = dict(plan=plans(v2=1), e=1, direction=1, src=P, src_ld=48, C=48, peers=_ptrs(3), n_peers=3, mc=None, row0=0,
             out_ld=48, stream=None)
    cases = [
        ({}, PASS), (dict(direction=0), PASS), (dict(C=44), PASS), (dict(peers=_ptrs(16), n_peers=16), PASS),
        (dict(mc=P), PASS), (dict(row0=64, out_ld=56), PASS), (dict(C=24, src_ld=24, out_ld=24), PASS),
        (dict(plan=None), EINVAL), (dict(src=None), EINVAL), (dict(e=2), EINVAL), (dict(direction=2), EINVAL),
        (dict(plan=plans(has_bwd=0, v2=1)), EINVAL),
        (dict(peers=None), EINVAL), (dict(n_peers=0), EINVAL), (dict(peers=_ptrs(17), n_peers=17), EINVAL),
        (dict(peers=_ptrs(3, null_at=2)), EINVAL), (dict(row0=-1), EINVAL), (dict(out_ld=0), EINVAL),
        (dict(out_ld=47), EINVAL), (dict(C=0), EINVAL), (dict(src_ld=47), EINVAL),
        (dict(peers=_ptrs(3, shift_at=1, by=16)), EUNSUPPORTED),        # 16- but not 32-byte aligned peer
        (dict(peers=_ptrs(3, shift_at=0, by=4)), EUNSUPPORTED),
        (dict(src=P + 16), EUNSUPPORTED), (dict(mc=P + 16), EUNSUPPORTED), (dict(src_ld=52), EUNSUPPORTED),
        (dict(out_ld=52), EUNSUPPORTED), (dict(plan=plans()), EUNSUPPORTED),   # no 32-bit offsets
        (dict(C=16, src_ld=16, out_ld=16), EUNSUPPORTED),               # a 64-byte row: only the grid epilogue has one
        (dict(C=8, src_ld=8, out_ld=8), EUNSUPPORTED),                  # a 32-byte row
        # order
        (dict(peers=None, C=16), EINVAL), (dict(row0=-1, src=P + 16), EINVAL), (dict(out_ld=47, src=P + 16), EINVAL),
    ]
    return lib.b200gf_hop_bcast, d, cases


def _hop_grid(lib, plans):
    d = dict(plan=plans(v2=1), e=1, direction=1, src=P, src_ld=16, C=16, bc_peers=_ptrs(2), n_bc=2, row0=0, bc_ld=16,
             sc_peers=_ptrs(2), n_sc=2, rows_per_peer=32, out_ld=96, out_col=8, gl=8, stride_b=48, stream=None)
    cases = [
        ({}, PASS), (dict(direction=0), PASS), (dict(C=48, src_ld=48, bc_ld=48), PASS),
        (dict(C=24, src_ld=24, bc_ld=24), PASS), (dict(bc_peers=None, n_bc=0), PASS),   # last hop: scatter only
        (dict(bc_peers=_ptrs(16), n_bc=16, sc_peers=_ptrs(16), n_sc=16, rows_per_peer=4), PASS),
        (dict(sc_peers=_ptrs(2, shift_at=1, by=16)), PASS),             # scatter peers need 16 bytes only
        (dict(plan=None), EINVAL), (dict(src=None), EINVAL), (dict(e=2), EINVAL), (dict(direction=2), EINVAL),
        (dict(plan=plans(has_bwd=0, v2=1)), EINVAL),
        (dict(bc_peers=None), EINVAL), (dict(bc_peers=_ptrs(17), n_bc=17), EINVAL),
        (dict(bc_peers=_ptrs(2, null_at=0)), EINVAL), (dict(row0=-1), EINVAL), (dict(bc_ld=0), EINVAL),
        (dict(bc_peers=None, n_bc=0, sc_peers=None, n_sc=0), EINVAL),   # neither all-gather nor scatter
        (dict(sc_peers=None), EINVAL), (dict(n_sc=0), EINVAL), (dict(sc_peers=_ptrs(17), n_sc=17), EINVAL),
        (dict(sc_peers=_ptrs(2, null_at=1)), EINVAL), (dict(sc_peers=_ptrs(2, shift_at=0, by=8)), EINVAL),
        (dict(rows_per_peer=31), EINVAL), (dict(C=20, src_ld=24, bc_ld=24), EINVAL), (dict(gl=0), EINVAL),
        (dict(bc_ld=15), EINVAL), (dict(src_ld=15), EINVAL),
        (dict(bc_peers=_ptrs(2, shift_at=1, by=16)), EUNSUPPORTED), (dict(src=P + 16), EUNSUPPORTED),
        (dict(out_col=4, gl=4, C=16), EUNSUPPORTED), (dict(out_col=4), EUNSUPPORTED), (dict(stride_b=52), EUNSUPPORTED),
        (dict(bc_ld=20), EUNSUPPORTED), (dict(plan=plans()), EUNSUPPORTED), (dict(C=8, gl=8, src_ld=8, bc_ld=8), EUNSUPPORTED),
        # order: all-gather peers, scatter peers, rows and C % gl, then the kernel's alignment
        (dict(bc_peers=None, sc_peers=None), EINVAL), (dict(n_sc=0, rows_per_peer=31), EINVAL),
        (dict(rows_per_peer=31, src=P + 16), EINVAL),
    ]
    return lib.b200gf_hop_grid, d, cases


def _bcast_rows(lib, plans):
    d = dict(dtype=F32, src=P, src_ld=8, n_rows=N, C=8, peers=_ptrs(2), n_peers=2, mc=None, row0=0, out_ld=8,
             stream=None)
    cases = [
        ({}, PASS), (dict(dtype=F64), PASS), (dict(mc=P), PASS), (dict(C=4, src_ld=12, out_ld=4, row0=5), PASS),
        (dict(peers=_ptrs(16), n_peers=16), PASS), (dict(peers=_ptrs(2, shift_at=1, by=16)), PASS), (dict(n_rows=0), OK),
        (dict(src=None), EINVAL), (dict(peers=None), EINVAL), (dict(n_peers=0), EINVAL),
        (dict(peers=_ptrs(17), n_peers=17), EINVAL), (dict(peers=_ptrs(2, null_at=1)), EINVAL), (dict(row0=-1), EINVAL),
        (dict(out_ld=0), EINVAL), (dict(out_ld=7), EINVAL), (dict(C=0), EINVAL), (dict(src_ld=7), EINVAL),
        (dict(peers=_ptrs(2, shift_at=1, by=4)), EUNSUPPORTED),         # every peer takes 16-byte stores
        (dict(dtype=F64, peers=_ptrs(2, shift_at=0, by=8)), EUNSUPPORTED),
        (dict(src=P + 8), EUNSUPPORTED), (dict(mc=P + 8), EUNSUPPORTED), (dict(C=6, src_ld=8), EUNSUPPORTED),
        (dict(dtype=F64, C=5), EUNSUPPORTED), (dict(src_ld=10), EUNSUPPORTED), (dict(out_ld=10), EUNSUPPORTED),
        (dict(dtype=7), EUNSUPPORTED),
        # order: an empty copy returns before the alignment and dtype checks
        (dict(n_rows=0, peers=_ptrs(2, shift_at=1, by=4)), OK), (dict(n_rows=0, dtype=7), OK),
        (dict(peers=_ptrs(2, null_at=0), src=P + 8), EINVAL), (dict(out_ld=7, peers=_ptrs(2, shift_at=1, by=4)), EINVAL),
    ]
    return lib.b200gf_bcast_rows, d, cases


def _scatter_rows(lib, plans):
    d = dict(dtype=F32, src=P, src_ld=16, n_rows=N, C=16, peers=_ptrs(2), n_peers=2, rows_per_peer=32, out_ld=96,
             out_col=8, gl=8, stride_b=48, stream=None)
    cases = [
        ({}, PASS), (dict(dtype=F64), PASS), (dict(gl=4, C=12, out_col=4), PASS),
        (dict(peers=_ptrs(16), n_peers=16, rows_per_peer=4), PASS), (dict(dtype=F64, src=P + 16), PASS),
        (dict(n_rows=0), OK),
        (dict(src=None), EINVAL), (dict(peers=None), EINVAL), (dict(n_peers=0), EINVAL),
        (dict(peers=_ptrs(17), n_peers=17), EINVAL), (dict(peers=_ptrs(2, null_at=1)), EINVAL),
        (dict(peers=_ptrs(2, shift_at=1, by=8)), EINVAL), (dict(rows_per_peer=0), EINVAL), (dict(gl=0), EINVAL),
        (dict(rows_per_peer=31), EINVAL), (dict(C=12), EINVAL), (dict(C=0), EINVAL), (dict(src_ld=15), EINVAL),
        (dict(src=P + 8), EUNSUPPORTED),                                # 16-byte vector loads of the source
        (dict(dtype=F64, src=P + 8), EUNSUPPORTED), (dict(src=P + 4), EUNSUPPORTED),
        (dict(out_col=2), EUNSUPPORTED), (dict(src_ld=18), EUNSUPPORTED), (dict(stride_b=50), EUNSUPPORTED),
        (dict(out_ld=98), EUNSUPPORTED), (dict(dtype=F64, out_col=1), EUNSUPPORTED), (dict(dtype=7), EUNSUPPORTED),
        # order
        (dict(n_rows=0, src=P + 8), OK), (dict(n_rows=0, dtype=7), OK), (dict(src=P + 8, C=12), EINVAL),
        (dict(rows_per_peer=31, src=P + 8), EINVAL), (dict(peers=_ptrs(2, shift_at=1, by=8), src=P + 8), EINVAL),
    ]
    return lib.b200gf_scatter_rows, d, cases


M = 4


def _nv_forward(lib, plans):
    plan = plans()
    need = lib.b200gf_nv_workspace_bytes(plan, B, G, F, K, M, 0) - 256
    d = dict(plan=plan, x=P, x_ld=C, W=P, node_tap=P, M=M, bias=P, bpn=0, y=P, y_ld=CF, ws=WS, wsb=need,
             B=B, G=G, F=F, K=K, stream=None)
    cases = [
        ({}, PASS), (dict(K=1, ws=None, wsb=0), PASS), (dict(bias=None, bpn=1), PASS),
        (dict(plan=None), EINVAL), (dict(x=None), EINVAL), (dict(W=None), EINVAL), (dict(node_tap=None), EINVAL),
        (dict(y=None), EINVAL), (dict(M=0), EINVAL), (dict(F=0), EINVAL), (dict(bpn=2), EINVAL),
        (dict(x_ld=C - 1), EINVAL), (dict(y_ld=CF - 1), EINVAL), (dict(plan=plans(n_cols=65)), EINVAL),
        (dict(K=25), EUNSUPPORTED),                                     # T = 1 + 2 * 24 = 49 > MAX_TERMS
        (dict(ws=MISALIGNED), EINVAL), (dict(ws=None), EWORKSPACE), (dict(wsb=need - 1), EWORKSPACE),
        # order
        (dict(K=25, ws=MISALIGNED), EUNSUPPORTED), (dict(x_ld=C - 1, K=25), EINVAL),
        (dict(ws=MISALIGNED, wsb=need - 1), EINVAL), (dict(ws=None, wsb=0), EWORKSPACE),
        (dict(plan=plans(N=0), ws=MISALIGNED), EINVAL), (dict(plan=plans(N=0), ws=None, wsb=0), OK),
    ]
    return lib.b200gf_nv_forward, d, cases


def _nv_backward(lib, plans):
    plan = plans()
    need = lib.b200gf_nv_workspace_bytes(plan, B, G, F, K, M, 1) - 256
    d = dict(plan=plan, dy=P, dy_ld=CF, x=P, x_ld=C, W=P, node_tap=P, M=M, tap_rowptr=P, tap_nodes=P, dx=P, dx_ld=C,
             dh=P, dbias=P, bpn=0, ws=WS, wsb=need, B=B, G=G, F=F, K=K, stream=None)
    cases = [
        ({}, PASS), (dict(K=1, wsb=lib.b200gf_nv_workspace_bytes(plan, B, G, F, 1, M, 1) - 256), PASS),
        (dict(dx=None, dx_ld=0), PASS), (dict(plan=plans(N=0)), PASS),
        (dict(plan=None), EINVAL), (dict(plan=plans(has_bwd=0)), EINVAL), (dict(dy=None), EINVAL),
        (dict(tap_rowptr=None), EINVAL), (dict(tap_nodes=None), EINVAL), (dict(dh=None), EINVAL),
        (dict(M=0), EINVAL), (dict(bpn=-1), EINVAL), (dict(dy_ld=CF - 1), EINVAL), (dict(x_ld=C - 1), EINVAL),
        (dict(dx_ld=C - 1), EINVAL), (dict(K=25), EUNSUPPORTED),
        (dict(ws=MISALIGNED), EINVAL), (dict(ws=None), EWORKSPACE), (dict(wsb=need - 1), EWORKSPACE),
        # order
        (dict(K=25, ws=None), EUNSUPPORTED), (dict(ws=MISALIGNED, wsb=need - 1), EINVAL),
        (dict(plan=plans(N=0), ws=None), EWORKSPACE), (dict(plan=plans(N=0), ws=MISALIGNED), EINVAL),
    ]
    return lib.b200gf_nv_backward, d, cases


def _nv_pack_taps(lib, plans):
    d = dict(dtype=F64, h=P, W=P, F=F, E=2, K=K, G=G, M=M, stream=None)
    cases = [({}, PASS), (dict(dtype=F32), PASS), (dict(h=None), EINVAL), (dict(W=None), EINVAL), (dict(M=0), EINVAL),
             (dict(E=0), EINVAL), (dict(dtype=7), EUNSUPPORTED), (dict(dtype=7, K=0), EINVAL)]
    return lib.b200gf_nv_pack_taps, d, cases


TMAX, PA = 2, 2
WIDE = dict(G=2000, F=2000, P=2000, x_ld=BIG, out_ld=BIG, dy_ld=BIG, dx_ld=BIG)   # F P G > INT32_MAX / 2


def _arma_forward(lib, plans):
    plan = plans()
    need = lib.b200gf_arma_workspace_bytes(plan, B, G, F, PA, TMAX, 0) - 256
    need_st = lib.b200gf_arma_workspace_bytes(plan, B, G, F, PA, TMAX, 1) - 256
    d = dict(plan=plan, d=P, psi=P, varphi=P, tMax=TMAX, B=B, G=G, F=F, P=PA, x=P, x_ld=C, out=P, out_ld=CF, states=None,
             ws=WS, wsb=need, stream=None)
    cases = [
        ({}, PASS), (dict(tMax=0), PASS), (dict(states=P, wsb=need_st), PASS), (dict(plan=plans(N=0)), OK),
        (dict(plan=None), EINVAL), (dict(d=None), EINVAL), (dict(varphi=None), EINVAL), (dict(out=None), EINVAL),
        (dict(tMax=-1), EINVAL), (dict(P=0), EINVAL), (dict(x_ld=C - 1), EINVAL), (dict(out_ld=CF - 1), EINVAL),
        (dict(plan=plans(n_cols=65)), EINVAL), (dict(WIDE), EUNSUPPORTED),
        (dict(ws=MISALIGNED), EINVAL), (dict(ws=None), EWORKSPACE), (dict(wsb=need - 1), EWORKSPACE),
        (dict(states=P, wsb=need_st - 1), EWORKSPACE), (dict(states=P + 8, wsb=need_st), EINVAL),
        # order
        (dict(tMax=-1, ws=None), EINVAL), (dict(WIDE, ws=None), EUNSUPPORTED),
        (dict(ws=MISALIGNED, wsb=need - 1), EINVAL),
        (dict(states=P + 8, ws=None), EWORKSPACE), (dict(states=P + 8, ws=MISALIGNED), EINVAL),
        (dict(states=P + 8, wsb=0), EINVAL),
        (dict(plan=plans(N=0), ws=None), EWORKSPACE), (dict(plan=plans(N=0), ws=MISALIGNED), EINVAL),
    ]
    return lib.b200gf_arma_forward, d, cases


def _arma_backward(lib, plans):
    plan = plans()
    need = lib.b200gf_arma_workspace_bytes(plan, B, G, F, PA, TMAX, 2) - 256
    d = dict(plan=plan, d=P, psi=P, varphi=P, tMax=TMAX, B=B, G=G, F=F, P=PA, dy=P, dy_ld=CF, states=P, dx=P, dx_ld=C,
             dpsi=P, dvarphi=P, ws=WS, wsb=need, stream=None)
    cases = [
        ({}, PASS), (dict(dx=None, dx_ld=0), PASS), (dict(plan=plans(N=0)), PASS),
        (dict(plan=None), EINVAL), (dict(plan=plans(has_bwd=0)), EINVAL), (dict(states=None), EINVAL),
        (dict(dpsi=None), EINVAL), (dict(tMax=-1), EINVAL), (dict(dy_ld=CF - 1), EINVAL), (dict(dx_ld=C - 1), EINVAL),
        (dict(WIDE), EUNSUPPORTED),
        (dict(ws=MISALIGNED), EINVAL), (dict(ws=None), EWORKSPACE), (dict(wsb=need - 1), EWORKSPACE),
        # order
        (dict(dy_ld=CF - 1, ws=None), EINVAL), (dict(WIDE, ws=None), EUNSUPPORTED),
        (dict(ws=MISALIGNED, wsb=need - 1), EINVAL),
        (dict(plan=plans(N=0), ws=None), EWORKSPACE), (dict(plan=plans(N=0), ws=MISALIGNED), EINVAL),
    ]
    return lib.b200gf_arma_backward, d, cases


# ------------------------------------------------------------------------------------------------ dtype-based
N, NNZ, BS = 64, 300, 3


def _attention_cases(two_scores):
    cases = [({}, PASS), (dict(dtype=F32), PASS), (dict(N=0, nnz=0), OK),
             (dict(dtype=7), EUNSUPPORTED), (dict(N=-1), EINVAL), (dict(nnz=-1), EINVAL), (dict(Bs=0), EINVAL),
             (dict(rowptr=None), EINVAL), (dict(col=None), EINVAL), (dict(mixer=None), EINVAL),
             (dict(N=BIG), EUNSUPPORTED), (dict(nnz=BIG), EUNSUPPORTED),
             (dict(nnz=0, col=None), PASS),
             # order
             (dict(dtype=7, mixer=None), EINVAL), (dict(dtype=7, N=BIG), EUNSUPPORTED), (dict(N=BIG, Bs=0), EINVAL),
             (dict(dtype=7, N=0, nnz=0), EUNSUPPORTED)]
    cases += [(dict(s_src=None), EINVAL), (dict(s_dst=None), EINVAL)] if two_scores else [(dict(s=None), EINVAL)]
    return cases


def _egate_attention_forward(lib, plans):
    d = dict(dtype=F64, N=N, nnz=NNZ, Bs=BS, rowptr=P, col=P, s=P, mixer=P, alpha=P, stream=None)
    return lib.b200gf_egate_attention_forward, d, _attention_cases(False) + [(dict(alpha=None), EINVAL)]


def _attention_forward(lib, plans):
    d = dict(dtype=F64, N=N, nnz=NNZ, Bs=BS, rowptr=P, col=P, s_src=P, s_dst=P, mixer=P, alpha=P, stream=None)
    return lib.b200gf_attention_forward, d, _attention_cases(True) + [(dict(alpha=None), EINVAL)]


def _backward_extra():
    return [(dict(rowptrT=None), EINVAL), (dict(permT=None), EINVAL), (dict(dalpha=None), EINVAL),
            (dict(dlogit=None), EINVAL), (dict(dsig1=None), EINVAL), (dict(dsig2=None), EINVAL),
            (dict(nnz=0, permT=None, alpha=None, dalpha=None, dlogit=None), PASS),
            (dict(N=0, nnz=0, dsig2=None), EINVAL)]


def _egate_attention_backward(lib, plans):
    d = dict(dtype=F64, N=N, nnz=NNZ, Bs=BS, rowptr=P, col=P, rowptrT=P, permT=P, s=P, mixer=P, alpha=P, dalpha=P,
             dlogit=P, dsig1=P, dsig2=P, stream=None)
    return lib.b200gf_egate_attention_backward, d, _attention_cases(False) + _backward_extra()


def _attention_backward(lib, plans):
    d = dict(dtype=F64, N=N, nnz=NNZ, Bs=BS, rowptr=P, col=P, rowptrT=P, permT=P, s_src=P, s_dst=P, mixer=P, alpha=P,
             dalpha=P, dlogit=P, dsig1=P, dsig2=P, stream=None)
    return lib.b200gf_attention_backward, d, _attention_cases(True) + _backward_extra()


GC = 4


def _gated_hop_forward(lib, plans):
    d = dict(dtype=F32, N=N, Bs=BS, C=GC, rowptrT=P, colT=P, valT=P, posT=P, gate=P, gate_sb=NNZ, gate_sp=1, src=P,
             src_ld=BS * GC, dst=P, dst_ld=BS * GC, stream=None)
    cases = [({}, PASS), (dict(dtype=F64), PASS), (dict(src_ld=BS * GC + 1), PASS), (dict(N=0), OK),
             (dict(dtype=7), EUNSUPPORTED), (dict(N=-1), EINVAL), (dict(Bs=0), EINVAL), (dict(C=0), EINVAL),
             (dict(valT=None), EINVAL), (dict(gate=None), EINVAL), (dict(dst=None), EINVAL),
             (dict(src_ld=BS * GC - 1), EINVAL), (dict(dst_ld=BS * GC - 1), EINVAL), (dict(N=BIG), EUNSUPPORTED),
             # order
             (dict(dtype=7, src_ld=1), EINVAL), (dict(N=BIG, gate=None), EINVAL), (dict(dtype=7, N=BIG), EUNSUPPORTED),
             (dict(dtype=7, N=0), EUNSUPPORTED)]
    return lib.b200gf_gated_hop_forward, d, cases


def _gated_hop_backward(lib, plans):
    ld = BS * GC
    d = dict(dtype=F32, N=N, Bs=BS, C=GC, rowptr=P, col=P, val=P, pos=P, m_rowptr=P, m_col=P, m_sval=P, gate=P,
             gate_sb=NNZ, gate_sp=1, src=P, src_ld=ld, ddst=P, ddst_ld=ld, dsrc=P, dsrc_ld=ld, dgate=P, dgate_sb=NNZ,
             dgate_sp=1, stream=None)
    cases = [({}, PASS), (dict(dtype=F64), PASS), (dict(dgate=None, m_rowptr=None, src=None), PASS),
             (dict(dsrc=None, rowptr=None, gate=None), PASS), (dict(N=0), OK), (dict(N=0, dsrc=None), OK),
             (dict(dtype=7), EUNSUPPORTED), (dict(dsrc=None, dgate=None), EINVAL), (dict(ddst=None), EINVAL),
             (dict(C=0), EINVAL), (dict(rowptr=None), EINVAL), (dict(m_sval=None), EINVAL), (dict(src=None), EINVAL),
             (dict(dsrc_ld=ld - 1), EINVAL), (dict(src_ld=ld - 1), EINVAL), (dict(ddst_ld=ld - 1), EINVAL),
             (dict(N=BIG), EUNSUPPORTED),
             # order
             (dict(dtype=7, ddst_ld=ld - 1), EINVAL), (dict(N=BIG, ddst_ld=ld - 1), EINVAL),
             (dict(dtype=7, N=0), EUNSUPPORTED)]
    return lib.b200gf_gated_hop_backward, d, cases


NA, EB, EG, EF, EK = 40, 4, 3, 2, 3


def _ev_forward(lib, plans):
    d = dict(dtype=F32, NA=NA, B=EB, G=EG, F=EF, K=EK, rowptr=P, col=P, diag=P, nnz=NNZ, w=P, xT=P, states=P,
             n_states=2, Y=P, stream=None)
    cases = [({}, PASS), (dict(dtype=F64), PASS), (dict(B=3), PASS), (dict(K=1, states=None, n_states=0), PASS),
             (dict(nnz=0, w=None), PASS), (dict(NA=0), OK),
             (dict(dtype=7), EUNSUPPORTED), (dict(NA=-1), EINVAL), (dict(B=0), EINVAL), (dict(K=0), EINVAL),
             (dict(nnz=-1), EINVAL), (dict(rowptr=None), EINVAL), (dict(xT=None), EINVAL), (dict(w=None), EINVAL),
             (dict(states=None), EINVAL), (dict(n_states=0), EINVAL), (dict(K=4, n_states=1), EINVAL),
             (dict(NA=BIG), EUNSUPPORTED),
             # order
             (dict(dtype=7, states=None), EINVAL), (dict(NA=BIG, states=None), EUNSUPPORTED),
             (dict(NA=BIG, Y=None), EINVAL), (dict(dtype=7, NA=0), EUNSUPPORTED)]
    return lib.b200gf_ev_forward, d, cases


def _ev_backward(lib, plans):
    d = dict(dtype=F32, NA=NA, B=EB, G=EG, F=EF, K=EK, rowptr=P, col=P, rowptrT=P, colT=P, perm=P, diag=P, nnz=NNZ,
             w=P, xT=P, states=P, dY=P, lam=P, dw=P, dxT=P, stream=None)
    cases = [({}, PASS), (dict(dtype=F64), PASS), (dict(B=3), PASS), (dict(K=1, states=None), PASS),
             (dict(NA=0), OK),
             (dict(dtype=7), EUNSUPPORTED), (dict(NA=-1), EINVAL), (dict(F=0), EINVAL), (dict(perm=None), EINVAL),
             (dict(lam=None), EINVAL), (dict(dxT=None), EINVAL), (dict(states=None), EINVAL), (dict(dw=None), EINVAL),
             (dict(nnz=BIG), EUNSUPPORTED),
             # order
             (dict(dtype=7, lam=None), EINVAL), (dict(nnz=BIG, dw=None), EINVAL), (dict(dtype=7, nnz=BIG), EUNSUPPORTED),
             (dict(dtype=7, NA=0), EUNSUPPORTED)]
    return lib.b200gf_ev_backward, d, cases


LC = 7


def _relu_backward(lib, plans):
    d = dict(dtype=F32, y=P, y_ld=LC, dy=P, dy_ld=LC, out=P, out_ld=LC, n_rows=N, C=LC, stream=None)
    cases = [({}, PASS), (dict(dtype=F64), PASS), (dict(n_rows=0), OK),
             (dict(dtype=7), EUNSUPPORTED), (dict(y=None), EINVAL), (dict(n_rows=-1), EINVAL), (dict(C=0), EINVAL),
             (dict(y_ld=LC - 1), EINVAL), (dict(dy_ld=LC - 1), EINVAL), (dict(out_ld=LC - 1), EINVAL),
             # order: an empty call returns before the dtype is looked at
             (dict(dtype=7, n_rows=0), OK), (dict(dtype=7, out=None), EINVAL)]
    return lib.b200gf_relu_backward, d, cases


def _maxpool_forward(lib, plans):
    d = dict(dtype=F32, x=P, x_ld=LC, n_in=N, C=LC, nb=P, n_out=N // 2, max_nb=5, out=P, out_ld=LC, argmax=None,
             stream=None)
    cases = [({}, PASS), (dict(dtype=F64, argmax=P), PASS), (dict(n_out=0), OK),
             (dict(dtype=7), EUNSUPPORTED), (dict(x=None), EINVAL), (dict(nb=None), EINVAL), (dict(n_in=0), EINVAL),
             (dict(n_out=-1), EINVAL), (dict(max_nb=0), EINVAL), (dict(x_ld=LC - 1), EINVAL),
             (dict(out_ld=LC - 1), EINVAL), (dict(n_in=BIG), EUNSUPPORTED),
             # order
             (dict(dtype=7, n_out=0), OK), (dict(n_in=BIG, n_out=0), EUNSUPPORTED), (dict(dtype=7, n_in=BIG), EUNSUPPORTED),
             (dict(n_in=BIG, x_ld=1), EINVAL)]
    return lib.b200gf_maxpool_forward, d, cases


def _maxpool_backward(lib, plans):
    d = dict(dtype=F32, dy=P, dy_ld=LC, argmax=P, n_out=N // 2, C=LC, dx=P, dx_ld=LC, n_in=N, stream=None)
    cases = [({}, PASS), (dict(dtype=F64), PASS), (dict(n_out=0), PASS),
             (dict(dtype=7), EUNSUPPORTED), (dict(dy=None), EINVAL), (dict(argmax=None), EINVAL), (dict(n_in=0), EINVAL),
             (dict(dy_ld=LC - 1), EINVAL), (dict(dx_ld=LC - 1), EINVAL),
             # order: the dtype is checked before dx is cleared, also for an empty call
             (dict(dtype=7, n_out=0), EUNSUPPORTED), (dict(dtype=7, dx=None), EINVAL)]
    return lib.b200gf_maxpool_backward, d, cases


def _to_node_major(lib, plans):
    d = dict(dtype=F32, src=P, dst=P, dst_ld=8, N=N, C=LC, stream=None)
    cases = [({}, PASS), (dict(dtype=F64), PASS), (dict(N=0), OK), (dict(N=65535 * 32 + 1), PASS),
             (dict(dtype=7), EUNSUPPORTED), (dict(src=None), EINVAL), (dict(N=-1), EINVAL), (dict(C=0), EINVAL),
             (dict(dst_ld=LC - 1), EINVAL), (dict(dtype=7, N=0), EUNSUPPORTED), (dict(dtype=7, dst_ld=1), EINVAL)]
    return lib.b200gf_to_node_major, d, cases


def _to_feature_major(lib, plans):
    d = dict(dtype=F32, src=P, src_ld=8, dst=P, N=N, C=LC, stream=None)
    cases = [({}, PASS), (dict(dtype=F64), PASS), (dict(N=0), OK),
             (dict(dtype=7), EUNSUPPORTED), (dict(dst=None), EINVAL), (dict(N=-1), EINVAL), (dict(C=-3), EINVAL),
             (dict(src_ld=LC - 1), EINVAL), (dict(dtype=7, N=0), EUNSUPPORTED), (dict(dtype=7, src_ld=1), EINVAL)]
    return lib.b200gf_to_feature_major, d, cases


def _pack_taps(lib, plans):
    d = dict(dtype=F32, h=P, W=P, F=F, E=2, K=K, G=G, transpose=0, stream=None)
    cases = [({}, PASS), (dict(dtype=F64, transpose=1), PASS),
             (dict(dtype=7), EUNSUPPORTED), (dict(h=None), EINVAL), (dict(W=None), EINVAL), (dict(E=0), EINVAL),
             (dict(G=-1), EINVAL), (dict(dtype=7, K=0), EINVAL)]
    return lib.b200gf_pack_taps, d, cases


TP, TQ, TT = 8, 12, 3


def _tap_contract(lib, plans):
    d = dict(dtype=F32, n_rows=N, B=B, P=TP, Q=TQ, T=TT, zs=_ptrs(TT), z_ld=_lds(TT, B * TP), W=P, bias=P, bpn=0,
             out=P, out_ld=B * TQ, accumulate=0, scratch=None, scratch_bytes=0, stream=None)
    many = TT + 48                                                   # more terms than one TermList holds
    cases = [({}, PASS), (dict(dtype=F64), PASS), (dict(accumulate=1), PASS), (dict(n_rows=0), OK),
             (dict(T=many, zs=_ptrs(many), z_ld=_lds(many, B * TP)), PASS),
             (dict(dtype=7), EUNSUPPORTED), (dict(n_rows=-1), EINVAL), (dict(T=0), EINVAL), (dict(zs=None), EINVAL),
             (dict(z_ld=None), EINVAL), (dict(W=None), EINVAL), (dict(out=None), EINVAL),
             (dict(out_ld=B * TQ - 1), EINVAL), (dict(zs=_ptrs(TT, null_at=1)), EINVAL),
             (dict(dtype=F64, zs=_ptrs(TT, null_at=2)), EINVAL), (dict(z_ld=_lds(TT, B * TP - 1)), EINVAL),
             # order: a null term is reported before an unsupported dtype
             (dict(dtype=7, zs=_ptrs(TT, null_at=0)), EINVAL), (dict(dtype=7, z_ld=_lds(TT, 1)), EINVAL),
             (dict(dtype=7, n_rows=0), OK), (dict(dtype=7, out_ld=1), EINVAL)]
    return lib.b200gf_tap_contract, d, cases


def _tap_grad(lib, plans):
    sb = lib.b200gf_tap_grad_scratch_bytes(F32, N, B, TP, TQ, TT)
    d = dict(dtype=F32, n_rows=N, B=B, P=TP, Q=TQ, T=TT, A=P, a_ld=B * TP, vs=_ptrs(TT), v_ld=_lds(TT, B * TQ), dW=P,
             scratch=WS, scratch_bytes=sb, stream=None)
    cases = [({}, PASS), (dict(dtype=F64, scratch_bytes=2 * sb), PASS), (dict(a_ld=B * TP + 1), PASS),
             (dict(dtype=7), EUNSUPPORTED), (dict(A=None), EINVAL), (dict(dW=None), EINVAL), (dict(scratch=None), EINVAL),
             (dict(T=0), EINVAL), (dict(a_ld=B * TP - 1), EINVAL), (dict(scratch_bytes=sb - 1), EWORKSPACE),
             (dict(vs=_ptrs(TT, null_at=2)), EINVAL), (dict(v_ld=_lds(TT, B * TQ - 1)), EINVAL),
             # order: workspace, then dtype, then the terms
             (dict(dtype=7, scratch_bytes=0), EWORKSPACE), (dict(dtype=7, vs=_ptrs(TT, null_at=0)), EUNSUPPORTED),
             (dict(scratch_bytes=0, a_ld=1), EINVAL)]
    return lib.b200gf_tap_grad, d, cases


ENTRY_POINTS = {f.__name__[1:]: f for f in (
    _lsigf_forward, _lsigf_forward_act, _lsigf_backward, _hop, _nv_forward, _nv_backward, _nv_pack_taps,
    _hop_scatter, _hop_bcast, _hop_grid, _bcast_rows, _scatter_rows, _arma_forward, _arma_backward, _egate_attention_forward, _egate_attention_backward, _attention_forward,
    _attention_backward, _gated_hop_forward, _gated_hop_backward, _ev_forward, _ev_backward, _relu_backward,
    _maxpool_forward, _maxpool_backward, _to_node_major, _to_feature_major, _pack_taps, _tap_contract, _tap_grad)}


@pytest.mark.parametrize("entry", sorted(ENTRY_POINTS))
def test_return_codes_and_check_order(entry, lib, plans):
    fn, defaults, cases = ENTRY_POINTS[entry](lib, plans)
    assert len(cases) >= 8
    bad = _check(fn, defaults, cases)
    assert not bad, "\n".join("%s: expected %s, got %d" % (over or "valid arguments", want, rc) for over, want, rc in bad)
