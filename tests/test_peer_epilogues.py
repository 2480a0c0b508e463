"""The hop kernels' peer epilogues and row copies of the sharded LSIGF paths (gnn_b200.distributed), on one GPU.

Every instantiation the fused multi-GPU data path can launch has a row in PEER_CASES:
  * EPI_SCATTER (b200gf_hop_scatter, feature sharding): every computed row slice is also stored into the contraction
    operand of the rank that owns the row: peer r // rows_per_peer, local row r % rows_per_peer, column
    b*stride_b + out_col + g of local column b*gl + g.  spmm_hop_v2_kernel (L = 8, 16, 32) and
    spmm_hop_multirow_v2_kernel carry it as MODE 1; spmm_hop_kernel and spmm_hop_multirow_kernel take the same
    ScatterArgs when rows are 16-byte but not 32-byte aligned, or narrower than 128 bytes.
  * EPI_BCAST (b200gf_hop_bcast, node sharding): rows [row0, row0 + n_rows) of every peer's full-height matrix.
  * EPI_GRID (b200gf_hop_grid, 2-D grid): both; n_bc = 0 (the last hop of a chain) only scatters.
  * bcast_rows_kernel / scatter_rows_kernel: the same stores of an existing row block (the k = 0 term).

The peers are plain device buffers of one GPU.  All peers of a launch live in one SENT-filled arena with guard rows
between them, so that a store to the wrong peer, row or column lands on a canary of the same allocation.  Plans are row
slices of S^T (HOP_FWD) and S (HOP_BWD) with global columns (Plan.from_ops + distributed.row_slice), as the sharded
paths build them, with row0 != 0 and fewer rows than columns; every row runs both directions.  Source pad columns hold
NaN.  Each row is held to:
  * the componentwise fp64 bound orc.dot_bound(row lengths, |op| @ |X|) on every written region: each peer's rows
    (all-gather), each owner's slices (scatter) and the local dst of EPI_SCATTER;
  * canaries: everything outside each peer's contract keeps SENT.  An all-gather stores a lane's whole 32 bytes, so peer
    columns [C, padded(C)) may be written and nothing past them;
  * bit-identity: all peer copies of a launch are equal; the local dst of EPI_SCATTER equals its scattered slices; where
    the plain b200gf_hop on the same plan and buffers launches the same kernel (MODE 0, same L, GS and U), the peer output
    equals the plain hop's bit for bit (the peer epilogues keep a lane's 32 bytes adjacent, the local ones split them:
    spmm_kernels.cuh LaneMap).  Rows whose plain hop takes another kernel say so and are held to the bound only;
  * a rerun is bit-identical (dispatch_harness.check_case).

Not covered: the multicast store of the all-gather (multimem.st through an NVSwitch multicast address) needs a multicast
object across GPUs, so bcast_store's multicast branch stays untested on one device.  The sharded layers end to end are in
tests/test_distributed.py.
"""
import ctypes
import re

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import lsigf_oracle as orc
from dispatch_harness import (F32, F64, NPD, SENT, Result, _check, _graph, _lib, _padded, _st, check_case, child_traced,
                              library_kernels)

GUARD = 3            # SENT rows before, between and after the buffers of an arena
T_TERMS, T_AT = 3, 2  # the scatter operand holds T_TERMS terms per batch; rows land in term T_AT (distributed.py layout)


def _es(dtype):
    return torch.empty(0, dtype=dtype).element_size()


def _wide(dtype):
    return "float,int,8" if dtype == F32 else "double,int,4"


def _v2(dtype, L, mode):
    return r"spmm_hop_v2_kernel<%s,%d,4,256,%d,3,%d,1>" % (_wide(dtype), L, 4 if dtype == F32 else 3, mode)


def _mr2(dtype, mode):
    """64-byte rows: 2 lanes x 32 bytes, 8-lane row groups, 2 loads in flight."""
    return r"spmm_hop_multirow_v2_kernel<%s,2,8,2,256,%d,3,%d>" % (_wide(dtype), 4 if dtype == F32 else 3, mode)


def _one(dtype, L):
    """The 16-byte-lane single-row kernel (launch_one) of rows wider than 128 bytes."""
    return r"spmm_hop_kernel<%s,%d,%d,4,256,%d,3,0,0>" % (("float", 4, L, 6) if dtype == F32 else ("double", 2, L, 4))


def _mr(dtype, nv):
    """The 16-byte-lane multi-row kernel (launch_multirow) of rows of nv 16-byte vectors."""
    L, GS, U, MINB = {1: (1, 8, 1, 6), 2: (2, 8, 2, 6), 4: (4, 16, 2, 8), 8: (8, 32, 4, 6)}[nv]
    if dtype == F32:
        return r"spmm_hop_multirow_kernel<float,4,%d,%d,%d,256,%d,3>" % (L, GS, U, MINB)
    return r"spmm_hop_multirow_kernel<double,2,%d,%d,%d,256,4,3>" % (L, GS, U)


def _arena(n, rows, ld, dtype):
    """n buffers of [rows, ld] in one SENT-filled allocation with GUARD rows around each: (arena, first row of each)."""
    arena = torch.full((GUARD + n * (rows + GUARD), ld), SENT, dtype=dtype, device="cuda")
    return arena, [GUARD + i * (rows + GUARD) for i in range(n)]


def _ptrs(arena, bases):
    import gnn_b200
    step = arena.stride(0) * arena.element_size()
    return gnn_b200._cabi.ptr_array([arena.data_ptr() + b * step for b in bases])


class _Owners:
    """The scatter targets: n_sc contraction operands [rows_per_peer, B*T*G] in one arena.  Local column b*gl + g of plan
    row r lands in operand r // rpp, row r % rpp, column b*stride_b + out_col + g, with stride_b = T*G and out_col =
    t*G + g0 (term t of the T terms, column group g0 of the G in-features)."""

    def __init__(self, dtype, n_rows, C, gl, n_sc, rpp):
        self.B, self.gl, self.n_sc = C // gl, gl, n_sc
        self.rpp = rpp or -(-n_rows // n_sc)
        G = 2 * gl                                  # two column groups: this rank owns the second
        self.stride_b, self.out_col, self.out_ld = T_TERMS * G, T_AT * G + gl, self.B * T_TERMS * G
        self.arena, bases = _arena(n_sc, self.rpp, self.out_ld, dtype)
        self.ptrs = _ptrs(self.arena, bases)
        r = np.arange(n_rows)
        rows = np.asarray(bases, dtype=np.int64)[r // self.rpp] + r % self.rpp
        cols = np.concatenate([b * self.stride_b + self.out_col + np.arange(gl) for b in range(self.B)])
        self.ri = torch.as_tensor(np.repeat(rows[:, None], C, 1), device="cuda")
        self.ci = torch.as_tensor(np.repeat(cols[None, :], n_rows, 0), device="cuda")

    def args(self):
        return (self.ptrs, self.n_sc, self.rpp, self.out_ld, self.out_col, self.gl, self.stride_b)

    def record(self, res, tag, ref=None, bound=None):
        """[n_rows, C]: the slices as the owners received them; their bound (or exactness) and canaries go into res."""
        got = self.arena[self.ri, self.ci]
        mask = torch.zeros_like(self.arena, dtype=torch.bool)
        mask[self.ri, self.ci] = True
        res.checks.append(("%s owners" % tag, got, ref, bound))
        res.canaries.append(("%s owners outside their slices" % tag, self.arena[~mask]))
        res.finite.append(("%s owners" % tag, got))
        res.outputs.append(got)
        return got


class _Gathers:
    """The all-gather targets: n_bc full-height matrices [n_total, bc_ld] in one arena; rows [row0, row0 + n_rows)."""

    def __init__(self, dtype, n_total, C, n_bc, bc_ld=None, lane_pad=True):
        self.C, self.n_bc = C, n_bc
        self.Cp = _padded(C, dtype) if lane_pad else C
        self.bc_ld = bc_ld or _padded(C, dtype) + 32 // _es(dtype)    # columns past the padded width are canaries
        self.arena, self.bases = _arena(n_bc, n_total, self.bc_ld, dtype)
        self.ptrs = _ptrs(self.arena, self.bases)

    def record(self, res, tag, row0, n_rows, ref=None, bound=None):
        """[n_rows, C] of the first peer; every peer's copy is checked and must equal it bit for bit."""
        may = torch.zeros_like(self.arena, dtype=torch.bool)
        views = []
        for p, b in enumerate(self.bases):
            v = self.arena[b + row0:b + row0 + n_rows]
            may[b + row0:b + row0 + n_rows, :self.Cp] = True
            res.checks.append(("%s peer %d" % (tag, p), v[:, :self.C], ref, bound))
            res.finite.append(("%s peer %d" % (tag, p), v[:, :self.C]))
            views.append(v[:, :self.Cp])
        for p, v in enumerate(views[1:], 1):
            res.same.append(("%s: peer %d == peer 0" % (tag, p), v, views[0]))
        res.canaries.append(("%s peers outside rows [row0, row0+n_rows) x cols [0, padded(C))" % tag, self.arena[~may]))
        res.outputs.append(views[0])
        return views[0][:, :self.C]


def _hop_case(kind, dtype, C, gl=None, ld=None, n_peers=3, n_sc=3, rpp=None, N=3000, r0=700, n_rows=1100, graph="rand",
              plain=True):
    """One peer-epilogue hop, both directions, on rows [r0, r0 + n_rows) of a graph of N nodes.
    kind 'scatter': b200gf_hop_scatter into n_sc owners (and dst); 'bcast': b200gf_hop_bcast into n_peers peers; 'grid':
    b200gf_hop_grid (n_peers = 0: the last hop, scatter only).  ld: the source's (and dst's) leading dimension, default
    padded(C).  plain: the plain b200gf_hop of the same plan and buffers launches the same kernel with MODE 0, and the
    peer outputs must equal its output bit for bit."""
    def run():
        import gnn_b200
        from gnn_b200.distributed import row_slice, transpose_csr
        cabi, lib = _lib()
        npd, VW = NPD[dtype], 32 // _es(dtype)
        src_ld = ld or _padded(C, dtype)
        dst_ld = src_ld + VW                                   # same residue mod 32 bytes: the plain hop takes the same path
        m = _graph(graph, N)
        csr = (m.indptr.astype(np.int64), m.indices.astype(np.int32), m.data.astype(npd))
        ops = {cabi.HOP_FWD: row_slice(transpose_csr(csr, N), r0, r0 + n_rows), cabi.HOP_BWD: row_slice(csr, r0, r0 + n_rows)}
        plan = gnn_b200.gso.Plan.from_ops([ops[cabi.HOP_FWD]], [ops[cabi.HOP_BWD]], n_rows, N, dtype, "cuda")
        g = torch.Generator(device="cpu").manual_seed(C * 131 + N + n_rows)
        X = torch.randn(N, C, generator=g, dtype=torch.float64).to(dtype)
        src = torch.full((N + GUARD, src_ld), float("nan"), dtype=dtype, device="cuda")
        src[:N, :C] = X.cuda()
        Xd = X.double().numpy()
        res = Result()
        main = {}
        for direction, (rp, ci, va) in ops.items():
            tag = "fwd" if direction == cabi.HOP_FWD else "bwd"
            op = sp.csr_matrix((va.astype(np.float64), ci, rp), shape=(n_rows, N))
            ref = op @ Xd
            bound = orc.dot_bound(np.maximum(np.diff(rp)[:, None], 1), abs(op) @ np.abs(Xd), npd)
            copies = []                                        # [n_rows, C] results of this launch
            if kind == "scatter":
                own = _Owners(dtype, n_rows, C, gl, n_sc, rpp)
                dst = torch.full((n_rows + GUARD, dst_ld), SENT, dtype=dtype, device="cuda")
                _check(lib.b200gf_hop_scatter(plan.handle, 0, direction, src.data_ptr(), src_ld, dst.data_ptr(), dst_ld, C,
                                              *own.args(), _st()))
                copies.append(own.record(res, tag, ref, bound))
                res.checks.append(("%s dst" % tag, dst[:n_rows, :C], ref, bound))
                res.canaries += [("%s dst cols >= C" % tag, dst[:, C:]), ("%s dst rows >= n_rows" % tag, dst[n_rows:])]
                res.finite.append(("%s dst" % tag, dst[:n_rows, :C]))
                res.outputs.append(dst[:n_rows, :C])
                res.same.append(("%s: dst == its scattered slices" % tag, dst[:n_rows, :C], copies[0]))
            else:
                gat = _Gathers(dtype, N, C, n_peers) if n_peers else None
                bc = (gat.ptrs, n_peers, r0, gat.bc_ld) if gat else (None, 0, r0, 0)
                if kind == "bcast":
                    _check(lib.b200gf_hop_bcast(plan.handle, 0, direction, src.data_ptr(), src_ld, C, bc[0], bc[1], None,
                                                r0, bc[3], _st()))
                else:
                    own = _Owners(dtype, n_rows, C, gl, n_sc, rpp)
                    _check(lib.b200gf_hop_grid(plan.handle, 0, direction, src.data_ptr(), src_ld, C, *bc, *own.args(), _st()))
                    copies.append(own.record(res, tag, ref, bound))
                if gat:
                    copies.append(gat.record(res, tag, r0, n_rows, ref, bound))
            for i, c in enumerate(copies[1:], 1):
                res.same.append(("%s: all-gathered rows == scattered slices" % tag, c, copies[0]))
            if plain:
                pdst = torch.full((n_rows, dst_ld), SENT, dtype=dtype, device="cuda")
                _check(lib.b200gf_hop(plan.handle, 0, direction, src.data_ptr(), src_ld, pdst.data_ptr(), dst_ld, C, _st()))
                res.same.append(("%s: peer epilogue == plain hop" % tag, copies[0], pdst[:, :C]))
            main[direction] = copies[0]
        if graph == "sym":
            res.same.append(("symmetric S: FWD == BWD", main[cabi.HOP_FWD], main[cabi.HOP_BWD]))
        return res
    return run


def _rows_case(kind, dtype, C, gl=None, n_peers=3, n_sc=3, N=3000, r0=700, n_rows=1100):
    """b200gf_bcast_rows / b200gf_scatter_rows of an existing row block [n_rows, src_ld] (pad columns NaN): exact copies."""
    def run():
        cabi, lib = _lib()
        dt = cabi.F32 if dtype == F32 else cabi.F64
        src_ld = _padded(C, dtype) + 32 // _es(dtype)
        g = torch.Generator(device="cpu").manual_seed(C * 17 + n_rows)
        src = torch.full((n_rows + GUARD, src_ld), float("nan"), dtype=dtype, device="cuda")
        src[:n_rows, :C] = torch.randn(n_rows, C, generator=g, dtype=torch.float64).to(dtype).cuda()
        res = Result()
        if kind == "bcast":
            gat = _Gathers(dtype, N, C, n_peers, lane_pad=False)      # 16-byte copies: exactly [0, C) is written
            _check(lib.b200gf_bcast_rows(dt, src.data_ptr(), src_ld, n_rows, C, gat.ptrs, n_peers, None, r0, gat.bc_ld, _st()))
            got = gat.record(res, "rows", r0, n_rows)
        else:
            own = _Owners(dtype, n_rows, C, gl, n_sc, None)
            _check(lib.b200gf_scatter_rows(dt, src.data_ptr(), src_ld, n_rows, C, *own.args(), _st()))
            got = own.record(res, "rows")
        res.same.append(("copy == source", got, src[:n_rows, :C]))
        return res
    return run


def _name(dtype):
    return "f32" if dtype == F32 else "f64"


def _rows():
    rows = []
    scatter = set()

    def add(cid, fn, kernels, scatters=False):
        rows.append((cid, fn, kernels))
        if scatters:
            scatter.add(cid)

    for dt in (F32, F64):
        q = 32 // _es(dt)                                      # columns per 32-byte lane
        n = _name(dt)
        # EPI_SCATTER, v2: the scatter sizes chunks by row width alone, L = 8 / 16 / 32; the plain hop of a partitioned
        # plan does too, so it launches the same geometry with MODE 0
        for L, C, gl in ((8, 6 * q, 3 * q), (16, 12 * q, 4 * q), (32, 75 * q, 25 * q) if dt == F32 else (32, 20 * q, 10 * q)):
            add("scatter-v2-L%d-C%d-%s" % (L, C, n), _hop_case("scatter", dt, C, gl),
                [_v2(dt, L, 1)] * 2 + [_v2(dt, L, 0)] * 2, True)
        add("scatter-mr2-C%d-%s" % (2 * q, n), _hop_case("scatter", dt, 2 * q, q), [_mr2(dt, 1)] * 2 + [_mr2(dt, 0)] * 2, True)
        # EPI_BCAST: C of 3-4 lanes -> L = 4, 5-8 -> 8, 9-16 -> 16, more -> 32 (C = 75 lanes: 3 column chunks)
        add("bcast-v2-L4-C%d-%s" % (3 * q, n), _hop_case("bcast", dt, 3 * q, plain=False),
            [_v2(dt, 4, 2)] * 2)    # the plain hop of 3 lanes is the 16-byte multirow kernel: bound only
        for L, C in ((8, 6 * q - q // 2), (16, 13 * q - q // 2), (32, 75 * q)):   # C not a whole number of lanes
            add("bcast-v2-L%d-C%d-%s" % (L, C, n), _hop_case("bcast", dt, C), [_v2(dt, L, 2)] * 2 + [_v2(dt, L, 0)] * 2)
        # EPI_GRID: 64-byte rows take the multi-row v2 kernel, as the plain hop does
        add("grid-mr2-C%d-%s" % (2 * q, n), _hop_case("grid", dt, 2 * q, q), [_mr2(dt, 3)] * 2 + [_mr2(dt, 0)] * 2, True)
        add("grid-v2-L4-C%d-%s" % (4 * q, n), _hop_case("grid", dt, 4 * q, 2 * q, plain=False),
            [_v2(dt, 4, 3)] * 2, True)    # the plain hop of 4 lanes is the 16-byte multirow kernel: bound only
        for L, C, gl in ((8, 6 * q, 2 * q), (16, 12 * q, 6 * q), (32, 40 * q, 20 * q)):
            add("grid-v2-L%d-C%d-%s" % (L, C, n), _hop_case("grid", dt, C, gl), [_v2(dt, L, 3)] * 2 + [_v2(dt, L, 0)] * 2, True)
        add("grid-v2-L8-last-hop-%s" % n, _hop_case("grid", dt, 6 * q, 2 * q, n_peers=0),
            [_v2(dt, 8, 3)] * 2 + [_v2(dt, 8, 0)] * 2, True)
        # 16-byte scatter route: a leading dimension of whole 16-byte vectors but not whole 32-byte lanes keeps the v2
        # kernels out for the scatter and the plain hop alike
        h = q // 2
        for L, C, gl in ((16, 6 * q, 3 * q), (32, 12 * q, 6 * q)):
            add("scatter-16B-L%d-C%d-%s" % (L, C, n), _hop_case("scatter", dt, C, gl, ld=C + h), [_one(dt, L)] * 4, True)
        # narrow rows: the 16-byte multi-row kernels, 1, 2, 4 and 8 vectors per row
        for nv in (1, 2, 4, 8):
            C = nv * h
            gl = h if nv <= 2 else C // 2
            add("scatter-mr-nv%d-C%d-%s" % (nv, C, n), _hop_case("scatter", dt, C, gl, ld=C + (h if nv > 1 else 0)),
                [_mr(dt, nv)] * 4, True)
        add("bcast-rows-C%d-%s" % (6 * q - q // 2, n), _rows_case("bcast", dt, 6 * q - q // 2),
            [r"bcast_rows_kernel<%s>" % ("float,4" if dt == F32 else "double,2")])
        add("scatter-rows-C%d-%s" % (6 * q, n), _rows_case("scatter", dt, 6 * q, 3 * q),
            [r"scatter_rows_kernel<%s>" % ("float,4" if dt == F32 else "double,2")], True)
    # 16 peers (MAX_PEERS): all-gather and scatter; the last owner gets 1100 - 15 * 69 = 65 rows
    add("bcast-v2-L8-16peers-f32", _hop_case("bcast", F32, 48, n_peers=16), [_v2(F32, 8, 2)] * 2 + [_v2(F32, 8, 0)] * 2)
    add("scatter-v2-L8-16peers-f32", _hop_case("scatter", F32, 48, 24, n_sc=16),
        [_v2(F32, 8, 1)] * 2 + [_v2(F32, 8, 0)] * 2, True)
    add("bcast-rows-16peers-f32", _rows_case("bcast", F32, 44, n_peers=16), [r"bcast_rows_kernel<float,4>"])
    # the hub graph: a 20 000-entry row and column
    add("scatter-v2-L8-hub-f32", _hop_case("scatter", F32, 48, 24, N=24000, r0=5000, n_rows=15000),
        [_v2(F32, 8, 1)] * 2 + [_v2(F32, 8, 0)] * 2, True)
    add("grid-mr2-hub-f32", _hop_case("grid", F32, 16, 8, N=24000, r0=5000, n_rows=15000),
        [_mr2(F32, 3)] * 2 + [_mr2(F32, 0)] * 2, True)
    # tiny graphs
    add("bcast-v2-L8-tinyN1-f32", _hop_case("bcast", F32, 48, N=1, r0=0, n_rows=1, graph="tiny"),
        [_v2(F32, 8, 2)] * 2 + [_v2(F32, 8, 0)] * 2)
    add("scatter-v2-L8-tinyN3-f32", _hop_case("scatter", F32, 48, 24, N=3, r0=1, n_rows=2, graph="tiny"),
        [_v2(F32, 8, 1)] * 2 + [_v2(F32, 8, 0)] * 2, True)
    add("grid-mr2-tinyN7-f32", _hop_case("grid", F32, 16, 8, N=7, r0=2, n_rows=4, graph="tiny"),
        [_mr2(F32, 3)] * 2 + [_mr2(F32, 0)] * 2, True)
    # a symmetric S: both directions gather with the same operator
    add("bcast-v2-L16-sym-f32", _hop_case("bcast", F32, 100, graph="sym"), [_v2(F32, 16, 2)] * 2 + [_v2(F32, 16, 0)] * 2)
    return rows, scatter


PEER_CASES, SCATTER_CASES = _rows()


def _template_args(name):
    """('spmm_hop_v2_kernel', ['float', 'int', '8', ...]) of a normalised kernel name."""
    m = re.search(r"(\w+)<([^<>]*)>", name)
    return (m.group(1), m.group(2).split(",")) if m else (None, [])


def test_every_peer_epilogue_instantiation_has_a_case():
    """Every kernel of the library with a peer epilogue (MODE 1, 2 or 3) is matched by a row, and every scatter-carrying
    16-byte kernel (spmm_hop_kernel with VEC > 1, spmm_hop_multirow_kernel) by a row with the scatter on."""
    names = library_kernels()
    if names is None:
        pytest.skip("cuobjdump / cu++filt or the library not available")
    mode_at = {"spmm_hop_v2_kernel": 8, "spmm_hop_multirow_v2_kernel": 9}
    peer, scatter16, copies = [], [], []
    for n in names:
        k, args = _template_args(n)
        if k in mode_at and int(args[mode_at[k]]) in (1, 2, 3):
            peer.append(n)
        elif (k == "spmm_hop_kernel" and int(args[1]) > 1) or k == "spmm_hop_multirow_kernel":
            scatter16.append(n)
        elif k in ("bcast_rows_kernel", "scatter_rows_kernel"):
            copies.append(n)
    assert (len(peer), len(scatter16), len(copies)) == (26, 12, 4), (sorted(peer), sorted(scatter16), sorted(copies))
    rx = [k for _, _, ks in PEER_CASES for k in ks]
    missing = [n for n in peer + copies if not any(re.search(k, n) for k in rx)]
    assert not missing, "peer-epilogue kernels without a case: %s" % missing
    rx_sc = [k for cid, _, ks in PEER_CASES if cid in SCATTER_CASES for k in ks]
    missing = [n for n in scatter16 if not any(re.search(k, n) for k in rx_sc)]
    assert not missing, "scatter-carrying kernels without a row that scatters: %s" % missing


traced = child_traced("test_peer_epilogues", "PEER_CASES")


@pytest.mark.gpu
@pytest.mark.parametrize("cid,fn,kernels", PEER_CASES, ids=[c[0] for c in PEER_CASES])
def test_peer_epilogue(cid, fn, kernels, traced):
    check_case(cid, fn, kernels, traced[cid])


@pytest.mark.gpu
def test_peer_flag_fence_with_one_participant():
    """b200gf_peer_signal / b200gf_peer_wait with a single rank: signal then wait returns, and the step counter and this
    rank's flag both count 1, 2, 3."""
    import gnn_b200
    cabi = gnn_b200._cabi
    lib = cabi.load()
    stream = torch.cuda.current_stream().cuda_stream
    flags = torch.zeros(32, dtype=torch.int64, device="cuda")    # [16 flags][step counter ...]
    for step in (1, 2, 3):
        assert lib.b200gf_peer_signal(cabi.ptr_array([flags.data_ptr()]), 1, 0, ctypes.c_void_p(flags.data_ptr() + 128),
                                      stream) == 0
        assert lib.b200gf_peer_wait(ctypes.c_void_p(flags.data_ptr()), 1, ctypes.c_void_p(flags.data_ptr() + 128), stream) == 0
        torch.cuda.synchronize()
        assert int(flags[0]) == step and int(flags[16]) == step
        assert int(flags[1:16].abs().sum()) == 0 and int(flags[17:].abs().sum()) == 0
