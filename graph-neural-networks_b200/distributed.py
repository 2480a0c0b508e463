"""Multi-GPU LSIGF (one process per GPU, torch.distributed over NCCL / NVLink) — SURVEY.md §8e.

Three shardings of  y = sum_{e,k} (x S_e^k) h_{e,k} + b  (each with its exchange fused into the hop kernel when the real
CUDA ops run under NCCL, and with plain collectives otherwise — the variant the gloo tests exercise):

  mode="nodes"     1-D node partition.  Rank p owns rows [r_p, r_{p+1}) of every node-major matrix and the matching
                   rows of the gather operators (global column indices).  Each of the K-1 hops is followed by an
                   NCCL all-gather of the freshly computed rows (the halo of an Erdős–Rényi graph is ~all remote
                   nodes, so the "boundary rows" are the whole block); the tap contraction and the bias are
                   row-local.  This is the sharding BASELINE.json names.
  mode="features"  The graph is replicated and the B*G feature columns are split: a hop never mixes columns, so the
                   K-1 hops need NO communication and each rank's gathered slab (N x C/P) shrinks towards the L2.
                   Every shifted slice z_k is sent to the ranks that own its node rows with an asynchronous NCCL
                   all-to-all that overlaps the next hop; one row-local contraction over all E*K*G inputs ends the
                   call (output sharded by node rows).  The right choice whenever S fits on each GPU (SURVEY §8e
                   "column split"); a reduce-scatter variant covers G not divisible by the world size.

  mode="grid"      2-D process grid P = P_r x P_c: rank (r, c) shifts the rows of row group r for the columns of
                   column group c.  Each hop all-gathers its rows inside the column group (P_r ranks, N*C/P_c elements
                   instead of N*C) and delivers its slice to the contraction owner inside the row group — both from the
                   kernel's epilogue (b200gf_hop_grid).  The all-gather that bounds the node sharding at 8 GPUs and the
                   replicated index work that bounds the feature sharding are both cut by the grid factors.  The
                   backward exists in the collective form only.

The arithmetic goes through `ops` (the C-ABI building blocks b200gf_hop / b200gf_tap_contract on CUDA).  The
world_size-2 / -4 gloo tests inject an oracle-backed `ops` to exercise the partitioning / collective choreography on CPU;
the product default has no CPU path.
"""
import numpy as np
import torch
import torch.distributed as dist

from . import _cabi
from .graphML import padded_ld
from .gso import Plan, SparseGSO


def row_slice(csr, r0, r1):
    """rows [r0, r1) of a host CSR (rowptr, col, val); rows beyond the matrix are empty (zero padding)."""
    rowptr, col, val = csr
    n = len(rowptr) - 1
    rp = rowptr[np.minimum(np.arange(r0, r1 + 1), n)]
    lo, hi = int(rp[0]), int(rp[-1])
    return (rp - lo).astype(np.int64), col[lo:hi], val[lo:hi]


def transpose_csr(csr, N):
    import scipy.sparse as sp
    rowptr, col, val = csr
    m = sp.csr_matrix((val, col, rowptr), shape=(N, N)).T.tocsr()
    m.sort_indices()
    return m.indptr.astype(np.int64), m.indices.astype(np.int32), m.data


def resolve_fused(requested, ops_injected, backend, world):
    """Whether the hop kernels move their rows over NVLink themselves (no NCCL collective on the data path).
    `requested` None = default: on whenever the real CUDA ops run under NCCL with at most 16 ranks (the peer-pointer
    arrays of the kernels hold 16 entries); True / False = the caller's explicit choice."""
    if requested is None:
        return bool((not ops_injected) and backend == "nccl" and world <= 16)
    return bool(requested)


def default_grid(world):
    """(P_r, P_c) for the 2-D sharding: two row groups, the rest column groups (8 -> 2 x 4, 4 -> 2 x 2)."""
    if world >= 4 and world % 2 == 0:
        return 2, world // 2
    return world, 1


class CudaOps:
    """Building blocks on the GPU through the C ABI (include/b200gf.h)."""

    def __init__(self, device):
        self.device = torch.device(device)
        self.lib = _cabi.load()

    def make_plan_ops(self, fwd, bwd, n_rows, n_cols, dtype):
        return Plan.from_ops(fwd, bwd, n_rows, n_cols, dtype, self.device)

    def make_plan_full(self, gso):
        return gso.plan(self.device)

    def hop(self, plan, e, direction, src, dst, C):
        _cabi.check(self.lib.b200gf_hop(plan.handle, e, direction, src.data_ptr(), src.stride(0), dst.data_ptr(),
                                        dst.stride(0), C, _cabi.stream()))

    def hop_scatter(self, plan, e, direction, src, dst, C, peers, rows_per_peer, out_ld, out_col, gl, stride_b):
        _cabi.check(self.lib.b200gf_hop_scatter(plan.handle, e, direction, src.data_ptr(), src.stride(0), dst.data_ptr(),
                                                dst.stride(0), C, _cabi.ptr_array(peers), len(peers), rows_per_peer,
                                                out_ld, out_col, gl, stride_b, _cabi.stream()))

    def scatter_rows(self, src, n_rows, C, peers, rows_per_peer, out_ld, out_col, gl, stride_b):
        _cabi.check(self.lib.b200gf_scatter_rows(_cabi.DTYPE[src.dtype], src.data_ptr(), src.stride(0), n_rows, C,
                                                 _cabi.ptr_array(peers), len(peers), rows_per_peer, out_ld, out_col, gl,
                                                 stride_b, _cabi.stream()))

    def hop_bcast(self, plan, e, direction, src, C, peers, mc, row0, out_ld):
        _cabi.check(self.lib.b200gf_hop_bcast(plan.handle, e, direction, src.data_ptr(), src.stride(0), C,
                                              _cabi.ptr_array(peers), len(peers), mc or None, row0, out_ld, _cabi.stream()))

    def hop_grid(self, plan, e, direction, src, C, bc_peers, row0, bc_ld, sc_peers, rows_per_peer, out_ld, out_col, gl, stride_b):
        _cabi.check(self.lib.b200gf_hop_grid(plan.handle, e, direction, src.data_ptr(), src.stride(0), C,
                                             _cabi.ptr_array(bc_peers) if bc_peers else None, len(bc_peers), row0, bc_ld,
                                             _cabi.ptr_array(sc_peers), len(sc_peers), rows_per_peer, out_ld, out_col, gl,
                                             stride_b, _cabi.stream()))

    def bcast_rows(self, src, n_rows, C, peers, mc, row0, out_ld):
        _cabi.check(self.lib.b200gf_bcast_rows(_cabi.DTYPE[src.dtype], src.data_ptr(), src.stride(0), n_rows, C,
                                               _cabi.ptr_array(peers), len(peers), mc or None, row0, out_ld, _cabi.stream()))

    def pack_taps(self, h, transpose):
        F, E, K, G = h.shape
        T = 1 + E * (K - 1)
        W = torch.empty((T, F, G) if transpose else (T, G, F), dtype=h.dtype, device=h.device)
        _cabi.check(self.lib.b200gf_pack_taps(_cabi.DTYPE[h.dtype], h.contiguous().data_ptr(), W.data_ptr(), F, E, K, G,
                                              1 if transpose else 0, _cabi.stream()))
        return W

    def tap_contract(self, zs, W, bias, out, n_rows, B, P, Q, bias_per_node=0):
        T = len(zs)
        sb = self.lib.b200gf_tap_contract_scratch_bytes(T, P, Q)
        scratch = torch.empty(sb, dtype=torch.uint8, device=out.device)
        _cabi.check(self.lib.b200gf_tap_contract(
            _cabi.DTYPE[out.dtype], n_rows, B, P, Q, T, _cabi.ptr_array([z.data_ptr() for z in zs]),
            _cabi.i64_array([z.stride(0) for z in zs]), W.data_ptr(), None if bias is None else bias.data_ptr(),
            bias_per_node, out.data_ptr(), out.stride(0), 0, scratch.data_ptr(), sb, _cabi.stream()))

    def tap_grad(self, A, vs, n_rows, B, P, Q):
        """dW[t][p][q] = sum_{n < n_rows, b} A[n, b*P + p] * vs[t][n, b*Q + q]   (b200gf_tap_grad)."""
        T = len(vs)
        dW = torch.empty((T, P, Q), dtype=A.dtype, device=A.device)
        sb = self.lib.b200gf_tap_grad_scratch_bytes(_cabi.DTYPE[A.dtype], n_rows, B, P, Q, T)
        scratch = torch.empty(max(int(sb), 1), dtype=torch.uint8, device=A.device)
        _cabi.check(self.lib.b200gf_tap_grad(
            _cabi.DTYPE[A.dtype], n_rows, B, P, Q, T, A.data_ptr(), A.stride(0), _cabi.ptr_array([v.data_ptr() for v in vs]),
            _cabi.i64_array([v.stride(0) for v in vs]), dW.data_ptr(), scratch.data_ptr(), sb, _cabi.stream()))
        return dW


class _RawMat:
    """A [rows, ld] device matrix known only by address (memory mapped from a symmetric allocation)."""

    def __init__(self, ptr, ld):
        self._ptr, self._ld = int(ptr), int(ld)

    def data_ptr(self):
        return self._ptr

    def stride(self, i):
        return self._ld if i == 0 else 1


class SymmetricArena:
    """`nbytes` of device memory on every rank that all ranks of the node can address, plus the peer-flag fence state.

    Plumbing only: the allocation and the address exchange go through torch.distributed's symmetric memory
    (torch.distributed._symmetric_memory: cuMem allocations, peer mappings and — when the NVSwitch supports it — a
    multicast alias), falling back to this library's CUDA-IPC calls (b200gf_symm_*: no multicast).  Everything that
    touches the memory afterwards is this library's kernels: hop_bcast / bcast_rows stores, peer_signal / peer_wait.
    Layout: [payload, 256-byte aligned][16 x u64 arrival flags][u64 local step counter]."""

    def __init__(self, lib, nbytes, group, device, prefer="auto"):
        import ctypes
        self.lib, self.group, self.device = lib, group, torch.device(device)
        self.payload = (int(nbytes) + 255) // 256 * 256
        self.flags_off = self.payload
        self.step_off = self.flags_off + 128
        total = self.payload + 256
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.peers, self.mc, self.kind = None, 0, None
        self._opened, self._own, self._keep = [], 0, None
        if prefer in ("auto", "torch"):
            try:
                import torch.distributed._symmetric_memory as symm
                t = symm.empty(total, dtype=torch.uint8, device=self.device)
                t.zero_()
                hdl = symm.rendezvous(t, group if group is not None else dist.group.WORLD)
                self.peers = [int(p) for p in hdl.buffer_ptrs]
                self.mc = int(hdl.multicast_ptr or 0)
                self._keep = (t, hdl)
                self.kind = "torch-symm" + ("+multicast" if self.mc else "")
            except Exception as exc:                       # older driver / no fabric support: plain CUDA IPC below
                if prefer == "torch":
                    raise
                self._why_not_torch = repr(exc)[:200]
                self.peers = None
            # the choice must be the same on every rank (the IPC path below is collective): all or nothing
            ok = torch.tensor([0 if self.peers is None else 1], device=self.device)
            dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=group)
            if int(ok.item()) == 0 and self.peers is not None:
                self.peers, self.mc, self._keep, self.kind = None, 0, None, None
                self._why_not_torch = "torch symmetric memory failed on another rank"
        if self.peers is None:
            mine = ctypes.c_void_p()
            _cabi.check(lib.b200gf_symm_alloc(ctypes.byref(mine), total))      # zero-filled
            self._own = mine.value
            handle = (ctypes.c_ubyte * 64)()
            _cabi.check(lib.b200gf_symm_export(ctypes.c_void_p(self._own), handle))
            t = torch.tensor(list(bytes(handle)), dtype=torch.uint8, device=self.device)
            allh = [torch.empty_like(t) for _ in range(self.world)]
            dist.all_gather(allh, t, group=group)
            self.peers = []
            for p in range(self.world):
                if p == self.rank:
                    self.peers.append(self._own)
                    continue
                raw = (ctypes.c_ubyte * 64)(*allh[p].cpu().tolist())
                ptr = ctypes.c_void_p()
                _cabi.check(lib.b200gf_symm_import(raw, ctypes.byref(ptr)))
                self.peers.append(ptr.value)
                self._opened.append(ptr.value)
            self.kind = "cuda-ipc"
        self.mine = self.peers[self.rank]
        torch.cuda.synchronize(self.device)
        dist.barrier(group=group)                          # every rank's memory is zeroed before anyone signals into it

    def peer_ptrs(self, offset):
        return [p + offset for p in self.peers]

    def mc_ptr(self, offset):
        return self.mc + offset if self.mc else 0

    def local(self, offset, ld):
        return _RawMat(self.mine + offset, ld)

    def fence(self, stream):
        """signal + wait on the symmetric flag arrays: returns (on the stream) once every rank's earlier stores have landed."""
        import ctypes
        _cabi.check(self.lib.b200gf_peer_signal(_cabi.ptr_array([p + self.flags_off for p in self.peers]), self.world,
                                                self.rank, ctypes.c_void_p(self.mine + self.step_off), stream))
        _cabi.check(self.lib.b200gf_peer_wait(ctypes.c_void_p(self.mine + self.flags_off), self.world,
                                              ctypes.c_void_p(self.mine + self.step_off), stream))

    def close(self):
        """Collective.  Nobody frees memory a peer may still have mapped: synchronise, barrier, unmap, barrier, free."""
        import ctypes
        torch.cuda.synchronize(self.device)
        dist.barrier(group=self.group)
        for p in self._opened:
            self.lib.b200gf_symm_close(ctypes.c_void_p(p))
        self._opened = []
        dist.barrier(group=self.group)
        if self._own:
            self.lib.b200gf_symm_free(ctypes.c_void_p(self._own))
            self._own = 0
        self._keep = None


class SymmetricOperand:
    """Double-buffered row-local contraction operand [2][R, row_elems] that every peer can write over NVLink
    (b200gf_symm_* : cudaMalloc + CUDA IPC).  Double buffering removes the write-after-read hazard between a fast
    rank's next scatter and a slow rank's current contraction; one tiny all-reduce per call orders the rest."""

    def __init__(self, lib, R, row_elems, dtype, group, device):
        import ctypes
        self.lib, self.R, self.row_elems, self.group = lib, R, row_elems, group
        es = 4 if dtype == torch.float32 else 8
        self.buf_bytes = (R * row_elems * es + 255) // 256 * 256
        # layout: [operand 0][operand 1][16 x u64 arrival flags][u64 local step counter]   (alloc zero-fills)
        self.flags_off = 2 * self.buf_bytes
        self.step_off = self.flags_off + 128
        mine = ctypes.c_void_p()
        _cabi.check(lib.b200gf_symm_alloc(ctypes.byref(mine), 2 * self.buf_bytes + 256))
        self.mine = mine.value
        handle = (ctypes.c_ubyte * 64)()
        _cabi.check(lib.b200gf_symm_export(ctypes.c_void_p(self.mine), handle))
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        t = torch.tensor(list(bytes(handle)), dtype=torch.uint8, device=device)
        allh = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(allh, t, group=group)
        self.peers, self._opened = [], []
        for p in range(world):
            if p == rank:
                self.peers.append(self.mine)
                continue
            raw = (ctypes.c_ubyte * 64)(*allh[p].cpu().tolist())
            ptr = ctypes.c_void_p()
            _cabi.check(lib.b200gf_symm_import(raw, ctypes.byref(ptr)))
            self.peers.append(ptr.value)
            self._opened.append(ptr.value)
        self.step = 0

    def peer_ptrs(self, buf):
        return [p + buf * self.buf_bytes for p in self.peers]

    def local(self, buf):
        return _RawMat(self.mine + buf * self.buf_bytes, self.row_elems)

    def fence(self, rank, stream):
        """signal + wait on the symmetric flag arrays: returns (on the stream) once every rank's scatters have landed."""
        import ctypes
        n = len(self.peers)
        _cabi.check(self.lib.b200gf_peer_signal(_cabi.ptr_array([p + self.flags_off for p in self.peers]), n, rank,
                                                ctypes.c_void_p(self.mine + self.step_off), stream))
        _cabi.check(self.lib.b200gf_peer_wait(ctypes.c_void_p(self.mine + self.flags_off), n,
                                              ctypes.c_void_p(self.mine + self.step_off), stream))

    def close(self):
        """Collective: a peer may still have this buffer mapped, so synchronise + barrier before unmapping and again
        before cudaFree (freeing IPC-exported memory that is still open elsewhere is undefined behaviour)."""
        import ctypes
        torch.cuda.synchronize()
        dist.barrier(group=self.group)
        for p in self._opened:
            self.lib.b200gf_symm_close(ctypes.c_void_p(p))
        self._opened = []
        dist.barrier(group=self.group)
        if self.mine:
            self.lib.b200gf_symm_free(ctypes.c_void_p(self.mine))
            self.mine = 0


class PartitionedLSIGF:
    """LSIGF forward sharded over the ranks of `group` (see module docstring).

    nodes mode:     forward(h, x_rows, b)  x_rows  node-major [rows_per_rank, B*G]  -> y_rows [rows_per_rank, B*F]
    features mode:  forward(h, x_cols, b)  x_cols  node-major [N, B*(G/P)]          -> y_rows [rows_per_rank, B*F]
    In both, row block p covers global nodes [p*rows_per_rank, (p+1)*rows_per_rank) (the last block is zero-padded).
    """

    def __init__(self, gso, mode="nodes", group=None, device=None, ops=None, fused=None, fence="flags", symm_backend="auto",
                 multicast=False, grid=None):
        assert mode in ("nodes", "features", "grid") and fence in ("flags", "nccl")
        self.mode = mode
        self.symm_backend = symm_backend   # "auto": torch symmetric memory, else CUDA IPC; "ipc"; "torch"
        # all-gather epilogue: one multimem.st through the NVSwitch multicast address instead of P peer stores.  Off by
        # default: a multicast store also returns to the issuing GPU through its NVLink ingress, so every GPU receives
        # N*C*s per hop instead of (P-1)/P of it, and the all-gather is ingress-bound
        self.multicast = bool(multicast)
        self.fence = fence          # "flags": peer flags in symmetric memory (no NCCL at all); "nccl": 4-byte all-reduce
        # fused = hop kernels scatter their rows over NVLink themselves (no NCCL collective on the data path);
        # default: on whenever the real CUDA ops run under NCCL with <= 16 ranks
        self._fused_req = fused
        self._symm = None
        self._symm_by_width = {}
        self._arenas = {}
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.N, self.E, self.dtype = gso.N, gso.E, gso.dtype
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.ops = ops if ops is not None else CudaOps(self.device)
        P = self.world
        self.rows_per_rank = (self.N + P - 1) // P
        self.n_pad = self.rows_per_rank * P
        self.r0 = self.rank * self.rows_per_rank
        self.r1 = self.r0 + self.rows_per_rank
        if mode == "grid":
            self.Pr, self.Pc = grid if grid is not None else default_grid(P)
            assert self.Pr * self.Pc == P and self.Pr >= 1 and self.Pc >= 1, "grid must factor the world size"
            self.rg, self.cg = self.rank // self.Pc, self.rank % self.Pc          # my row group, my column group
            self.rows_per_group = self.rows_per_rank * self.Pc                    # rows my row group shifts per hop
            g0, g1 = self.rg * self.rows_per_group, (self.rg + 1) * self.rows_per_group
            fwd = [row_slice(transpose_csr(gso.csr[e], self.N), g0, g1) for e in range(self.E)]
            self.local_nnz = int(sum(f[0][-1] for f in fwd))
            self.plan = self.ops.make_plan_ops(fwd, None, self.rows_per_group, self.n_pad, self.dtype)
            self._grid_step = 0
            self._grid_gso = gso                                                  # backward: rows of S_e, plan built on first use
        elif mode == "nodes":
            fwd, bwd = [], []
            for e in range(self.E):
                st = transpose_csr(gso.csr[e], self.N)
                fwd.append(row_slice(st, self.r0, self.r1))
                bwd.append(row_slice(gso.csr[e], self.r0, self.r1))
            self.local_nnz = int(sum(f[0][-1] for f in fwd))
            self.plan = self.ops.make_plan_ops(fwd, bwd, self.rows_per_rank, self.n_pad, self.dtype)
        else:
            self.local_nnz = gso.nnz()
            self.plan = self.ops.make_plan_full(gso)
        self._bufs = {}
        self.fused = resolve_fused(self._fused_req, ops is not None, dist.get_backend(group), self.world)
        self._grid_groups_cache = None
        self._grid_bwd_plan = None

    def close(self):
        """Collective: release the symmetric memory of this object (arenas of the node sharding, operands of the feature
        sharding).  Every rank must call it; nothing may be in flight on other ranks' streams (it synchronises + barriers)."""
        for a in list(self._arenas.values()):
            a.close()
        self._arenas = {}
        for sy in list(self._symm_by_width.values()):
            sy.close()
        self._symm_by_width = {}
        self._symm = None
        self._graph_keepalive = None

    # -- helpers -----------------------------------------------------------------------------------
    def feature_slice(self, G):
        """[g0, g1) of the in-features this rank owns in features mode."""
        per = (G + self.world - 1) // self.world
        g0 = min(G, self.rank * per)
        return g0, min(G, g0 + per)

    def _buffers(self, key, shape):
        b = self._bufs.get(key)
        if b is None or tuple(b.shape) != tuple(shape):
            b = torch.zeros(shape, dtype=self.dtype, device=self.device)
            self._bufs[key] = b
        return b

    # -- forward -----------------------------------------------------------------------------------
    def forward(self, h, x_local, b=None, B=1):
        """B (batch size) is only read in features mode, where it cannot be inferred from an empty column slice."""
        if self.mode == "grid":
            if self.fused and self._grid_fused_ok(h.shape[3], B):
                return self._forward_grid(h, x_local, b, B)
            return self._forward_grid_collective(h, x_local, b, B)
        if self.mode == "nodes":
            if self.fused and self._nodes_fused_ok(x_local.shape[1]):
                return self._forward_nodes_fused(h, x_local, b)
            return self._forward_nodes(h, x_local, b)
        return self._forward_features(h, x_local, b, B)

    def _forward_nodes(self, h, x_rows, b):
        F, E, K, G = h.shape
        C = x_rows.shape[1]
        B = C // G
        assert E == self.E and C == B * G and x_rows.shape[0] == self.rows_per_rank
        ld = padded_ld(C, self.dtype)
        R = self.rows_per_rank
        W = self.ops.pack_taps(h, False)
        # full-height sources for every hop that has a successor; the last hop of each e only needs local rows
        full0 = self._buffers(("z0", C), (self.n_pad, ld))
        full0[self.r0:self.r1, :C].copy_(x_rows)
        dist.all_gather_into_tensor(full0.view(-1), full0[self.r0:self.r1].reshape(-1), group=self.group)
        zs = [full0[self.r0:self.r1]]
        for e in range(E):
            src = full0
            for k in range(1, K):
                last = k == K - 1
                if last:
                    dst_rows = self._buffers(("zl", e, C), (R, ld))
                    self.ops.hop(self.plan, e, _cabi.HOP_FWD, src, dst_rows, C)
                else:
                    full = self._buffers(("z", e, k, C), (self.n_pad, ld))
                    dst_rows = full[self.r0:self.r1]
                    self.ops.hop(self.plan, e, _cabi.HOP_FWD, src, dst_rows, C)
                    dist.all_gather_into_tensor(full.view(-1), dst_rows.reshape(-1), group=self.group)
                    src = full
                zs.append(dst_rows)
        y = torch.empty((R, padded_ld(B * F, self.dtype)), dtype=self.dtype, device=self.device)
        bias = None
        if b is not None:
            assert b.shape[1] == 1, "per-node bias is not supported by the partitioned path"
            bias = b.contiguous()
        self.ops.tap_contract(zs, W, bias, y, R, B, G, F)
        return y[:, :B * F]

    # -- node sharding with the all-gather fused into the hop kernel ------------------------------------
    def _nodes_fused_ok(self, C):
        q = 8 if self.dtype == torch.float32 else 4
        return C * (4 if self.dtype == torch.float32 else 8) > 128 and padded_ld(C, self.dtype) % q == 0

    def _arena(self, key, n_bufs, ld):
        """Symmetric arena of n_bufs full-height node-major matrices [n_pad, ld] (cached per shape)."""
        a = self._arenas.get(key)
        if a is None:
            es = 4 if self.dtype == torch.float32 else 8
            buf = (self.n_pad * ld * es + 255) // 256 * 256
            a = SymmetricArena(self.ops.lib, n_bufs * buf, self.group, self.device, prefer=self.symm_backend)
            a.buf_bytes = buf
            if not self.multicast:
                a.mc = 0
                a.kind = a.kind.replace("+multicast", " (multicast available, peer stores used)")
            self._arenas[key] = a
        return a

    def _chain_nodes_fused(self, direction, rows, E, K, key):
        """[z_0 rows, z_{e,k} rows ...] (T node-major row blocks of this rank) for the shift chains of `rows`
        ([rows_per_rank, C]) with the forward (z S_e) or backward (S_e z) operator.  Every hop that has a successor runs
        b200gf_hop_bcast: its rows land in the full-height matrix of every rank (NVLink peer stores or one NVSwitch
        multicast store per row) while the kernel is still gathering, a peer-flag fence separates the hops; the last hop
        of a chain stays local.  No NCCL call, no host synchronisation.

        Hazards across calls (same arena reused by the next step): a rank may store into a peer's buffer t only after it
        passed a fence that the peer signals after its last read of buffer t.  Buffer t >= 1 is written by hop t of the
        next call, which follows that call's z_0 fence; the peer signals that fence after everything it enqueued for
        this call.  Buffer 0 is written first thing in the next call, so its readers (hop 1 of every chain) must precede
        the last fence of this call: true for K >= 3 (fence after hop K-2 of the last chain), enforced for K == 2 by
        the trailing fence below."""
        C = rows.shape[1]
        ld = padded_ld(C, self.dtype)
        es = rows.element_size()
        T = 1 + E * (K - 1)
        R, r0 = self.rows_per_rank, self.r0
        ar = self._arena((key, ld, T), T, ld)
        st = _cabi.stream()
        local_rows = lambda t: ar.local(t * ar.buf_bytes + r0 * ld * es, ld)      # noqa: E731
        local_full = lambda t: ar.local(t * ar.buf_bytes, ld)                     # noqa: E731
        if K > 1:
            self.ops.bcast_rows(rows, R, C, ar.peer_ptrs(0), ar.mc_ptr(0), r0, ld)   # all-gather of the k = 0 block
            ar.fence(st)
        out = [rows]
        for e in range(E):
            src = local_full(0)
            for k in range(1, K):
                t = 1 + e * (K - 1) + (k - 1)
                if k < K - 1:
                    self.ops.hop_bcast(self.plan, e, direction, src, C, ar.peer_ptrs(t * ar.buf_bytes),
                                       ar.mc_ptr(t * ar.buf_bytes), r0, ld)
                    ar.fence(st)
                else:
                    self.ops.hop(self.plan, e, direction, src, local_rows(t), C)
                out.append(local_rows(t))
                src = local_full(t)
        if K == 2:
            # with a single hop per chain nothing above orders "every rank has read z_0" before a faster rank's next call
            # stores its new z_0 rows into this rank's buffer 0; for K >= 3 the fence after hop K-2 of the last chain does
            # (every reader of buffer 0 precedes it in stream order)
            ar.fence(st)
        return out

    def _forward_nodes_fused(self, h, x_rows, b):
        F, E, K, G = h.shape
        C = x_rows.shape[1]
        B = C // G
        assert E == self.E and C == B * G and x_rows.shape[0] == self.rows_per_rank
        R = self.rows_per_rank
        if x_rows.stride(1) != 1 or (x_rows.stride(0) * x_rows.element_size()) % 16 or x_rows.data_ptr() % 16:
            x_rows = x_rows.contiguous()
        zs = self._chain_nodes_fused(_cabi.HOP_FWD, x_rows, E, K, "fwd")
        W = self.ops.pack_taps(h, False)
        y = torch.empty((R, padded_ld(B * F, self.dtype)), dtype=self.dtype, device=self.device)
        bias = None
        if b is not None:
            assert b.shape[1] == 1, "per-node bias is not supported by the partitioned path"
            bias = b.contiguous()
        self.ops.tap_contract(zs, W, bias, y, R, B, G, F)
        return y[:, :B * F]

    def _backward_nodes_fused(self, h, x_rows, dy_rows, want_db):
        F, E, K, G = h.shape
        R = self.rows_per_rank
        C = x_rows.shape[1]
        B = C // G
        CF = B * F
        if dy_rows.stride(1) != 1 or (dy_rows.stride(0) * dy_rows.element_size()) % 16 or dy_rows.data_ptr() % 16:
            dy_rows = dy_rows.contiguous()
        vs = self._chain_nodes_fused(_cabi.HOP_BWD, dy_rows, E, K, "bwd")     # V_{e,k} = S_e^k dY, my rows
        dW = self.ops.tap_grad(x_rows, vs, R, B, G, F)                          # [T, G, F]
        dist.all_reduce(dW, group=self.group)
        dh = _unpack_tap_grads(dW.transpose(1, 2), E, K)
        dx = torch.empty((R, padded_ld(C, self.dtype)), dtype=self.dtype, device=self.device)
        self.ops.tap_contract(vs, self.ops.pack_taps(h, True), None, dx, R, B, F, G)
        return dh, dx[:, :C], (self._bias_grad(dy_rows, B, F) if want_db else None)

    # -- 2-D process grid --------------------------------------------------------------------------------
    def grid_tile(self, x_nm, B, G):
        """This rank's input tile of a node-major x [N, B*G]: rows of its row group (zero-padded), features of its column
        group -> [rows_per_group, B*(G/P_c)] (column b*(G/P_c) + g)."""
        Gl = G // self.Pc
        xp = torch.cat((x_nm, torch.zeros(self.n_pad - x_nm.shape[0], B * G, dtype=x_nm.dtype, device=x_nm.device)))
        r0 = self.rg * self.rows_per_group
        return xp[r0:r0 + self.rows_per_group].view(self.rows_per_group, B, G)[:, :, self.cg * Gl:(self.cg + 1) * Gl] \
            .reshape(self.rows_per_group, B * Gl).contiguous()

    def _forward_grid(self, h, x_tile, b, B):
        """forward(h, x_tile, b, B): x_tile from grid_tile() -> y rows [rows_per_rank, B*F] of global nodes
        [rank*rows_per_rank, ...), like the other shardings.  Per hop: b200gf_hop_grid (all-gather inside the column group +
        scatter inside the row group, both in the kernel's epilogue), then a peer-flag fence; the contraction operand is
        double-buffered across steps exactly like the feature sharding's."""
        F, E, K, G = h.shape
        Pr, Pc = self.Pr, self.Pc
        assert E == self.E and G % Pc == 0
        Gl = G // Pc
        Cl = B * Gl
        q = 8 if self.dtype == torch.float32 else 4
        if Gl % q != 0 or Cl < 2 * q:                                  # forward() routes such shapes to the collective variant
            raise RuntimeError("b200gf: the fused grid kernels need G / P_c a multiple of %d columns (32-byte lanes) and rows "
                               "of at least 64 bytes; got G = %d, P_c = %d, B = %d" % (q, G, Pc, B))
        Rc, Rr = self.rows_per_rank, self.rows_per_group
        assert x_tile.shape[0] == Rr and x_tile.shape[1] == Cl
        T = 1 + E * (K - 1)
        ld = padded_ld(Cl, self.dtype)
        es = x_tile.element_size()
        row_elems = B * T * G
        key = ("grid", ld, T, row_elems)
        ar = self._arenas.get(key)
        if ar is None:
            buf = (self.n_pad * ld * es + 255) // 256 * 256
            opb = (Rc * row_elems * es + 255) // 256 * 256
            ar = SymmetricArena(self.ops.lib, T * buf + 2 * opb, self.group, self.device, prefer=self.symm_backend)
            ar.buf_bytes, ar.op_bytes, ar.op_off = buf, opb, T * buf
            ar.mc = 0                                      # the grid epilogue uses peer stores only
            ar.kind = ar.kind.replace("+multicast", " (multicast available, peer stores used)")
            self._arenas[key] = ar
        pbuf = self._grid_step & 1
        self._grid_step += 1
        col_group = [r * Pc + self.cg for r in range(Pr)]          # ranks holding the same feature columns
        row_group = [self.rg * Pc + c for c in range(Pc)]          # ranks sharing my rows: the contraction owners
        bc = lambda t: [ar.peers[p] + t * ar.buf_bytes for p in col_group]                     # noqa: E731
        sc = [ar.peers[p] + ar.op_off + pbuf * ar.op_bytes for p in row_group]
        row0 = self.rg * Rr
        g0 = self.cg * Gl
        st = _cabi.stream()
        if x_tile.stride(1) != 1 or (x_tile.stride(0) * es) % 32 or x_tile.data_ptr() % 32:
            xt = self._buffers(("gx", Cl), (Rr, ld))
            xt[:, :Cl].copy_(x_tile)
            x_tile = xt
        local_full = lambda t: ar.local(t * ar.buf_bytes, ld)                                  # noqa: E731
        if K > 1:
            self.ops.bcast_rows(x_tile, Rr, Cl, bc(0), 0, row0, ld)                            # z_0 for my column group
        self.ops.scatter_rows(x_tile, Rr, Cl, sc, Rc, row_elems, g0, Gl, T * G)                # k = 0 slices to their owners
        ar.fence(st)
        for e in range(E):
            src = local_full(0)
            for k in range(1, K):
                t = 1 + e * (K - 1) + (k - 1)
                last = k == K - 1
                self.ops.hop_grid(self.plan, e, _cabi.HOP_FWD, src, Cl, [] if last else bc(t), row0, ld, sc, Rc, row_elems,
                                  t * G + g0, Gl, T * G)
                ar.fence(st)
                src = local_full(t)
        W = self.ops.pack_taps(h, False).reshape(1, T * G, F)
        y = torch.empty((Rc, padded_ld(B * F, self.dtype)), dtype=self.dtype, device=self.device)
        bias = None
        if b is not None:
            assert b.shape[1] == 1, "per-node bias is not supported by the partitioned path"
            bias = b.contiguous()
        self.ops.tap_contract([ar.local(ar.op_off + pbuf * ar.op_bytes, row_elems)], W, bias, y, Rc, B, T * G, F)
        return y[:, :B * F]

    # -- 2-D process grid, collective variant (and the backward) --------------------------------------------
    def _grid_fused_ok(self, G, B):
        q = 8 if self.dtype == torch.float32 else 4
        return G % self.Pc == 0 and (G // self.Pc) % q == 0 and B * (G // self.Pc) >= 2 * q

    def _grid_groups(self):
        """(row group, column group) process groups of this rank; None for a group of one.  Collective on first use: every
        rank of `self.group` creates every sub-group, in the same order (torch.distributed's rule for new_group)."""
        if self._grid_groups_cache is None:
            base = dist.get_process_group_ranks(self.group) if self.group is not None else list(range(self.world))
            Pr, Pc = self.Pr, self.Pc
            rows = [dist.new_group([base[r * Pc + c] for c in range(Pc)]) if Pc > 1 else None for r in range(Pr)]
            cols = [dist.new_group([base[r * Pc + c] for r in range(Pr)]) if Pr > 1 else None for c in range(Pc)]
            self._grid_groups_cache = (rows[self.rg], cols[self.cg])
        return self._grid_groups_cache

    def _grid_gather_rows(self, full, colg):
        """all-gather of the row-group blocks of a full-height matrix inside the column group (in place)."""
        if colg is not None:
            g0 = self.rg * self.rows_per_group
            dist.all_gather_into_tensor(full.view(-1), full[g0:g0 + self.rows_per_group].reshape(-1), group=colg)

    def _grid_operand(self, E, K, G, x_tile, B):
        """The row-local contraction operand [rows_per_rank, B*T*G] (column b*T*G + t*G + g) of this rank: K-1 hops per
        edge feature on the rank's tile (rows of its row group x features of its column group), every hop output
        all-gathered inside the column group, then one all-to-all inside the row group hands every rank the slices of its
        own rows.  Same data flow as the fused kernel's two epilogues (_forward_grid), with collectives."""
        Pr, Pc = self.Pr, self.Pc
        assert G % Pc == 0, "the grid sharding splits the G input features evenly over the column groups"
        Gl = G // Pc
        Cl = B * Gl
        Rc, Rr = self.rows_per_rank, self.rows_per_group
        assert x_tile.shape[0] == Rr and x_tile.shape[1] == Cl
        T = 1 + E * (K - 1)
        rowg, colg = self._grid_groups()
        ld = padded_ld(Cl, self.dtype)
        g0 = self.rg * Rr
        full0 = self._buffers(("gz0", Cl), (self.n_pad, ld))
        full0[g0:g0 + Rr, :Cl].copy_(x_tile)
        if K > 1:
            self._grid_gather_rows(full0, colg)
        tiles = [full0[g0:g0 + Rr]]
        for e in range(E):
            src = full0
            for k in range(1, K):
                if k == K - 1:
                    dst = self._buffers(("gzl", e, Cl), (Rr, ld))
                    self.ops.hop(self.plan, e, _cabi.HOP_FWD, src, dst, Cl)
                else:
                    full = self._buffers(("gz", e, k, Cl), (self.n_pad, ld))
                    dst = full[g0:g0 + Rr]
                    self.ops.hop(self.plan, e, _cabi.HOP_FWD, src, dst, Cl)
                    self._grid_gather_rows(full, colg)
                    src = full
                tiles.append(dst)
        # block c of `send` = rows of rank (rg, c) inside my row group, my feature slab, every term t
        send = torch.stack([t_[:, :Cl].reshape(Pc, Rc, Cl) for t_ in tiles], dim=1).contiguous()        # [Pc, T, Rc, Cl]
        if rowg is not None:
            recv = torch.empty_like(send)
            all_to_all_blocks(recv, send, rowg)                 # recv[c] = my rows as computed by rank (rg, c): slab c
        else:
            recv = send
        return recv.reshape(Pc, T, Rc, B, Gl).permute(2, 3, 1, 0, 4).reshape(Rc, B * T * G)

    def _forward_grid_collective(self, h, x_tile, b, B):
        F, E, K, G = h.shape
        assert E == self.E
        T = 1 + E * (K - 1)
        Rc = self.rows_per_rank
        zrow = self._grid_operand(E, K, G, x_tile, B)
        W = self.ops.pack_taps(h, False).reshape(1, T * G, F)
        y = torch.empty((Rc, padded_ld(B * F, self.dtype)), dtype=self.dtype, device=self.device)
        bias = None
        if b is not None:
            assert b.shape[1] == 1, "per-node bias is not supported by the partitioned path"
            bias = b.contiguous()
        self.ops.tap_contract([zrow], W, bias, y, Rc, B, T * G, F)
        return y[:, :B * F]

    def _backward_grid_collective(self, h, x_tile, dy_rows, B, want_db):
        """Gradients for the grid sharding (collectives; the fused forward has no fused backward yet).  dy_rows
        [rows_per_rank, B*F] of this rank's output rows -> (dh, dx_tile laid out like x_tile, db).
        dh: the operand Z of the forward is row-local again (recomputed by the same exchange), dW_t = dY^T Z_t over my rows,
        all-reduced.  dx: U = dY [H_0^T .. H_{T-1}^T] is row-local; one all-to-all inside the row group turns it into
        tiles (rows of my row group x my feature slab), then Horner with the rows of S_e, every intermediate all-gathered
        inside the column group."""
        F, E, K, G = h.shape
        assert E == self.E
        Pr, Pc = self.Pr, self.Pc
        Gl = G // Pc
        Cl = B * Gl
        CF = B * F
        Rc, Rr = self.rows_per_rank, self.rows_per_group
        T = 1 + E * (K - 1)
        assert dy_rows.shape[1] == CF
        rowg, colg = self._grid_groups()
        dy_rows = dy_rows.contiguous()
        # ---- dh
        zrow = self._grid_operand(E, K, G, x_tile, B).view(Rc, B, T, G)
        zs = [zrow[:, :, t, :].reshape(Rc, B * G) for t in range(T)]
        dW = self.ops.tap_grad(dy_rows, zs, Rc, B, F, G)                           # [T, F, G] = dY^T Z_t over my rows
        dist.all_reduce(dW, group=self.group)
        dh = _unpack_tap_grads(dW, E, K)
        # ---- dx
        Wall = self.ops.pack_taps(h, True).permute(1, 0, 2).reshape(1, F, T * G).contiguous()
        U = torch.empty((Rc, padded_ld(B * T * G, self.dtype)), dtype=self.dtype, device=self.device)
        self.ops.tap_contract([dy_rows], Wall, None, U, Rc, B, F, T * G)
        send = U[:, :B * T * G].reshape(Rc, B, T, Pc, Gl).permute(3, 2, 0, 1, 4).contiguous()        # [Pc, T, Rc, B, Gl]
        if rowg is not None:
            recv = torch.empty_like(send)
            all_to_all_blocks(recv, send, rowg)                 # recv[c] = rows of rank (rg, c), my feature slab
        else:
            recv = send
        Ut = recv.permute(1, 0, 2, 3, 4).reshape(T, Rr, Cl)                        # tiles: rows of my row group
        dx = Ut[0].clone()                                                          # k = 0 term (shared by every e)
        if K > 1:
            if self._grid_bwd_plan is None:
                g0, g1 = self.rg * Rr, (self.rg + 1) * Rr
                rows = [row_slice(self._grid_gso.csr[e], g0, g1) for e in range(E)]
                self._grid_bwd_plan = self.ops.make_plan_ops(rows, None, Rr, self.n_pad, self.dtype)    # S_e w: gather with rows of S_e
            ld = padded_ld(Cl, self.dtype)
            g0 = self.rg * Rr
            for e in range(E):
                w = Ut[1 + e * (K - 1) + (K - 2)]                                   # W_{e,K-1} = U_{e,K-1}
                for k in range(K - 2, -1, -1):                                      # W_{e,k} = U_{e,k} + S_e W_{e,k+1}
                    full = self._buffers(("gw", k & 1, Cl), (self.n_pad, ld))
                    full[g0:g0 + Rr, :Cl].copy_(w)
                    self._grid_gather_rows(full, colg)
                    out = self._buffers(("go", k & 1, Cl), (Rr, ld))
                    self.ops.hop(self._grid_bwd_plan, e, _cabi.HOP_FWD, full, out, Cl)
                    if k > 0:
                        w = out[:, :Cl] + Ut[1 + e * (K - 1) + (k - 1)]
                    else:
                        dx += out[:, :Cl]
        return dh, dx, (self._bias_grad(dy_rows, B, F) if want_db else None)

    def _forward_features(self, h, x_cols, b, B):
        """Column-sharded hops (no communication inside a hop) + an all-to-all of every shifted slice to the rank that
        owns the node rows, overlapped with the following hops; then ONE row-local contraction over all E*K*G inputs.
        Bytes on NVLink per rank: T * N * B*(G/P) * s * (P-1)/P, all but the last slice hidden behind compute."""
        F, E, K, G = h.shape
        P = self.world
        if G % P != 0:
            return self._forward_features_rs(h, x_cols, b, B)
        vec = 4 if self.dtype == torch.float32 else 2
        if self.fused and (G // P) % vec == 0 and G % vec == 0:
            return self._forward_features_fused(h, x_cols, b, B)
        Gl = G // P
        Cl = B * Gl
        R = self.rows_per_rank
        T = 1 + E * (K - 1)
        assert x_cols.shape[0] == self.N and x_cols.shape[1] == Cl
        ld = padded_ld(Cl, self.dtype)
        z0 = self._buffers(("fz0", Cl), (self.n_pad, ld))
        z0[:self.N, :Cl].copy_(x_cols)
        recv = self._buffers(("frecv", T, Cl), (T, P, R, ld))   # recv[t, p]: my rows, column slice of rank p
        works = [all_to_all_rows(recv[0], z0, self.group)]
        for e in range(E):
            src = z0
            for k in range(1, K):
                t = 1 + e * (K - 1) + (k - 1)
                dst = self._buffers(("fz", e, k, Cl), (self.n_pad, ld))
                self.ops.hop(self.plan, e, _cabi.HOP_FWD, src, dst, Cl)
                works.append(all_to_all_rows(recv[t], dst, self.group))   # overlaps the next hop
                src = dst
        for w in works:
            if w is not None:
                w.wait()
        # [T, P, R, B, Gl] -> row-local operand [R, B, T*G] (column t*G + p*Gl + gl == t*G + g)
        zrow = recv[:, :, :, :Cl].reshape(T, P, R, B, Gl).permute(2, 3, 0, 1, 4).reshape(R, B * T * G)
        W = self.ops.pack_taps(h, False).reshape(1, T * G, F)
        y = torch.empty((R, padded_ld(B * F, self.dtype)), dtype=self.dtype, device=self.device)
        bias = None
        if b is not None:
            assert b.shape[1] == 1, "per-node bias is not supported by the partitioned path"
            bias = b.contiguous()
        self.ops.tap_contract([zrow], W, bias, y, R, B, T * G, F)
        return y[:, :B * F]

    def _forward_features_fused(self, h, x_cols, b, B):
        """features sharding with the exchange fused into the hop kernel (b200gf_hop_scatter): every computed row slice
        is stored over NVLink directly into the owning rank's contraction operand [R, B*T*G]; no NCCL collective moves
        data, one 4-byte all-reduce orders "all scatters done" before the row-local tensor-core contraction."""
        F, E, K, G = h.shape
        P = self.world
        Gl = G // P
        Cl = B * Gl
        R = self.rows_per_rank
        T = 1 + E * (K - 1)
        row_elems = B * T * G
        assert x_cols.shape[0] == self.N and x_cols.shape[1] == Cl
        sy = self._symm_by_width.get(row_elems)        # one operand per width: layers of different widths alternate
        if sy is None:
            sy = SymmetricOperand(self.ops.lib, R, row_elems, self.dtype, self.group, self.device)
            self._symm_by_width[row_elems] = sy
            if not hasattr(self, "_flag"):
                self._flag = torch.zeros(1, dtype=torch.float32, device=self.device)
        self._symm = sy
        buf = sy.step & 1
        sy.step += 1
        peers = sy.peer_ptrs(buf)
        g0 = self.rank * Gl
        ld = padded_ld(Cl, self.dtype)
        vecb = 16
        if x_cols.stride(1) == 1 and (x_cols.stride(0) * x_cols.element_size()) % vecb == 0 and x_cols.data_ptr() % vecb == 0:
            z0 = x_cols                                 # the caller's buffer is the k = 0 source: no staging copy
        else:
            z0 = self._buffers(("fz0", Cl), (self.n_pad, ld))
            z0[:self.N, :Cl].copy_(x_cols)
        self.ops.scatter_rows(z0, self.N, Cl, peers, R, row_elems, g0, Gl, T * G)
        for e in range(E):
            src = z0
            for k in range(1, K):
                t = 1 + e * (K - 1) + (k - 1)
                dst = self._buffers(("fz", e, k, Cl), (self.n_pad, ld))
                self.ops.hop_scatter(self.plan, e, _cabi.HOP_FWD, src, dst, Cl, peers, R, row_elems, t * G + g0, Gl, T * G)
                src = dst
        if self.fence == "flags":
            sy.fence(self.rank, _cabi.stream())             # every rank's scatters precede its flag store
        else:
            dist.all_reduce(self._flag, group=self.group)   # every rank's scatters precede its contribution
        W = self.ops.pack_taps(h, False).reshape(1, T * G, F)
        y = torch.empty((R, padded_ld(B * F, self.dtype)), dtype=self.dtype, device=self.device)
        bias = None
        if b is not None:
            assert b.shape[1] == 1, "per-node bias is not supported by the partitioned path"
            bias = b.contiguous()
        self.ops.tap_contract([sy.local(buf)], W, bias, y, R, B, T * G, F)
        return y[:, :B * F]

    # -- backward ----------------------------------------------------------------------------------
    def backward(self, h, x_local, dy_rows, B=1, want_db=True):
        """Gradients of `forward(h, x_local, b, B)` for the upstream gradient dy_rows [rows_per_rank, B*F] of this
        rank's output rows (zero in the padding rows of the last block).  Collective: every rank calls it.
        Returns (dh [F, E, K, G], dx_local laid out like x_local, db [F, 1] or None); dh and db are summed over the
        ranks (identical everywhere), dx_local stays sharded.  SURVEY.md §8 a-8 / §8e: the K-1 shifts of dY use the
        other operator (rows of S_e), exchanged like the forward's; dh and db end in one small all-reduce."""
        assert dy_rows.shape[0] == self.rows_per_rank
        if self.mode == "grid":
            return self._backward_grid_collective(h, x_local, dy_rows, B, want_db)
        if self.mode == "nodes":
            if self.fused and self._nodes_fused_ok(x_local.shape[1]) and self._nodes_fused_ok(dy_rows.shape[1]):
                return self._backward_nodes_fused(h, x_local, dy_rows, want_db)
            return self._backward_nodes(h, x_local, dy_rows, want_db)
        return self._backward_features(h, x_local, dy_rows, B, want_db)

    def apply(self, h, x_local, b=None, B=1):
        """Differentiable forward: autograd routes the gradient through `backward` (collective on every rank)."""
        return _PartitionedFunction.apply(self, B, h, x_local, b)

    def _bias_grad(self, dy_rows, B, F):
        db = dy_rows[:, :B * F].reshape(self.rows_per_rank, B, F).sum((0, 1))
        dist.all_reduce(db, group=self.group)
        return db.reshape(F, 1)

    def _backward_nodes(self, h, x_rows, dy_rows, want_db):
        F, E, K, G = h.shape
        R = self.rows_per_rank
        C = x_rows.shape[1]
        B = C // G
        CF = B * F
        assert E == self.E and C == B * G and x_rows.shape[0] == R and dy_rows.shape[1] == CF
        ldf = padded_ld(CF, self.dtype)
        full0 = self._buffers(("v0", CF), (self.n_pad, ldf))
        full0[self.r0:self.r1, :CF].copy_(dy_rows)
        dist.all_gather_into_tensor(full0.view(-1), full0[self.r0:self.r1].reshape(-1), group=self.group)
        vs = [full0[self.r0:self.r1]]                   # V_{e,k} = S_e^k dY, my rows
        for e in range(E):
            src = full0
            for k in range(1, K):
                if k == K - 1:
                    dst_rows = self._buffers(("vl", e, CF), (R, ldf))
                    self.ops.hop(self.plan, e, _cabi.HOP_BWD, src, dst_rows, CF)
                else:
                    full = self._buffers(("v", e, k, CF), (self.n_pad, ldf))
                    dst_rows = full[self.r0:self.r1]
                    self.ops.hop(self.plan, e, _cabi.HOP_BWD, src, dst_rows, CF)
                    dist.all_gather_into_tensor(full.view(-1), dst_rows.reshape(-1), group=self.group)
                    src = full
                vs.append(dst_rows)
        dW = self.ops.tap_grad(x_rows, vs, R, B, G, F)  # [T, G, F]: x_rows^T V_t over my rows
        dist.all_reduce(dW, group=self.group)
        dh = _unpack_tap_grads(dW.transpose(1, 2), E, K)
        dx = torch.empty((R, padded_ld(C, self.dtype)), dtype=self.dtype, device=self.device)
        self.ops.tap_contract(vs, self.ops.pack_taps(h, True), None, dx, R, B, F, G)   # sum_t V_t H_t^T, row-local
        return dh, dx[:, :C], (self._bias_grad(dy_rows, B, F) if want_db else None)

    def _backward_features(self, h, x_cols, dy_rows, B, want_db):
        """x is column-sharded, y / dY row-sharded.  dh needs Z_t^T dY with Z_t column-sharded: all-gather dY, recompute
        the shifted slices locally (K-1 hops per e, no communication), contract; the slices of dh are concatenated.
        dx needs sum_k S^k (dY H_k^T) for my columns: U = dY [H_0^T .. H_{T-1}^T] is row-local (one contraction), one
        all-to-all turns it from row- to column-sharded, then Horner with the other operator, again without
        communication.  NVLink bytes per rank: N*B*F*s (all-gather) + T*N*B*(G/P)*s*(P-1)/P (all-to-all)."""
        F, E, K, G = h.shape
        P = self.world
        R = self.rows_per_rank
        T = 1 + E * (K - 1)
        per = (G + P - 1) // P
        g0, g1 = self.feature_slice(G)
        Gl = g1 - g0
        Cl = B * Gl
        CF = B * F
        assert dy_rows.shape[1] == CF
        ldf = padded_ld(CF, self.dtype)
        ld = padded_ld(max(Cl, 1), self.dtype)
        dyf = self._buffers(("bdy", CF), (self.n_pad, ldf))
        dyf[self.r0:self.r1, :CF].copy_(dy_rows)
        dist.all_gather_into_tensor(dyf.view(-1), dyf[self.r0:self.r1].reshape(-1), group=self.group)
        # ---- dh: my in-feature columns
        dWl = torch.zeros((T, F, per), dtype=self.dtype, device=self.device)
        if Gl > 0:
            assert x_cols.shape[0] == self.N and x_cols.shape[1] == Cl
            z0 = self._buffers(("fz0", Cl), (self.n_pad, ld))
            z0[:self.N, :Cl].copy_(x_cols)
            zs = [z0]
            for e in range(E):
                src = z0
                for k in range(1, K):
                    dst = self._buffers(("fz", e, k, Cl), (self.n_pad, ld))
                    self.ops.hop(self.plan, e, _cabi.HOP_FWD, src, dst, Cl)
                    zs.append(dst)
                    src = dst
            dWl[:, :, :Gl] = self.ops.tap_grad(dyf, zs, self.N, B, F, Gl)       # [T, F, Gl] = dY^T Z_t
        parts = [torch.empty_like(dWl) for _ in range(P)]
        dist.all_gather(parts, dWl, group=self.group)
        dW = torch.cat([parts[p][:, :, :max(0, min(G, (p + 1) * per) - min(G, p * per))] for p in range(P)], dim=2)
        dh = _unpack_tap_grads(dW, E, K)
        # ---- dx: U[n, b, t, g] = sum_f dY[n, b, f] h_t[f, g] for my rows, every g
        Wt = self.ops.pack_taps(h, True)                                         # [T, F, G]
        Wall = Wt.permute(1, 0, 2).reshape(1, F, T * G).contiguous()
        U = torch.empty((R, padded_ld(B * T * G, self.dtype)), dtype=self.dtype, device=self.device)
        self.ops.tap_contract([dyf[self.r0:self.r1]], Wall, None, U, R, B, F, T * G)
        Uv = U[:, :B * T * G].reshape(R, B, T, G)
        if P * per != G:
            Uv = torch.cat((Uv, torch.zeros((R, B, T, P * per - G), dtype=self.dtype, device=self.device)), dim=3)
        send = Uv.reshape(R, B, T, P, per).permute(3, 0, 1, 2, 4).contiguous()   # [P, R, B, T, per]: block p -> rank p
        recv = torch.empty_like(send)                                             # block q: rows of rank q, my columns
        all_to_all_blocks(recv, send, self.group)
        dx = None
        if Gl > 0:
            Ub = self._buffers(("bU", T, Cl), (T, self.n_pad, ld))
            Ub[:, :, :Cl] = recv[..., :Gl].permute(3, 0, 1, 2, 4).reshape(T, self.n_pad, Cl)
            dxb = Ub[0]                                  # k = 0 term (shared by every e)
            tmp = [self._buffers(("bw", i, Cl), (self.n_pad, ld)) for i in range(2)]
            for e in range(E):
                if K == 1:
                    break
                w = Ub[1 + e * (K - 1) + (K - 2)]        # W_{e,K-1} = U_{e,K-1}
                for k in range(K - 2, -1, -1):           # W_{e,k} = U_{e,k} + S_e W_{e,k+1}
                    out = tmp[k & 1]
                    self.ops.hop(self.plan, e, _cabi.HOP_BWD, w, out, Cl)
                    if k > 0:
                        out[:self.N, :Cl] += Ub[1 + e * (K - 1) + (k - 1)][:self.N, :Cl]
                        w = out
                    else:
                        dxb[:self.N, :Cl] += out[:self.N, :Cl]
            dx = dxb[:self.N, :Cl]
        else:
            dx = torch.zeros((self.N, 0), dtype=self.dtype, device=self.device)
        return dh, dx, (self._bias_grad(dy_rows, B, F) if want_db else None)

    def graphed(self, h, x_static, b=None, B=1):
        """CUDA-graph version of the fused features path for a fixed input buffer: two graphs (one per operand buffer)
        are captured after two eager warm-up calls and replayed alternately, so a step costs one graph launch on the
        host.  Needs fence="flags" (everything in the step is then a kernel of this library or a device copy).
        Returns a callable; each call replays one step on the current contents of x_static / h / b.
        The two graphs own the two buffer parities: do not interleave eager forward() calls on this object with replays
        unless a collective on the stream (e.g. dist.barrier()) separates them on every rank — two consecutive steps on
        the same operand buffer have no fence between a fast rank's stores and a slow rank's contraction."""
        assert self.fused and self.fence == "flags"
        for _ in range(2):
            self.forward(h, x_static, b, B)
        torch.cuda.synchronize()
        if self.mode == "grid":
            assert self._grid_step % 2 == 0
        if self.mode == "features":
            if self._symm is None:
                raise RuntimeError("b200gf: graphed() needs the fused path (G/world a multiple of the 16-byte vector width)")
            assert self._symm.step % 2 == 0
        graphs, outs = [], []
        for _ in range(2):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                y = self.forward(h, x_static, b, B)
            graphs.append(g)
            outs.append(y)
        state = {"i": 0}

        def run():
            k = state["i"] & 1
            state["i"] += 1
            graphs[k].replay()
            return outs[k]

        self._graph_keepalive = (graphs, outs)
        return run

    def _forward_features_rs(self, h, x_cols, b, B):
        """Fallback when G is not divisible by the world size: partial contraction + reduce-scatter of [N, B*F]."""
        F, E, K, G = h.shape
        g0, g1 = self.feature_slice(G)
        Gl = g1 - g0
        R = self.rows_per_rank
        Cl = B * Gl
        ldf = padded_ld(B * F, self.dtype)
        part = self._buffers(("part", B, F), (self.n_pad, ldf))
        if Gl > 0:
            assert x_cols.shape[0] == self.N and x_cols.shape[1] == Cl
            ld = padded_ld(Cl, self.dtype)
            z0 = self._buffers(("fz0", Cl), (self.N, ld))
            z0[:, :Cl].copy_(x_cols)
            zs = [z0]
            for e in range(E):
                src = z0
                for k in range(1, K):
                    dst = self._buffers(("fz", e, k, Cl), (self.N, ld))
                    self.ops.hop(self.plan, e, _cabi.HOP_FWD, src, dst, Cl)
                    zs.append(dst)
                    src = dst
            W = self.ops.pack_taps(h[:, :, :, g0:g1].contiguous(), False)
            self.ops.tap_contract(zs, W, None, part[:self.N], self.N, B, Gl, F)
        else:
            part.zero_()
        y = torch.empty((R, ldf), dtype=self.dtype, device=self.device)
        reduce_scatter_rows(y, part, self.group)
        y = y[:, :B * F]
        if b is not None:
            assert b.shape[1] == 1
            y = y.view(R, B, F) + b.view(1, 1, F)
            y = y.reshape(R, B * F)
        return y


def all_to_all_rows(out, inp, group=None):
    """out[p] (my row block as held by rank p) <- rank p's inp row block `rank`.  inp is [P*R, ld], out [P, R, ld].
    NCCL: asynchronous all_to_all_single (returns the Work handle).  gloo (CPU tests): all-gather + slice."""
    if dist.get_backend(group) == "nccl":
        return dist.all_to_all_single(out.view(-1), inp.view(-1), group=group, async_op=True)
    P = dist.get_world_size(group)
    r = dist.get_rank(group)
    bufs = [torch.empty_like(inp) for _ in range(P)]
    dist.all_gather(bufs, inp.contiguous(), group=group)
    for p in range(P):
        out[p].copy_(bufs[p].view(P, out.shape[1], out.shape[2])[r])
    return None


def all_to_all_blocks(out, inp, group=None):
    """out[q] <- rank q's inp[rank]   (inp, out: [P, ...] contiguous, equal blocks).  gloo: all-gather + slice."""
    if dist.get_backend(group) == "nccl":
        dist.all_to_all_single(out.view(-1), inp.view(-1), group=group)
        return
    P = dist.get_world_size(group)
    r = dist.get_rank(group)
    bufs = [torch.empty_like(inp) for _ in range(P)]
    dist.all_gather(bufs, inp, group=group)
    for q in range(P):
        out[q].copy_(bufs[q][r])


def _unpack_tap_grads(dW, E, K):
    """dW [T, F, G] in the packed term order (t = 0: the k = 0 tap shared by every e; t = 1 + e*(K-1) + (k-1)) ->
    dh [F, E, K, G] (the k = 0 gradient is the same for every e: all of them multiply the unshifted x)."""
    T, F, G = dW.shape
    dh = torch.empty((F, E, K, G), dtype=dW.dtype, device=dW.device)
    dh[:, :, 0, :] = dW[0].unsqueeze(1)
    if K > 1:
        dh[:, :, 1:, :] = dW[1:].reshape(E, K - 1, F, G).permute(2, 0, 1, 3)
    return dh


class _PartitionedFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, part, B, h, x_local, b):
        ctx.part, ctx.B, ctx.has_bias = part, B, b is not None
        ctx.save_for_backward(h, x_local)
        return part.forward(h.detach(), x_local.detach(), None if b is None else b.detach(), B)

    @staticmethod
    def backward(ctx, dy):
        h, x_local = ctx.saved_tensors
        dh, dx, db = ctx.part.backward(h, x_local, dy.contiguous(), ctx.B, want_db=ctx.has_bias)
        return None, None, dh, dx, db


def reduce_scatter_rows(out_rows, full, group=None):
    """out_rows[rank block] = sum over ranks of full[rank block]; NCCL reduce-scatter (gloo: all-reduce + slice)."""
    backend = dist.get_backend(group)
    if backend == "nccl":
        dist.reduce_scatter_tensor(out_rows.view(-1), full.view(-1), op=dist.ReduceOp.SUM, group=group)
    else:
        tmp = full.clone()
        dist.all_reduce(tmp, op=dist.ReduceOp.SUM, group=group)
        r = dist.get_rank(group)
        R = out_rows.shape[0]
        out_rows.copy_(tmp[r * R:(r + 1) * R])
