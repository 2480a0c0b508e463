"""Sparse graph-shift-operator containers and the device plan.

The reference stores the GSO as a dense E x N x N tensor (`GraphFilter.addGSO`, alegnn/utils/graphML.py:2116-2123)
and cannot represent the graphs of BASELINE.json's configs (N = 1e5 .. 2e6).  `SparseGSO` is the sparse
description accepted everywhere a dense GSO is (SURVEY.md §8b "Extension over reference"); `Plan` is the opaque
device object of include/b200gf.h (CSR of S_e^T and S_e on the GPU).
"""
import ctypes
import weakref

import numpy as np
import torch

from . import _cabi

_NP2TORCH = {np.dtype("float32"): torch.float32, np.dtype("float64"): torch.float64}


class SparseGSO:
    """E sparse N x N shift operators in CSR (row i lists the non-zeros S_e[i, j]), held on the host.

    Quacks enough like the dense tensor for the reference's call sites: `.shape == (E, N, N)`, `.dtype`,
    `.to(device)`, `len(shape) == 3`.
    """

    def __init__(self, csr_list, N, dtype=None):
        self.csr = []
        for (rowptr, col, val) in csr_list:
            rowptr = np.ascontiguousarray(np.asarray(rowptr, dtype=np.int64))
            col = np.ascontiguousarray(np.asarray(col, dtype=np.int32))
            val = np.asarray(val)
            if dtype is not None:
                val = val.astype(np.dtype(str(dtype).replace("torch.", "")))
            val = np.ascontiguousarray(val)
            assert rowptr.shape == (N + 1,) and col.shape == val.shape and rowptr[-1] == col.shape[0]
            self.csr.append((rowptr, col, val))
        self.N = int(N)
        self.E = len(self.csr)
        self.shape = (self.E, self.N, self.N)
        self.dtype = _NP2TORCH[self.csr[0][2].dtype]
        self.device = torch.device("cpu")
        self.requires_grad = False
        self._plans = {}

    # -- constructors ------------------------------------------------------------------------------
    @classmethod
    def from_scipy(cls, mats, dtype=None):
        import scipy.sparse as sp
        mats = [sp.csr_matrix(m) for m in mats]
        for m in mats:
            m.sort_indices()
        N = mats[0].shape[0]
        return cls([(m.indptr, m.indices, m.data) for m in mats], N, dtype)

    @classmethod
    def from_dense(cls, S):
        """S: torch tensor or array [E, N, N]; pattern = (S != 0)."""
        S = torch.as_tensor(S)
        assert S.dim() == 3 and S.shape[1] == S.shape[2]
        csr = [dense_to_csr(S[e]) for e in range(S.shape[0])]
        return cls([(r.cpu().numpy(), c.cpu().numpy(), v.cpu().numpy()) for (r, c, v) in csr], S.shape[1])

    @classmethod
    def from_torch_sparse(cls, S, dtype=None):
        """torch sparse GSO: one [E, N, N] tensor (COO, or batched CSR) or a list of E [N, N] sparse tensors (COO / CSR /
        CSC, any device).  Duplicate COO entries are summed; columns come out sorted inside every row."""
        import scipy.sparse as sp
        mats2d = list(S) if isinstance(S, (list, tuple)) else [S[e] for e in range(S.shape[0])]
        mats = []
        for m in mats2d:
            assert m.dim() == 2 and m.shape[0] == m.shape[1]
            c = (m if m.layout == torch.sparse_coo else m.to_sparse_coo()).coalesce().cpu()
            idx = c.indices().numpy()
            mats.append(sp.csr_matrix((c.values().numpy(), (idx[0], idx[1])), shape=tuple(m.shape)))
        return cls.from_scipy(mats, dtype)

    # -- tensor-like surface -------------------------------------------------------------------------
    def to(self, *args, **kwargs):
        return self  # plans are created per device on demand

    def nnz(self):
        return int(sum(c[0][-1] for c in self.csr))

    def astype(self, torch_dtype):
        if torch_dtype == self.dtype:
            return self
        npd = np.float32 if torch_dtype == torch.float32 else np.float64
        return SparseGSO([(r, c, v.astype(npd)) for (r, c, v) in self.csr], self.N)

    def to_dense(self):
        out = np.zeros(self.shape, dtype=self.csr[0][2].dtype)
        for e, (r, c, v) in enumerate(self.csr):
            rows = np.repeat(np.arange(self.N), np.diff(r))
            out[e, rows, c] = v
        return torch.from_numpy(out)

    def plan(self, device):
        device = torch.device(device)
        key = (device.type, device.index if device.index is not None else torch.cuda.current_device())
        p = self._plans.get(key)
        if p is None:
            p = Plan.from_host_csr(self.csr, self.N, self.dtype, device)
            self._plans[key] = p
        return p


def dense_to_csr(S2d):
    """[N, N] tensor (any device) -> (rowptr int64, col int32, val) tensors on the same device, sorted by (row, col)."""
    N = S2d.shape[0]
    nz = (S2d != 0).nonzero(as_tuple=False)  # row-major order
    rows, cols = nz[:, 0], nz[:, 1]
    vals = S2d[rows, cols].contiguous()
    counts = torch.bincount(rows, minlength=N)
    rowptr = torch.zeros(N + 1, dtype=torch.int64, device=S2d.device)
    rowptr[1:] = torch.cumsum(counts, 0)
    return rowptr, cols.to(torch.int32).contiguous(), vals


class Plan:
    """Owns a `b200gf_plan*` (include/b200gf.h)."""

    def __init__(self, handle, N_rows, N_cols, E, dtype, device):
        self._h = handle
        self.n_rows, self.n_cols, self.E, self.dtype, self.device = N_rows, N_cols, E, dtype, device
        self._finalizer = weakref.finalize(self, _destroy, handle)

    @property
    def handle(self):
        return self._h

    @property
    def shape(self):  # what the LSIGF argument checks read off a dense GSO
        return (self.E, self.n_rows, self.n_cols)

    requires_grad = False

    @classmethod
    def from_host_csr(cls, csr_list, N, dtype, device):
        lib = _cabi.load()
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("b200gf: a plan needs a CUDA device (there is no CPU fallback)")
        idx = device.index if device.index is not None else torch.cuda.current_device()
        E = len(csr_list)
        keep = []
        rp, ci, va = [], [], []
        for (r, c, v) in csr_list:
            if isinstance(r, torch.Tensor):
                r = r.to(torch.int64).contiguous(); c = c.to(torch.int32).contiguous(); v = v.to(dtype).contiguous()
                keep += [r, c, v]
                rp.append(r.data_ptr()); ci.append(c.data_ptr()); va.append(v.data_ptr())
            else:
                r = np.ascontiguousarray(r, dtype=np.int64); c = np.ascontiguousarray(c, dtype=np.int32)
                v = np.ascontiguousarray(v, dtype=np.float32 if dtype == torch.float32 else np.float64)
                keep += [r, c, v]
                rp.append(r.ctypes.data); ci.append(c.ctypes.data); va.append(v.ctypes.data)
        out = ctypes.c_void_p()
        with torch.cuda.device(idx):
            torch.cuda.synchronize()
            rc = lib.b200gf_plan_create(ctypes.byref(out), idx, N, E, _cabi.ptr_array(rp), _cabi.ptr_array(ci),
                                        _cabi.ptr_array(va), _cabi.DTYPE[dtype])
        _cabi.check(rc)
        del keep
        return cls(out.value, N, N, E, dtype, torch.device("cuda", idx))

    @classmethod
    def from_ops(cls, fwd, bwd, n_rows, n_cols, dtype, device):
        """fwd / bwd: lists (per e) of host (rowptr, col, val) arrays for rows [r0, r1) of S_e^T / S_e."""
        lib = _cabi.load()
        device = torch.device(device)
        idx = device.index if device.index is not None else torch.cuda.current_device()
        npd = np.float32 if dtype == torch.float32 else np.float64
        keep = []

        def pack(ops):
            rp, ci, va = [], [], []
            for (r, c, v) in ops:
                r = np.ascontiguousarray(r, dtype=np.int64); c = np.ascontiguousarray(c, dtype=np.int32)
                v = np.ascontiguousarray(v, dtype=npd)
                keep.extend([r, c, v])
                rp.append(r.ctypes.data); ci.append(c.ctypes.data); va.append(v.ctypes.data)
            return _cabi.ptr_array(rp), _cabi.ptr_array(ci), _cabi.ptr_array(va)

        f = pack(fwd)
        b = pack(bwd) if bwd is not None else (None, None, None)
        out = ctypes.c_void_p()
        with torch.cuda.device(idx):
            rc = lib.b200gf_plan_create_ops(ctypes.byref(out), idx, n_rows, n_cols, len(fwd), f[0], f[1], f[2],
                                            b[0], b[1], b[2], _cabi.DTYPE[dtype])
        _cabi.check(rc)
        return cls(out.value, n_rows, n_cols, len(fwd), dtype, torch.device("cuda", idx))

    @classmethod
    def from_device_ops(cls, fwd, bwd, N, dtype, device):
        """fwd / bwd: lists (per e) of DEVICE tensors (rowptr int64 [N+1], col int32, val) — rows of S_e^T / of S_e.
        No host round trip (b200gf_plan_create_device)."""
        lib = _cabi.load()
        device = torch.device(device)
        idx = device.index if device.index is not None else torch.cuda.current_device()
        keep = []

        def pack(ops):
            rp, ci, va = [], [], []
            for (r, c, v) in ops:
                r = r.to(torch.int64).contiguous(); c = c.to(torch.int32).contiguous(); v = v.to(dtype).contiguous()
                keep.extend([r, c, v])
                rp.append(r.data_ptr()); ci.append(c.data_ptr()); va.append(v.data_ptr())
            return _cabi.ptr_array(rp), _cabi.ptr_array(ci), _cabi.ptr_array(va)

        f = pack(fwd)
        b = pack(bwd) if bwd is not None else (None, None, None)
        out = ctypes.c_void_p()
        with torch.cuda.device(idx):
            torch.cuda.current_stream().synchronize()          # the arrays were produced on the caller's stream
            rc = lib.b200gf_plan_create_device(ctypes.byref(out), idx, N, len(fwd), f[0], f[1], f[2], b[0], b[1], b[2],
                                               _cabi.DTYPE[dtype])
        _cabi.check(rc)
        del keep
        return cls(out.value, N, N, len(fwd), dtype, torch.device("cuda", idx))

    def info(self, what):
        return int(_cabi.load().b200gf_plan_info(self._h, what))

    @property
    def nnz(self):
        return self.info(5)

    @property
    def symmetric(self):
        return bool(self.info(6))


def _destroy(handle):
    try:
        _cabi.load().b200gf_plan_destroy(ctypes.c_void_p(handle))
    except Exception:
        pass


# ---------------------------------------------------------------------------------------------------
# plan cache for dense GSOs: LSIGF(h, S, x, b) is called with the same dense S tensor on every step
# (graphML.py:2137); converting it once per (storage, version, device) is the `addGSO` hook of SURVEY §3.3.
# ---------------------------------------------------------------------------------------------------
_PLAN_CACHE = {}
_PLAN_CACHE_MAX = 16


def _purge_dead_plans():
    """Drop cache entries whose GSO tensor has been collected, so their device CSR memory is released now rather than
    when FIFO eviction reaches them (a new dense S every step — edge-failure sampling — would otherwise pin 16 plans)."""
    dead = [k for k, hit in _PLAN_CACHE.items() if hit[0]() is None]
    for k in dead:
        del _PLAN_CACHE[k]


def _dense_key(S):
    return (S.data_ptr(), S._version, tuple(S.shape), tuple(S.stride()), S.dtype, str(S.device))


def plan_for(S, device=None):
    """Returns the Plan for a GSO given as dense tensor [E,N,N], SparseGSO, or Plan."""
    if isinstance(S, Plan):
        return S
    if isinstance(S, SparseGSO):
        return S.plan(device if device is not None else torch.device("cuda", torch.cuda.current_device()))
    if not isinstance(S, torch.Tensor):
        raise TypeError("b200gf: GSO must be a torch.Tensor [E,N,N], SparseGSO or Plan, got %r" % type(S))
    if S.requires_grad:
        raise NotImplementedError("b200gf: gradients w.r.t. the GSO are not part of the LSIGF path "
                                  "(the reference keeps S as a plain attribute, graphML.py:2099)")
    _purge_dead_plans()
    if S.layout != torch.strided:
        # torch sparse GSO (SURVEY §8b extension): never densified — converted once to host CSR, cached per tensor
        assert S.dim() == 3 and S.shape[1] == S.shape[2]
        key = ("sparse", id(S), S._version)
        hit = _PLAN_CACHE.get(key)
        if hit is None or hit[0]() is not S:
            if len(_PLAN_CACHE) >= _PLAN_CACHE_MAX:
                _PLAN_CACHE.pop(next(iter(_PLAN_CACHE)))
            hit = (weakref.ref(S), SparseGSO.from_torch_sparse(S))
            _PLAN_CACHE[key] = hit
        if device is None:
            device = S.device if S.device.type == "cuda" else torch.device("cuda", torch.cuda.current_device())
        return hit[1].plan(device)
    assert S.dim() == 3 and S.shape[1] == S.shape[2]
    if S.device.type != "cuda":
        raise RuntimeError("b200gf: LSIGF needs CUDA tensors (there is no CPU fallback); got GSO on %s" % S.device)
    key = _dense_key(S)
    hit = _PLAN_CACHE.get(key)
    if hit is not None and hit[0]() is S:  # same tensor object, same version: the plan is current
        return hit[1]
    csr = [dense_to_csr(S[e]) for e in range(S.shape[0])]
    p = Plan.from_host_csr(csr, S.shape[1], S.dtype, S.device)
    if len(_PLAN_CACHE) >= _PLAN_CACHE_MAX:
        _PLAN_CACHE.pop(next(iter(_PLAN_CACHE)))
    _PLAN_CACHE[key] = (weakref.ref(S), p)
    return p


def clear_plan_cache():
    _PLAN_CACHE.clear()
