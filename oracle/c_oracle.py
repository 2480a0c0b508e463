"""Builds and binds oracle/lsigf_oracle.c (plain-C float64 restatement of LSIGF and its gradients).

TEST INFRASTRUCTURE.  The shared object goes to oracle/_build/ (git-ignored, a build product like the library's .so).
`build()` is called by __graft_entry__.build(); nothing in the product imports this.
"""
import ctypes
import os
import shutil
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "lsigf_oracle.c")
OUT_DIR = os.path.join(HERE, "_build")
LIB = os.path.join(OUT_DIR, "liblsigf_oracle.so")

_lib = None


def build(force=False):
    os.makedirs(OUT_DIR, exist_ok=True)
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < os.path.getmtime(SRC):
        gcc = shutil.which("gcc") or shutil.which("cc")
        if gcc is None:
            raise RuntimeError("no C compiler for the C oracle")
        subprocess.check_call([gcc, "-O2", "-std=c99", "-Wall", "-shared", "-fPIC", "-o", LIB, SRC])
    return LIB


def load():
    global _lib
    if _lib is None:
        lib = ctypes.CDLL(build())
        lib.lsigf_oracle_forward.restype = ctypes.c_int
        lib.lsigf_oracle_backward.restype = ctypes.c_int
        _lib = lib
    return _lib


def _csr_args(S_list):
    import scipy.sparse as sp
    mats = [sp.csr_matrix(np.asarray(m) if not sp.issparse(m) else m).astype(np.float64) for m in S_list]
    keep = []
    for m in mats:
        m.sort_indices()
        keep.append((np.ascontiguousarray(m.indptr, dtype=np.int64), np.ascontiguousarray(m.indices, dtype=np.int32),
                     np.ascontiguousarray(m.data, dtype=np.float64)))
    arr = lambda xs: (ctypes.c_void_p * len(xs))(*[x.ctypes.data for x in xs])  # noqa: E731
    return keep, arr([k[0] for k in keep]), arr([k[1] for k in keep]), arr([k[2] for k in keep])


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def lsigf_forward(h, S_list, x, b=None):
    """h [F,E,K,G], S_list: E matrices (dense arrays or scipy sparse), x [B,G,N], b [F,1] / [F,N] / None -> y [B,F,N]."""
    lib = load()
    h = np.ascontiguousarray(h, dtype=np.float64)
    x = np.ascontiguousarray(x, dtype=np.float64)
    F, E, K, G = h.shape
    B, _, N = x.shape
    keep, rp, ci, va = _csr_args(S_list)
    bias, per_node = None, 0
    if b is not None:
        b = np.asarray(b, dtype=np.float64)
        per_node = 0 if b.shape[1] == 1 else 1
        bias = np.ascontiguousarray(b.reshape(-1) if per_node == 0 else b)
    y = np.empty((B, F, N), dtype=np.float64)
    rc = lib.lsigf_oracle_forward(ctypes.c_int64(N), E, K, G, F, B, rp, ci, va, _p(h), _p(x), _p(bias), per_node, _p(y))
    assert rc == 0
    return y


def lsigf_backward(h, S_list, x, dy, bias_shape=None):
    lib = load()
    h = np.ascontiguousarray(h, dtype=np.float64)
    x = np.ascontiguousarray(x, dtype=np.float64)
    dy = np.ascontiguousarray(dy, dtype=np.float64)
    F, E, K, G = h.shape
    B, _, N = x.shape
    keep, rp, ci, va = _csr_args(S_list)
    dh = np.empty_like(h)
    dx = np.empty_like(x)
    db, per_node = None, 0
    if bias_shape is not None:
        per_node = 0 if bias_shape[1] == 1 else 1
        db = np.empty(bias_shape, dtype=np.float64)
    rc = lib.lsigf_oracle_backward(ctypes.c_int64(N), E, K, G, F, B, rp, ci, va, _p(h), _p(x), _p(dy), per_node, _p(dh),
                                   _p(dx), _p(db))
    assert rc == 0
    return dh, dx, db
