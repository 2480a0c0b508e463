"""Which kernel every hop entry point launches, and with which grid and block, checked on the CPU.

A child process loads libb200gf.so under a preloaded helper that stands in for three CUDA runtime calls:
cudaOccupancyMaxActiveBlocksPerMultiprocessorWithFlags reports a fixed occupancy, cudaLaunchKernel records the
kernel's symbol, grid, block, dynamic shared memory, stream and (for the hop kernels) the row offsets, source,
destination and column count it was given, and launches nothing; cudaGetLastError reports success.  The child also
hides every CUDA device, so placeholder pointers never reach one.  The same helper builds host-only plans (as in
test_cabi_return_codes.py) with the sm count, L2 size, gather spread and source windows each case needs; each operator
(edge feature e, direction) gets its own placeholder pointers, so a launch shows which operator it read.

Each case expects a return code and the ordered launches "kernel<template arguments> grid block".  Together the cases
launch every hop and row-copy kernel compiled into the library."""
import json
import os
import re
import shutil
import subprocess
import sys

import pytest

from dispatch_harness import _norm, library_kernels

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "graph-neural-networks_b200", "csrc")

OK, EUNSUPPORTED = 0, -2
OCC = 3                          # blocks per SM the stand-in occupancy query reports
SRC, DST, MC = 0x10000000, 0x20000000, 0x30000000
PEER = 0x40000000                # peer i at PEER + i * 0x1000000
STREAM = 0x5000
N = 3000

# operator (e, direction) of a host-only plan: placeholders at OP << 36, (1 + e + 8 * direction) << 36 + offset
RP64, RP32, WIN_RP32 = 0x0, 0x100000, 0x400000

_HELPER = r"""
#include <cxxabi.h>
#include <dlfcn.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include "common.cuh"

static std::string g_log;

extern "C" cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessorWithFlags(int* n, const void*, int, size_t,
                                                                              unsigned) {
  *n = OCC;
  return cudaSuccess;
}
extern "C" cudaError_t cudaGetLastError() { return cudaSuccess; }
extern "C" cudaError_t cudaLaunchKernel(const void* fn, dim3 g, dim3 b, void** args, size_t smem, cudaStream_t st) {
  Dl_info info{};
  const char* sym = dladdr(fn, &info) && info.dli_sname ? info.dli_sname : "?";
  int status = 0;
  char* name = abi::__cxa_demangle(sym, nullptr, nullptr, &status);
  char line[2048];
  int n = snprintf(line, sizeof line, "%s;%u %u %u;%u %u %u;%zu;%p", name ? name : sym, g.x, g.y, g.z, b.x, b.y, b.z,
                   smem, (void*)st);
  free(name);
  if (strstr(sym, "spmm_hop"))   // every hop kernel: (row offsets, col, val, src, src_ld, dst, dst_ld, n_rows, C, ...)
    snprintf(line + n, sizeof line - n, ";%p %p %p %d", *(void**)args[0], *(void**)args[3], *(void**)args[5],
             *(int*)args[8]);
  g_log += line;
  g_log += '\n';
  return cudaSuccess;
}
extern "C" const char* hl_take() {
  static std::string out;
  out.swap(g_log);
  g_log.clear();
  return out.c_str();
}

extern "C" b200gf_plan* hl_plan(int64_t n_rows, int64_t n_cols, int dtype, int v2, int sm_count, int64_t l2_bytes,
                                int spread, int n_win) {
  b200gf_plan* p = new b200gf_plan();
  p->dtype = dtype; p->n_rows = n_rows; p->n_cols = n_cols; p->E = 2; p->has_bwd = true;
  p->sm_count = sm_count; p->l2_bytes = l2_bytes;
  p->fwd.resize(2); p->bwd.resize(2);
  for (int d = 0; d < 2; ++d)
    for (int e = 0; e < 2; ++e) {
      b200gf::CsrDev& A = d ? p->bwd[e] : p->fwd[e];
      char* base = (char*)((int64_t)(1 + e + 8 * d) << 36);
      A.rowptr = (int64_t*)(base + RP64);
      A.rowptr32 = v2 ? (int32_t*)(base + RP32) : nullptr;
      A.col = (int32_t*)(base + 0x200000); A.val = base + 0x300000;
      A.spread = spread != 0; A.n_win = n_win;
      if (n_win) {
        A.win_rows = (n_cols + n_win - 1) / n_win;
        A.win_rowptr32 = (int32_t*)(base + WIN_RP32);
        A.win_col = (int32_t*)(base + 0x500000); A.win_val = base + 0x600000;
      }
    }
  return p;
}
extern "C" void hl_plan_free(b200gf_plan* p) { delete p; }
"""

_CHILD = r"""
import ctypes, json, sys
import gnn_b200
helper_path, cases_path, out_path = sys.argv[1:]
h = ctypes.CDLL(helper_path)
h.hl_take.restype = ctypes.c_char_p
h.hl_plan.restype = ctypes.c_void_p
h.hl_plan.argtypes = [ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int64,
                      ctypes.c_int, ctypes.c_int]
lib = gnn_b200._cabi.load()
plans = {}

def arg(a):
    if isinstance(a, dict) and "plan" in a:
        key = json.dumps(a["plan"], sort_keys=True)
        if key not in plans:
            plans[key] = h.hl_plan(*a["plan"])
        return plans[key]
    if isinstance(a, dict):
        return gnn_b200._cabi.ptr_array(a["ptrs"])
    return a

out = {}
h.hl_take()
for cid, fn, args in json.load(open(cases_path)):
    rc = getattr(lib, fn)(*[arg(a) for a in args])
    out[cid] = [rc, [l for l in h.hl_take().decode().split("\n") if l]]
json.dump(out, open(out_path, "w"))
"""


def _ptrs(n, shift_at=None, by=0):
    return {"ptrs": [PEER + 0x1000000 * i + (by if i == shift_at else 0) for i in range(n)]}


def _plan(dt, n_rows=N, n_cols=None, v2=1, sm_count=132, l2=0, spread=0, n_win=0):
    return {"plan": [n_rows, n_rows if n_cols is None else n_cols, dt, v2, sm_count, l2, spread, n_win]}


def _cases(dt):
    """(id, entry point, arguments) of every case in one dtype; widths in bytes, so both dtypes take the same routes."""
    s = 4 if dt == 0 else 8
    v16, v32 = 16 // s, 32 // s

    def c(nbytes):
        return nbytes // s

    def pad(C):
        return (C + v32 - 1) // v32 * v32

    def hop(nbytes, ld=None, src=0, dst=0, e=0, d=0, **plan):
        C = c(nbytes)
        ld = ld or pad(C)
        return "b200gf_hop", [_plan(dt, **plan), e, d, SRC + src, ld, DST + dst, ld, C, STREAM]

    def scatter(nbytes, src=0, out_col=None, **plan):
        C = c(nbytes)
        oc = C if out_col is None else out_col
        return "b200gf_hop_scatter", [_plan(dt, **plan), 1, 0, SRC + src, pad(C), DST, pad(C), C, _ptrs(2), 2, N // 2,
                                      4 * pad(C), oc, C, 2 * pad(C), STREAM]

    def bcast(nbytes, peers=None, mc=None, **plan):
        C = c(nbytes)
        return "b200gf_hop_bcast", [_plan(dt, **plan), 0, 1, SRC, pad(C), C, peers or _ptrs(3), 3, mc, 0, pad(C),
                                    STREAM]

    def grid(nbytes, n_bc=2, out_col=None, **plan):
        C = c(nbytes)
        oc = C if out_col is None else out_col
        return "b200gf_hop_grid", [_plan(dt, **plan), 1, 1, SRC, pad(C), C, _ptrs(n_bc) if n_bc else None, n_bc, 0,
                                   pad(C), _ptrs(2), 2, N // 2, 4 * pad(C), oc, C, 2 * pad(C), STREAM]

    wide = 65536 * 1024            # bytes per row: 65536 chunks of 1 KB
    win = dict(l2=1000000, n_win=3)
    cases = {
        # plain hop, the row width alone picks the kernel
        "plain-1col": hop(s), "plain-32B": hop(32), "plain-48B-16B-ld": hop(48, ld=c(48)), "plain-64B": hop(64),
        "plain-64B-no-32bit-offsets": hop(64, v2=0), "plain-128B": hop(128), "plain-256B": hop(256),
        "plain-512B-bwd-e1": hop(512, e=1, d=1), "plain-1KB": hop(1024), "plain-4400B": hop(4400),
        # unaligned and 16-byte-only operands, no 32-bit offsets, more rows than int32 holds
        "plain-unaligned-src": hop(256, src=s if s == 4 else 8), "plain-odd-ld": hop(64, ld=c(64) + 1),
        "plain-16B-src-256B": hop(256, src=16), "plain-16B-dst-1KB": hop(1024, dst=16),
        "plain-no-32bit-offsets-256B": hop(256, v2=0), "plain-no-32bit-offsets-1KB-bwd": hop(1024, v2=0, d=1),
        "plain-rows-over-int32": hop(256, n_rows=1 << 31),
        # empty hops, the chunk limit of the v2 kernel, and grids capped at sm_count x occupancy
        "plain-empty": hop(256, n_rows=0), "plain-empty-too-many-chunks": hop(wide, n_rows=0),
        "plain-too-many-chunks": hop(wide), "plain-empty-unaligned": hop(256, src=8, n_rows=0),
        "plain-cap-v2": hop(256, n_rows=100000), "plain-cap-multirow": hop(16, n_rows=100000),
        "plain-cap-multirow-v2": hop(64, n_rows=100000, sm_count=16),
        "plain-cap-scalar": hop(256, src=8, n_rows=100000),
        "plain-cap-v1": hop(1024, v2=0, n_rows=100000),
        # L2-sized column chunks (N = 3000 source rows)
        "l2-1KB-L16": hop(1024, l2=1600000), "l2-1KB-L8": hop(1024, l2=800000), "l2-1KB-L4": hop(1024, l2=400000),
        "l2-1KB-nothing-fits": hop(1024, l2=100000), "l2-256B-spread-L4": hop(256, l2=300000, spread=1),
        "l2-256B-no-spread": hop(256, l2=300000), "l2-1KB-partitioned-plan": hop(1024, l2=400000, n_cols=2 * N),
        # windowed hop: chunk-major, then window-major
        "win-256B": hop(256, **win), "win-160B": hop(160, **win), "win-128B-bwd-e1": hop(128, e=1, d=1, **win),
        "win-96B": hop(96, **win), "win-no-l2": hop(256, n_win=3), "win-16B-src": hop(256, src=16, **win),
        "win-empty": hop(256, n_rows=0, **win), "win-scatter": scatter(256, **win),
        # fused NVLink scatter
        "scatter-16B": scatter(16), "scatter-64B": scatter(64), "scatter-64B-16B-fields": scatter(64, out_col=v16),
        "scatter-256B-l2": scatter(256, l2=300000, spread=1), "scatter-512B": scatter(512),
        "scatter-1KB": scatter(1024),
        "scatter-256B-16B-fields": scatter(256, out_col=v16), "scatter-1KB-no-32bit-offsets": scatter(1024, v2=0),
        "scatter-unaligned-src": scatter(256, src=8), "scatter-8B-fields": scatter(256, out_col=c(8) or 1),
        "scatter-empty": scatter(256, n_rows=0),
        # fused all-gather
        "bcast-96B": bcast(96), "bcast-256B": bcast(256), "bcast-512B-mc": bcast(512, mc=MC),
        "bcast-1KB-l2": bcast(1024, l2=400000), "bcast-64B": bcast(64), "bcast-32B": bcast(32),
        "bcast-peer-16B": bcast(256, peers=_ptrs(3, shift_at=1, by=16)), "bcast-mc-16B": bcast(256, mc=MC + 16),
        "bcast-no-32bit-offsets": bcast(256, v2=0), "bcast-empty": bcast(256, n_rows=0),
        # all-gather + scatter
        "grid-64B": grid(64), "grid-96B": grid(96), "grid-256B": grid(256), "grid-512B": grid(512),
        "grid-1KB-l2": grid(1024, l2=400000), "grid-scatter-only-256B": grid(256, n_bc=0),
        "grid-scatter-only-64B": grid(64, n_bc=0), "grid-16B-fields": grid(256, out_col=v16), "grid-32B": grid(32),
        "grid-no-32bit-offsets": grid(256, v2=0), "grid-empty": grid(256, n_rows=0),
        # row copies of the k = 0 term
        "bcast-rows": ("b200gf_bcast_rows", [dt, SRC, c(256), N, c(256), _ptrs(2), 2, None, 0, c(256), STREAM]),
        "bcast-rows-unaligned": ("b200gf_bcast_rows", [dt, SRC + 8, c(256), N, c(256), _ptrs(2), 2, None, 0, c(256),
                                                       STREAM]),
        "scatter-rows": ("b200gf_scatter_rows", [dt, SRC, c(256), N, c(256), _ptrs(2), 2, N // 2, c(1024), c(256),
                                                 c(256), c(512), STREAM]),
        "scatter-rows-8B-fields": ("b200gf_scatter_rows", [dt, SRC, c(256), N, c(256), _ptrs(2), 2, N // 2, c(1024),
                                                           c(8) or 1, c(256), c(512), STREAM]),
    }
    name = "f32" if dt == 0 else "f64"
    return [("%s-%s" % (name, k), fn, args) for k, (fn, args) in cases.items()]


CASES = _cases(0) + _cases(1)
ARGS = {cid: args for cid, _, args in CASES}

EXPECTED = {   # recorded from the library before its hop launchers were restructured
    "f32-plain-1col": (OK, ["spmm_hop_multirow_kernel<float,4,1,8,1,256,6,3> 94x1x1 256x1x1"]),
    "f32-plain-32B": (OK, ["spmm_hop_multirow_kernel<float,4,2,8,2,256,6,3> 94x1x1 256x1x1"]),
    "f32-plain-48B-16B-ld": (OK, ["spmm_hop_multirow_kernel<float,4,4,16,2,256,8,3> 188x1x1 256x1x1"]),
    "f32-plain-64B": (OK, ["spmm_hop_multirow_v2_kernel<float,int,8,2,8,2,256,4,3,0> 94x1x1 256x1x1"]),
    "f32-plain-64B-no-32bit-offsets": (OK, ["spmm_hop_multirow_kernel<float,4,4,16,2,256,8,3> 188x1x1 256x1x1"]),
    "f32-plain-128B": (OK, ["spmm_hop_multirow_kernel<float,4,8,32,4,256,6,3> 375x1x1 256x1x1"]),
    "f32-plain-256B": (OK, ["spmm_hop_v2_kernel<float,int,8,8,4,256,4,3,0,1> 375x1x1 256x1x1"]),
    "f32-plain-512B-bwd-e1": (OK, ["spmm_hop_v2_kernel<float,int,8,16,4,256,4,3,0,1> 375x1x1 256x1x1"]),
    "f32-plain-1KB": (OK, ["spmm_hop_v2_kernel<float,int,8,32,4,256,4,3,0,1> 375x1x1 256x1x1"]),
    "f32-plain-4400B": (OK, ["spmm_hop_v2_kernel<float,int,8,32,4,256,4,3,0,1> 375x5x1 256x1x1"]),
    "f32-plain-unaligned-src": (OK, ["spmm_hop_kernel<float,1,32,4,256,6,3,0,0> 396x1x1 256x1x1"]),
    "f32-plain-odd-ld": (OK, ["spmm_hop_kernel<float,1,32,4,256,6,3,0,0> 375x1x1 256x1x1"]),
    "f32-plain-16B-src-256B": (OK, ["spmm_hop_kernel<float,4,16,4,256,6,3,0,0> 375x1x1 256x1x1"]),
    "f32-plain-16B-dst-1KB": (OK, ["spmm_hop_kernel<float,4,32,4,256,6,3,0,0> 396x1x1 256x1x1"]),
    "f32-plain-no-32bit-offsets-256B": (OK, ["spmm_hop_kernel<float,4,16,4,256,6,3,0,0> 375x1x1 256x1x1"]),
    "f32-plain-no-32bit-offsets-1KB-bwd": (OK, ["spmm_hop_kernel<float,4,32,4,256,6,3,0,0> 396x1x1 256x1x1"]),
    "f32-plain-rows-over-int32": (OK, ["spmm_hop_kernel<float,4,16,4,256,6,3,0,0> 396x1x1 256x1x1"]),
    "f32-plain-empty": (OK, []),
    "f32-plain-empty-too-many-chunks": (OK, []),
    "f32-plain-too-many-chunks": (EUNSUPPORTED, []),
    "f32-plain-empty-unaligned": (OK, []),
    "f32-plain-cap-v2": (OK, ["spmm_hop_v2_kernel<float,int,8,8,4,256,4,3,0,1> 396x1x1 256x1x1"]),
    "f32-plain-cap-multirow": (OK, ["spmm_hop_multirow_kernel<float,4,1,8,1,256,6,3> 396x1x1 256x1x1"]),
    "f32-plain-cap-multirow-v2": (OK, ["spmm_hop_multirow_v2_kernel<float,int,8,2,8,2,256,4,3,0> 48x1x1 256x1x1"]),
    "f32-plain-cap-scalar": (OK, ["spmm_hop_kernel<float,1,32,4,256,6,3,0,0> 396x1x1 256x1x1"]),
    "f32-plain-cap-v1": (OK, ["spmm_hop_kernel<float,4,32,4,256,6,3,0,0> 396x1x1 256x1x1"]),
    "f32-l2-1KB-L16": (OK, ["spmm_hop_v2_kernel<float,int,8,16,4,256,4,3,0,1> 375x2x1 256x1x1"]),
    "f32-l2-1KB-L8": (OK, ["spmm_hop_v2_kernel<float,int,8,8,4,256,4,3,0,1> 375x4x1 256x1x1"]),
    "f32-l2-1KB-L4": (OK, ["spmm_hop_v2_kernel<float,int,8,4,4,256,4,3,0,1> 375x8x1 256x1x1"]),
    "f32-l2-1KB-nothing-fits": (OK, ["spmm_hop_v2_kernel<float,int,8,32,4,256,4,3,0,1> 375x1x1 256x1x1"]),
    "f32-l2-256B-spread-L4": (OK, ["spmm_hop_v2_kernel<float,int,8,4,4,256,4,3,0,1> 375x2x1 256x1x1"]),
    "f32-l2-256B-no-spread": (OK, ["spmm_hop_v2_kernel<float,int,8,8,4,256,4,3,0,1> 375x1x1 256x1x1"]),
    "f32-l2-1KB-partitioned-plan": (OK, ["spmm_hop_v2_kernel<float,int,8,32,4,256,4,3,0,1> 375x1x1 256x1x1"]),
    "f32-win-256B": (OK, [
        "spmm_hop_multirow_v2_kernel<float,int,8,4,4,4,256,4,3,0> 47x1x1 256x1x1",
        "spmm_hop_multirow_v2_kernel<float,int,8,4,4,4,256,4,3,4> 47x1x1 256x1x1",
        "spmm_hop_multirow_v2_kernel<float,int,8,4,4,4,256,4,3,4> 47x1x1 256x1x1",
        "spmm_hop_multirow_v2_kernel<float,int,8,4,4,4,256,4,3,0> 47x1x1 256x1x1",
        "spmm_hop_multirow_v2_kernel<float,int,8,4,4,4,256,4,3,4> 47x1x1 256x1x1",
        "spmm_hop_multirow_v2_kernel<float,int,8,4,4,4,256,4,3,4> 47x1x1 256x1x1",
    ]),
    "f32-win-160B": (OK, [
        "spmm_hop_multirow_v2_kernel<float,int,8,4,4,4,256,4,3,0> 47x1x1 256x1x1",
        "spmm_hop_multirow_v2_kernel<float,int,8,4,4,4,256,4,3,4> 47x1x1 256x1x1",
        "spmm_hop_multirow_v2_kernel<float,int,8,4,4,4,256,4,3,4> 47x1x1 256x1x1",
        "spmm_hop_multirow_v2_kernel<float,int,8,4,4,4,256,4,3,0> 47x1x1 256x1x1",
        "spmm_hop_multirow_v2_kernel<float,int,8,4,4,4,256,4,3,4> 47x1x1 256x1x1",
        "spmm_hop_multirow_v2_kernel<float,int,8,4,4,4,256,4,3,4> 47x1x1 256x1x1",
    ]),
    "f32-win-128B-bwd-e1": (OK, [
        "spmm_hop_multirow_v2_kernel<float,int,8,4,4,4,256,4,3,0> 47x1x1 256x1x1",
        "spmm_hop_multirow_v2_kernel<float,int,8,4,4,4,256,4,3,4> 47x1x1 256x1x1",
        "spmm_hop_multirow_v2_kernel<float,int,8,4,4,4,256,4,3,4> 47x1x1 256x1x1",
    ]),
    "f32-win-96B": (OK, ["spmm_hop_multirow_kernel<float,4,8,32,4,256,6,3> 375x1x1 256x1x1"]),
    "f32-win-no-l2": (OK, ["spmm_hop_v2_kernel<float,int,8,8,4,256,4,3,0,1> 375x1x1 256x1x1"]),
    "f32-win-16B-src": (OK, ["spmm_hop_kernel<float,4,16,4,256,6,3,0,0> 375x1x1 256x1x1"]),
    "f32-win-empty": (OK, []),
    "f32-win-scatter": (OK, ["spmm_hop_v2_kernel<float,int,8,8,4,256,4,3,1,1> 375x1x1 256x1x1"]),
    "f32-scatter-16B": (OK, ["spmm_hop_multirow_kernel<float,4,1,8,1,256,6,3> 94x1x1 256x1x1"]),
    "f32-scatter-64B": (OK, ["spmm_hop_multirow_v2_kernel<float,int,8,2,8,2,256,4,3,1> 94x1x1 256x1x1"]),
    "f32-scatter-64B-16B-fields": (OK, ["spmm_hop_multirow_kernel<float,4,4,16,2,256,8,3> 188x1x1 256x1x1"]),
    "f32-scatter-256B-l2": (OK, ["spmm_hop_v2_kernel<float,int,8,8,4,256,4,3,1,1> 375x1x1 256x1x1"]),
    "f32-scatter-512B": (OK, ["spmm_hop_v2_kernel<float,int,8,16,4,256,4,3,1,1> 375x1x1 256x1x1"]),
    "f32-scatter-1KB": (OK, ["spmm_hop_v2_kernel<float,int,8,32,4,256,4,3,1,1> 375x1x1 256x1x1"]),
    "f32-scatter-256B-16B-fields": (OK, ["spmm_hop_kernel<float,4,16,4,256,6,3,0,0> 375x1x1 256x1x1"]),
    "f32-scatter-1KB-no-32bit-offsets": (OK, ["spmm_hop_kernel<float,4,32,4,256,6,3,0,0> 396x1x1 256x1x1"]),
    "f32-scatter-unaligned-src": (EUNSUPPORTED, []),
    "f32-scatter-8B-fields": (EUNSUPPORTED, []),
    "f32-scatter-empty": (OK, []),
    "f32-bcast-96B": (OK, ["spmm_hop_v2_kernel<float,int,8,4,4,256,4,3,2,1> 375x1x1 256x1x1"]),
    "f32-bcast-256B": (OK, ["spmm_hop_v2_kernel<float,int,8,8,4,256,4,3,2,1> 375x1x1 256x1x1"]),
    "f32-bcast-512B-mc": (OK, ["spmm_hop_v2_kernel<float,int,8,16,4,256,4,3,2,1> 375x1x1 256x1x1"]),
    "f32-bcast-1KB-l2": (OK, ["spmm_hop_v2_kernel<float,int,8,32,4,256,4,3,2,1> 375x1x1 256x1x1"]),
    "f32-bcast-64B": (EUNSUPPORTED, []),
    "f32-bcast-32B": (EUNSUPPORTED, []),
    "f32-bcast-peer-16B": (EUNSUPPORTED, []),
    "f32-bcast-mc-16B": (EUNSUPPORTED, []),
    "f32-bcast-no-32bit-offsets": (EUNSUPPORTED, []),
    "f32-bcast-empty": (OK, []),
    "f32-grid-64B": (OK, ["spmm_hop_multirow_v2_kernel<float,int,8,2,8,2,256,4,3,3> 94x1x1 256x1x1"]),
    "f32-grid-96B": (OK, ["spmm_hop_v2_kernel<float,int,8,4,4,256,4,3,3,1> 375x1x1 256x1x1"]),
    "f32-grid-256B": (OK, ["spmm_hop_v2_kernel<float,int,8,8,4,256,4,3,3,1> 375x1x1 256x1x1"]),
    "f32-grid-512B": (OK, ["spmm_hop_v2_kernel<float,int,8,16,4,256,4,3,3,1> 375x1x1 256x1x1"]),
    "f32-grid-1KB-l2": (OK, ["spmm_hop_v2_kernel<float,int,8,32,4,256,4,3,3,1> 375x1x1 256x1x1"]),
    "f32-grid-scatter-only-256B": (OK, ["spmm_hop_v2_kernel<float,int,8,8,4,256,4,3,3,1> 375x1x1 256x1x1"]),
    "f32-grid-scatter-only-64B": (OK, ["spmm_hop_multirow_v2_kernel<float,int,8,2,8,2,256,4,3,3> 94x1x1 256x1x1"]),
    "f32-grid-16B-fields": (EUNSUPPORTED, []),
    "f32-grid-32B": (EUNSUPPORTED, []),
    "f32-grid-no-32bit-offsets": (EUNSUPPORTED, []),
    "f32-grid-empty": (OK, []),
    "f32-bcast-rows": (OK, ["bcast_rows_kernel<float,4> 1056x1x1 256x1x1"]),
    "f32-bcast-rows-unaligned": (EUNSUPPORTED, []),
    "f32-scatter-rows": (OK, ["scatter_rows_kernel<float,4> 1056x1x1 256x1x1"]),
    "f32-scatter-rows-8B-fields": (EUNSUPPORTED, []),
    "f64-plain-1col": (OK, ["spmm_hop_multirow_kernel<double,2,1,8,1,256,4,3> 94x1x1 256x1x1"]),
    "f64-plain-32B": (OK, ["spmm_hop_multirow_kernel<double,2,2,8,2,256,4,3> 94x1x1 256x1x1"]),
    "f64-plain-48B-16B-ld": (OK, ["spmm_hop_multirow_kernel<double,2,4,16,2,256,4,3> 188x1x1 256x1x1"]),
    "f64-plain-64B": (OK, ["spmm_hop_multirow_v2_kernel<double,int,4,2,8,2,256,3,3,0> 94x1x1 256x1x1"]),
    "f64-plain-64B-no-32bit-offsets": (OK, ["spmm_hop_multirow_kernel<double,2,4,16,2,256,4,3> 188x1x1 256x1x1"]),
    "f64-plain-128B": (OK, ["spmm_hop_multirow_kernel<double,2,8,32,4,256,4,3> 375x1x1 256x1x1"]),
    "f64-plain-256B": (OK, ["spmm_hop_v2_kernel<double,int,4,8,4,256,3,3,0,1> 375x1x1 256x1x1"]),
    "f64-plain-512B-bwd-e1": (OK, ["spmm_hop_v2_kernel<double,int,4,16,4,256,3,3,0,1> 375x1x1 256x1x1"]),
    "f64-plain-1KB": (OK, ["spmm_hop_v2_kernel<double,int,4,32,4,256,3,3,0,1> 375x1x1 256x1x1"]),
    "f64-plain-4400B": (OK, ["spmm_hop_v2_kernel<double,int,4,32,4,256,3,3,0,1> 375x5x1 256x1x1"]),
    "f64-plain-unaligned-src": (OK, ["spmm_hop_kernel<double,1,32,4,256,4,3,0,0> 375x1x1 256x1x1"]),
    "f64-plain-odd-ld": (OK, ["spmm_hop_kernel<double,1,32,4,256,4,3,0,0> 375x1x1 256x1x1"]),
    "f64-plain-16B-src-256B": (OK, ["spmm_hop_kernel<double,2,16,4,256,4,3,0,0> 375x1x1 256x1x1"]),
    "f64-plain-16B-dst-1KB": (OK, ["spmm_hop_kernel<double,2,32,4,256,4,3,0,0> 396x1x1 256x1x1"]),
    "f64-plain-no-32bit-offsets-256B": (OK, ["spmm_hop_kernel<double,2,16,4,256,4,3,0,0> 375x1x1 256x1x1"]),
    "f64-plain-no-32bit-offsets-1KB-bwd": (OK, ["spmm_hop_kernel<double,2,32,4,256,4,3,0,0> 396x1x1 256x1x1"]),
    "f64-plain-rows-over-int32": (OK, ["spmm_hop_kernel<double,2,16,4,256,4,3,0,0> 396x1x1 256x1x1"]),
    "f64-plain-empty": (OK, []),
    "f64-plain-empty-too-many-chunks": (OK, []),
    "f64-plain-too-many-chunks": (EUNSUPPORTED, []),
    "f64-plain-empty-unaligned": (OK, []),
    "f64-plain-cap-v2": (OK, ["spmm_hop_v2_kernel<double,int,4,8,4,256,3,3,0,1> 396x1x1 256x1x1"]),
    "f64-plain-cap-multirow": (OK, ["spmm_hop_multirow_kernel<double,2,1,8,1,256,4,3> 396x1x1 256x1x1"]),
    "f64-plain-cap-multirow-v2": (OK, ["spmm_hop_multirow_v2_kernel<double,int,4,2,8,2,256,3,3,0> 48x1x1 256x1x1"]),
    "f64-plain-cap-scalar": (OK, ["spmm_hop_kernel<double,1,32,4,256,4,3,0,0> 396x1x1 256x1x1"]),
    "f64-plain-cap-v1": (OK, ["spmm_hop_kernel<double,2,32,4,256,4,3,0,0> 396x1x1 256x1x1"]),
    "f64-l2-1KB-L16": (OK, ["spmm_hop_v2_kernel<double,int,4,16,4,256,3,3,0,1> 375x2x1 256x1x1"]),
    "f64-l2-1KB-L8": (OK, ["spmm_hop_v2_kernel<double,int,4,8,4,256,3,3,0,1> 375x4x1 256x1x1"]),
    "f64-l2-1KB-L4": (OK, ["spmm_hop_v2_kernel<double,int,4,4,4,256,3,3,0,1> 375x8x1 256x1x1"]),
    "f64-l2-1KB-nothing-fits": (OK, ["spmm_hop_v2_kernel<double,int,4,32,4,256,3,3,0,1> 375x1x1 256x1x1"]),
    "f64-l2-256B-spread-L4": (OK, ["spmm_hop_v2_kernel<double,int,4,4,4,256,3,3,0,1> 375x2x1 256x1x1"]),
    "f64-l2-256B-no-spread": (OK, ["spmm_hop_v2_kernel<double,int,4,8,4,256,3,3,0,1> 375x1x1 256x1x1"]),
    "f64-l2-1KB-partitioned-plan": (OK, ["spmm_hop_v2_kernel<double,int,4,32,4,256,3,3,0,1> 375x1x1 256x1x1"]),
    "f64-win-256B": (OK, [
        "spmm_hop_multirow_v2_kernel<double,int,4,4,4,4,256,3,3,0> 47x1x1 256x1x1",
        "spmm_hop_multirow_v2_kernel<double,int,4,4,4,4,256,3,3,4> 47x1x1 256x1x1",
        "spmm_hop_multirow_v2_kernel<double,int,4,4,4,4,256,3,3,4> 47x1x1 256x1x1",
        "spmm_hop_multirow_v2_kernel<double,int,4,4,4,4,256,3,3,0> 47x1x1 256x1x1",
        "spmm_hop_multirow_v2_kernel<double,int,4,4,4,4,256,3,3,4> 47x1x1 256x1x1",
        "spmm_hop_multirow_v2_kernel<double,int,4,4,4,4,256,3,3,4> 47x1x1 256x1x1",
    ]),
    "f64-win-160B": (OK, [
        "spmm_hop_multirow_v2_kernel<double,int,4,4,4,4,256,3,3,0> 47x1x1 256x1x1",
        "spmm_hop_multirow_v2_kernel<double,int,4,4,4,4,256,3,3,4> 47x1x1 256x1x1",
        "spmm_hop_multirow_v2_kernel<double,int,4,4,4,4,256,3,3,4> 47x1x1 256x1x1",
        "spmm_hop_multirow_v2_kernel<double,int,4,4,4,4,256,3,3,0> 47x1x1 256x1x1",
        "spmm_hop_multirow_v2_kernel<double,int,4,4,4,4,256,3,3,4> 47x1x1 256x1x1",
        "spmm_hop_multirow_v2_kernel<double,int,4,4,4,4,256,3,3,4> 47x1x1 256x1x1",
    ]),
    "f64-win-128B-bwd-e1": (OK, [
        "spmm_hop_multirow_v2_kernel<double,int,4,4,4,4,256,3,3,0> 47x1x1 256x1x1",
        "spmm_hop_multirow_v2_kernel<double,int,4,4,4,4,256,3,3,4> 47x1x1 256x1x1",
        "spmm_hop_multirow_v2_kernel<double,int,4,4,4,4,256,3,3,4> 47x1x1 256x1x1",
    ]),
    "f64-win-96B": (OK, ["spmm_hop_multirow_kernel<double,2,8,32,4,256,4,3> 375x1x1 256x1x1"]),
    "f64-win-no-l2": (OK, ["spmm_hop_v2_kernel<double,int,4,8,4,256,3,3,0,1> 375x1x1 256x1x1"]),
    "f64-win-16B-src": (OK, ["spmm_hop_kernel<double,2,16,4,256,4,3,0,0> 375x1x1 256x1x1"]),
    "f64-win-empty": (OK, []),
    "f64-win-scatter": (OK, ["spmm_hop_v2_kernel<double,int,4,8,4,256,3,3,1,1> 375x1x1 256x1x1"]),
    "f64-scatter-16B": (OK, ["spmm_hop_multirow_kernel<double,2,1,8,1,256,4,3> 94x1x1 256x1x1"]),
    "f64-scatter-64B": (OK, ["spmm_hop_multirow_v2_kernel<double,int,4,2,8,2,256,3,3,1> 94x1x1 256x1x1"]),
    "f64-scatter-64B-16B-fields": (OK, ["spmm_hop_multirow_kernel<double,2,4,16,2,256,4,3> 188x1x1 256x1x1"]),
    "f64-scatter-256B-l2": (OK, ["spmm_hop_v2_kernel<double,int,4,8,4,256,3,3,1,1> 375x1x1 256x1x1"]),
    "f64-scatter-512B": (OK, ["spmm_hop_v2_kernel<double,int,4,16,4,256,3,3,1,1> 375x1x1 256x1x1"]),
    "f64-scatter-1KB": (OK, ["spmm_hop_v2_kernel<double,int,4,32,4,256,3,3,1,1> 375x1x1 256x1x1"]),
    "f64-scatter-256B-16B-fields": (OK, ["spmm_hop_kernel<double,2,16,4,256,4,3,0,0> 375x1x1 256x1x1"]),
    "f64-scatter-1KB-no-32bit-offsets": (OK, ["spmm_hop_kernel<double,2,32,4,256,4,3,0,0> 396x1x1 256x1x1"]),
    "f64-scatter-unaligned-src": (EUNSUPPORTED, []),
    "f64-scatter-8B-fields": (EUNSUPPORTED, []),
    "f64-scatter-empty": (OK, []),
    "f64-bcast-96B": (OK, ["spmm_hop_v2_kernel<double,int,4,4,4,256,3,3,2,1> 375x1x1 256x1x1"]),
    "f64-bcast-256B": (OK, ["spmm_hop_v2_kernel<double,int,4,8,4,256,3,3,2,1> 375x1x1 256x1x1"]),
    "f64-bcast-512B-mc": (OK, ["spmm_hop_v2_kernel<double,int,4,16,4,256,3,3,2,1> 375x1x1 256x1x1"]),
    "f64-bcast-1KB-l2": (OK, ["spmm_hop_v2_kernel<double,int,4,32,4,256,3,3,2,1> 375x1x1 256x1x1"]),
    "f64-bcast-64B": (EUNSUPPORTED, []),
    "f64-bcast-32B": (EUNSUPPORTED, []),
    "f64-bcast-peer-16B": (EUNSUPPORTED, []),
    "f64-bcast-mc-16B": (EUNSUPPORTED, []),
    "f64-bcast-no-32bit-offsets": (EUNSUPPORTED, []),
    "f64-bcast-empty": (OK, []),
    "f64-grid-64B": (OK, ["spmm_hop_multirow_v2_kernel<double,int,4,2,8,2,256,3,3,3> 94x1x1 256x1x1"]),
    "f64-grid-96B": (OK, ["spmm_hop_v2_kernel<double,int,4,4,4,256,3,3,3,1> 375x1x1 256x1x1"]),
    "f64-grid-256B": (OK, ["spmm_hop_v2_kernel<double,int,4,8,4,256,3,3,3,1> 375x1x1 256x1x1"]),
    "f64-grid-512B": (OK, ["spmm_hop_v2_kernel<double,int,4,16,4,256,3,3,3,1> 375x1x1 256x1x1"]),
    "f64-grid-1KB-l2": (OK, ["spmm_hop_v2_kernel<double,int,4,32,4,256,3,3,3,1> 375x1x1 256x1x1"]),
    "f64-grid-scatter-only-256B": (OK, ["spmm_hop_v2_kernel<double,int,4,8,4,256,3,3,3,1> 375x1x1 256x1x1"]),
    "f64-grid-scatter-only-64B": (OK, ["spmm_hop_multirow_v2_kernel<double,int,4,2,8,2,256,3,3,3> 94x1x1 256x1x1"]),
    "f64-grid-16B-fields": (EUNSUPPORTED, []),
    "f64-grid-32B": (EUNSUPPORTED, []),
    "f64-grid-no-32bit-offsets": (EUNSUPPORTED, []),
    "f64-grid-empty": (OK, []),
    "f64-bcast-rows": (OK, ["bcast_rows_kernel<double,2> 1056x1x1 256x1x1"]),
    "f64-bcast-rows-unaligned": (EUNSUPPORTED, []),
    "f64-scatter-rows": (OK, ["scatter_rows_kernel<double,2> 1056x1x1 256x1x1"]),
    "f64-scatter-rows-8B-fields": (EUNSUPPORTED, []),
}


def _short(line):
    """'kernel<template arguments> grid block' of one recorded launch."""
    name, g, b = line.split(";")[:3]
    name = _norm(name.split("(")[0]).replace("voidb200gf::", "").replace("b200gf::", "")
    return "%s %s %s" % (name, "x".join(g.split()), "x".join(b.split()))


@pytest.fixture(scope="module")
def launches(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    import gnn_b200
    if not os.path.exists(gnn_b200._cabi.LIB_PATH):
        pytest.skip("libb200gf.so is not built")
    d = tmp_path_factory.mktemp("hop_launches")
    src, so, cases, out = d / "hop_shim.cpp", d / "hop_shim.so", d / "cases.json", d / "out.json"
    defs = "".join("#define %s %d\n" % kv for kv in dict(OCC=OCC, RP64=RP64, RP32=RP32, WIN_RP32=WIN_RP32).items())
    src.write_text(defs + _HELPER)
    r = subprocess.run([nvcc, "-std=c++17", "-shared", "-cudart", "none", "-Xcompiler", "-fPIC", "-I", CSRC, str(src),
                        "-o", str(so), "-ldl"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    cases.write_text(json.dumps(CASES))
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, LD_PRELOAD=str(so), CUDA_VISIBLE_DEVICES="", PYTHONDONTWRITEBYTECODE="1",
               PYTHONPATH=os.pathsep.join([here, ROOT] + [p for p in os.environ.get("PYTHONPATH", "").split(os.pathsep)
                                                          if p]))
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", _CHILD, str(so), str(cases), str(out)], env=env, cwd=ROOT,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    return json.loads(out.read_text())


@pytest.mark.parametrize("cid", sorted(ARGS))
def test_hop_launch(cid, launches):
    rc, lines = launches[cid]
    want_rc, want = EXPECTED[cid]
    assert (rc, [_short(l) for l in lines]) == (want_rc, want)
    args = ARGS[cid]
    for line in lines:
        fields = line.split(";")
        assert fields[3] == "0" and int(fields[4], 16) == STREAM, line        # no dynamic smem, the caller's stream
        if len(fields) > 5:
            rowptr = int(fields[5].split()[0], 16)
            assert rowptr >> 36 == 1 + args[1] + 8 * args[2], line          # the operator of (e, direction)


@pytest.mark.parametrize("cid", ["%s-%s" % (dt, k) for dt in ("f32", "f64") for k in ("win-256B", "win-160B",
                                                                                      "win-128B-bwd-e1")])
def test_windowed_hop_runs_chunk_major_then_window_major(cid, launches):
    """One launch per (128-byte column chunk, source window): window w's row offsets, the chunk's columns of src and
    dst, EPI_NONE for window 0 and EPI_ACCUM after it."""
    args = ARGS[cid]
    dt, C, n_win, n_rows = args[0]["plan"][2], args[7], args[0]["plan"][7], args[0]["plan"][0]
    s = 4 if dt == 0 else 8
    base = (1 + args[1] + 8 * args[2]) << 36
    want = []
    for c0 in range(0, C, 128 // s):
        for w in range(n_win):
            want.append((base + WIN_RP32 + 4 * w * (n_rows + 1), SRC + s * c0, DST + s * c0, min(128 // s, C - c0)))
    got = []
    for line in launches[cid][1]:
        rp, src, dst, cc = line.split(";")[5].split()
        got.append((int(rp, 16), int(src, 16), int(dst, 16), int(cc)))
    assert got == want
    epi = [re.search(r",(\d+)>", _short(l).split()[0]).group(1) for l in launches[cid][1]]
    assert epi == [("0" if i % n_win == 0 else "4") for i in range(len(want))]


def test_cases_launch_every_hop_and_row_copy_kernel(launches):
    kernels = library_kernels()
    if kernels is None:
        pytest.skip("no cuobjdump / cu++filt")
    pat = re.compile(r"((?:spmm_hop\w*|bcast_rows_kernel|scatter_rows_kernel)<[^()]*>)")
    compiled = {m.group(1) for k in kernels for m in [pat.search(k)] if m}
    launched = {_short(l).split()[0] for rc, lines in launches.values() for l in lines}
    assert len(compiled) >= 58, sorted(compiled)
    assert compiled == launched, (sorted(compiled - launched), sorted(launched - compiled))
