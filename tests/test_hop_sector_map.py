"""The lane map of the wide-row hop kernels (csrc/spmm_kernels.cuh: LaneMap, split_lanes).

A 32-byte lane loads and stores its columns as two 16-byte halves.  With the local epilogues (EPI_NONE, EPI_ACCUM) the
first halves of a row chunk's L lanes are the chunk's first L*16 bytes and the second halves the rest, so that every
warp-wide 16-byte access of a lane group covers whole 32-byte sectors; the NVLink epilogues keep a lane's 32 bytes
adjacent.  The CPU test checks the map the kernels use, compiled host-side: every column of a chunk belongs to exactly
one live (lane, half), nothing at or past the padded width is touched, and each access covers whole sectors.  The GPU
tests run the partial last chunks in which only some lanes' second halves are live, on every wide-row kernel, with the
checks of tests/dispatch_harness.py (a CPU test holds their kernel regexes and case ids to the checks
tests/test_dispatch_tables.py runs on the registered tables), and the headline graph's hops (N = 1M, 64 columns) against the componentwise fp64
bound, windows on and off, bit-identical across two runs.
"""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import lsigf_oracle as orc
import test_hop_windows as thw
import test_kernel_dispatch as tkd
import test_spmm_l2_chunks as tlc
from dispatch_harness import (F32, F64, NPD, SENT, _bits, _check, _lib, check_case, child_traced, kernel_names,
                              library_kernels)

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "graph-neural-networks_b200", "csrc")

_HELPER = r"""
#include "spmm_kernels.cuh"
using namespace b200gf;

template <int VEC, int L, bool SPLIT>
static int put(int cl, int* lo, int* hi) {
  *lo = LaneMap<VEC, L, SPLIT>::lo(cl);
  *hi = LaneMap<VEC, L, SPLIT>::HI;
  return 0;
}
template <int VEC, int L>
static int by_mode(int mode, int cl, int* lo, int* hi) {
  switch (mode) {
    case EPI_NONE: return put<VEC, L, split_lanes<EPI_NONE>>(cl, lo, hi);
    case EPI_SCATTER: return put<VEC, L, split_lanes<EPI_SCATTER>>(cl, lo, hi);
    case EPI_BCAST: return put<VEC, L, split_lanes<EPI_BCAST>>(cl, lo, hi);
    case EPI_GRID: return put<VEC, L, split_lanes<EPI_GRID>>(cl, lo, hi);
    case EPI_ACCUM: return put<VEC, L, split_lanes<EPI_ACCUM>>(cl, lo, hi);
  }
  return -1;
}
template <int VEC>
static int by_lanes(int L, int mode, int cl, int* lo, int* hi) {
  switch (L) {
    case 2: return by_mode<VEC, 2>(mode, cl, lo, hi);
    case 4: return by_mode<VEC, 4>(mode, cl, lo, hi);
    case 8: return by_mode<VEC, 8>(mode, cl, lo, hi);
    case 16: return by_mode<VEC, 16>(mode, cl, lo, hi);
    case 32: return by_mode<VEC, 32>(mode, cl, lo, hi);
  }
  return -1;
}
// column of lane cl's first half in its row chunk, and the second half's offset from it
extern "C" int lane_map(int vec, int L, int mode, int cl, int* lo, int* hi) {
  if (vec == 8) return by_lanes<8>(L, mode, cl, lo, hi);
  if (vec == 4) return by_lanes<4>(L, mode, cl, lo, hi);
  return -1;
}
"""

# (L, VEC) of every wide-row instantiation: spmm_hop_v2_kernel L = 4, 8, 16, 32; spmm_hop_multirow_v2_kernel L = 2
# (64-byte rows) and L = 4 (source windows); VEC = 8 fp32 / 4 fp64 columns per 32-byte lane
GEOMETRIES = [(L, vec) for L in (2, 4, 8, 16, 32) for vec in (8, 4)]
EPI_NONE, EPI_SCATTER, EPI_BCAST, EPI_GRID, EPI_ACCUM = range(5)


@pytest.fixture(scope="module")
def lane_map(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    d = tmp_path_factory.mktemp("lane_map")
    src, so = d / "lane_map.cu", d / "lane_map.so"
    src.write_text(_HELPER)
    out = subprocess.run([nvcc, "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-I", CSRC, str(src), "-o", str(so)],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    h = ctypes.CDLL(str(so))

    def get(vec, L, mode, cl):
        lo, hi = ctypes.c_int(), ctypes.c_int()
        assert h.lane_map(vec, L, mode, cl, ctypes.byref(lo), ctypes.byref(hi)) == 0
        return lo.value, hi.value
    return get


def test_lane_halves_cover_each_column_once_in_whole_sectors(lane_map):
    for L, vec in GEOMETRIES:
        H, esz = vec // 2, 32 // vec                  # columns per half, bytes per column
        for mode in (EPI_NONE, EPI_SCATTER, EPI_BCAST, EPI_GRID, EPI_ACCUM):
            split = mode in (EPI_NONE, EPI_ACCUM)
            halves = []
            for cl in range(L):
                lo, hi = lane_map(vec, L, mode, cl)
                if split:
                    assert (lo, hi) == (cl * H, L * H), (L, vec, mode, cl)
                else:
                    assert (lo, hi) == (cl * vec, H), (L, vec, mode, cl)   # a lane's 32 bytes stay adjacent
                halves += [(cl, 0, lo), (cl, 1, lo + hi)]
            # every padded width a chunk can end at: one to L lanes' worth of columns
            for Cp in range(vec, L * vec + 1, vec):
                owner = np.zeros(L * vec, np.int64)
                for cl, h, c in halves:
                    live = c < Cp                   # the kernels' predicate: the half starts below the padded width
                    if live:
                        assert c + H <= Cp, "a live half reaches past the padded width"
                        owner[c:c + H] += 1
                    if h == 1 and live:
                        assert lane_map(vec, L, mode, cl)[0] < Cp, "second half live without the first"
                assert (owner[:Cp] == 1).all() and (owner[Cp:] == 0).all(), (L, vec, mode, Cp)
                if not split:
                    continue
                for h in (0, 1):                    # one warp-wide 16-byte access of a lane group
                    touched = np.zeros(L * vec * esz, bool)
                    for cl, hh, c in halves:
                        if hh == h and c < Cp:
                            touched[c * esz:(c + H) * esz] = True
                    sectors = touched.reshape(-1, 32)
                    assert (sectors.all(axis=1) | ~sectors.any(axis=1)).all(), "partial sector: %s" % ((L, vec, Cp, h),)
                    if L >= 8 and Cp == L * vec:
                        lines = touched.reshape(-1, 128)
                        assert touched.sum() == L * 16 and (lines.all(axis=1) | ~lines.any(axis=1)).all(), \
                            "whole 128-byte lines: %s" % ((L, vec, h),)


# ------------------------------------------------------------------------------------------------------ GPU rows
def _plain(dtype, L):
    return r"spmm_hop_v2_kernel<%s,int,%d,%d,4,256,%d,3,0," % ("float" if dtype == F32 else "double", 8 if dtype == F32 else 4,
                                                             L, 4 if dtype == F32 else 3)


def _rows():
    """Last row chunks in which some lanes' second halves are live and the others' are not (padded width in the chunk's
    second half), where the existing tables have none: (padded C) mod (chunk width) = 40 of 64 fp32 columns (L = 8),
    24 of 32 fp64 (L = 8), 176 of 256 fp32 (L = 32), 24 of 32 fp32 and 12 of 16 fp64 (L = 4, forced by the plan's L2
    size, and on the source-window path).  Every row's ld exceeds the padded width by one 32-byte vector, so the canary
    columns [padded(C), ld) check that no live half reaches past the padded width."""
    rows = [
        ("sector-hop-f32-C37-ld48-L8", tkd._hop_case(F32, 37, 48), [_plain(F32, 8)]),
        ("sector-hop-f64-C21-ld28-L8", tkd._hop_case(F64, 21, 28), [_plain(F64, 8)]),
        ("sector-hop-f32-C1200-ld1208-L32", tkd._hop_case(F32, 1200, 1208), [_plain(F32, 32)]),
        ("sector-chunk-f32-C88-ld96-L4", tlc._hop_case(F32, 88, 96, 4), [_plain(F32, 4)]),
        ("sector-chunk-f64-C44-ld48-L4", tlc._hop_case(F64, 44, 48, 4), [_plain(F64, 4)]),
    ]
    for dt, C, ld in ((F32, 88, 96), (F64, 44, 48)):
        rows.append(("sector-win-%s-C%d-ld%d-R1100" % ("f32" if dt == F32 else "f64", C, ld), thw._hop_case(dt, C, ld, 1100),
                     [thw._win(dt, 0), thw._win(dt, 4)]))
    return rows


CASES = _rows()


def test_rows_name_hop_kernels_of_the_library_under_unique_ids():
    """The checks tests/test_dispatch_tables.py runs on the registered tables, for this one: every regex names a kernel of
    csrc/spmm_kernels.cuh and matches a kernel compiled into the library, and no case id is used twice here or by a
    registered table."""
    import test_dispatch_tables as tdt
    hop = tdt._package_kernels()["csrc/spmm_kernels.cuh"]
    assert kernel_names(CASES) <= hop, sorted(kernel_names(CASES) - hop)
    ids = [cid for cid, _, _ in CASES]
    assert len(set(ids)) == len(ids), ids
    others = {cid for m in tdt.TABLES for cid, _, _ in tdt._rows(m)}
    assert not set(ids) & others, sorted(set(ids) & others)
    names = library_kernels()
    if names is None:
        pytest.skip("cuobjdump / cu++filt or the library not available")
    for cid, _, ks in CASES:
        for k in ks:
            assert any(re.search(k, n) for n in names), (cid, k)

traced = child_traced("test_hop_sector_map", "CASES")


@pytest.mark.gpu
@pytest.mark.parametrize("cid,fn,kernels", CASES, ids=[c[0] for c in CASES])
def test_partial_second_halves(cid, fn, kernels, traced):
    check_case(cid, fn, kernels, traced[cid])


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
def test_headline_hops_within_bound_and_repeatable(dtype):
    """bench.py's headline graph (N = 1M, degree 32, 64 columns): both hop directions, with the plan's default window
    copy and without it, within the componentwise fp64 bound, and bit-identical across two runs."""
    import gnn_b200
    from gnn_b200 import graphs
    cabi, lib = _lib()
    N, C = 1_000_000, 64
    npd = NPD[dtype]
    gso = graphs.er_gso(N, 32, seed=1, E=1).astype(dtype)
    plan = gnn_b200.gso.Plan.from_host_csr(gso.csr, N, dtype, torch.device("cuda"))
    rows = plan.info(8)
    assert rows > 0, "the headline graph takes the windowed hop by default"
    assert plan.info(6) == 1, "symmetric GSO: both directions gather with the same operator"
    r, c, v = gso.csr[0]
    m = sp.csr_matrix((np.asarray(v, npd).astype(np.float64), c, r), shape=(N, N))
    X = torch.randn(N, C, generator=torch.Generator().manual_seed(5), dtype=torch.float64).to(dtype)
    Xd = X.double().numpy()
    ref = m @ Xd
    bound = orc.dot_bound(np.maximum(np.diff(m.indptr)[:, None], 1), abs(m) @ np.abs(Xd), npd)
    src = X.cuda()
    for windows in (rows, 0):
        _check(lib.b200gf_plan_set_hop_windows(plan.handle, windows))
        for direction in (cabi.HOP_FWD, cabi.HOP_BWD):
            outs = []
            for _ in range(2):
                dst = torch.full((N, C), SENT, dtype=dtype, device="cuda")
                _check(lib.b200gf_hop(plan.handle, 0, direction, src.data_ptr(), C, dst.data_ptr(), C, C,
                                      torch.cuda.current_stream().cuda_stream))
                outs.append(dst)
            torch.cuda.synchronize()
            assert torch.equal(_bits(outs[0]), _bits(outs[1])), "windows %d, direction %d: two runs differ" % (windows, direction)
            v = orc.bound_violation(outs[0].double().cpu().numpy(), ref, bound)
            print("windows %d direction %d: worst error / bound %.3g" % (windows, direction, v))
            assert v <= 1.0, "windows %d, direction %d: error %.3g x its bound" % (windows, direction, v)
