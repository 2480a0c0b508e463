// Kernels of tools/hop_sector_probe.py: the windowed hop's gather (spmm_hop_multirow_v2_kernel, 4 lanes x 32 bytes per
// 128-byte row chunk, 4-lane row groups, U = 4, evict_last) in four forms, fp32, launched over window-major CSR arrays
// the probe builds itself.  In variants 0 to 2 every window stores its sums (no accumulation).  Variants 0 and 1 differ
// only in the gather loads (both store through the EPI_SCATTER epilogue with no peers: a lane's 32 bytes as two adjacent
// 16-byte stores); variant 2 also stores with the split map, through EPI_NONE (each 16-byte store covers whole sectors).
//   variant 0  adjacent halves: lane cl owns 32 adjacent bytes and loads them as two 16-byte halves (the mapping the
//              library used before LaneMap split the halves)
//   variant 1  adjacent halves, first half only: the same sectors with half the load instructions.  Its sums are wrong
//              by design, which is why it lives here and not in the library
//   variant 2  split halves (LaneMap, the library's mapping): each warp-wide 16-byte load covers whole sectors
//   variant 3  the library's windowed hop: split halves, window 0 stores (EPI_NONE), every later window adds its sums into
//              dst (EPI_ACCUM), by read-add-write when built with -DB200GF_HOP_WIN_RED=0 and by L2 vector reductions
//              when built with the default B200GF_HOP_WIN_RED=1
// Not part of the library:
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -shared -Xcompiler -fPIC tools/hop_sector_probe.cu -o probe.so
#include <algorithm>

#include "../graph-neural-networks_b200/csrc/spmm_kernels.cuh"

namespace b200gf {
// HINT 7 (used by no library kernel): the first 16-byte half of an adjacent-halves lane only, with the library's
// L1::no_allocate + evict_last load; the second half repeats it
template <>
__device__ __forceinline__ Acc<float, 8> load_lane<float, 8, 7, 4>(const float* p, bool lo_ok, bool, uint64_t pol) {
  Acc<float, 4> lo;
  if (lo_ok) lo = load_vec<float, 4, 7>(p, pol); else lo.zero();
  Acc<float, 8> a;
#pragma unroll
  for (int i = 0; i < 4; ++i) { a.v[i] = lo.v[i]; a.v[4 + i] = lo.v[i]; }
  return a;
}
}  // namespace b200gf

using namespace b200gf;

template <int HINT, int MODE, int MODE_REST = MODE>
static int launch(const int32_t* win_rowptr, int n_win, const int32_t* col, const float* val, const float* src, int ld,
                  float* dst, int n_rows, int C, int sm_count, cudaStream_t st) {
  constexpr int VEC = 8, L = 4, GS = 4, U = 4, THREADS = 256, MINB = 4;
  auto kern = spmm_hop_multirow_v2_kernel<float, int32_t, VEC, L, GS, U, THREADS, MINB, HINT, MODE>;
  auto rest = spmm_hop_multirow_v2_kernel<float, int32_t, VEC, L, GS, U, THREADS, MINB, HINT, MODE_REST>;
  constexpr int rows_per_block = (THREADS / 32) * (32 / GS);
  // one resident wave of variant 0's occupancy for all three: the first-half-only kernel needs fewer registers, and more
  // resident warps would time occupancy, not loads
  int occ = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(
          &occ, spmm_hop_multirow_v2_kernel<float, int32_t, VEC, L, GS, U, THREADS, MINB, 3, EPI_SCATTER>, THREADS, 0) != cudaSuccess)
    return -1;
  const int64_t blocks = std::min<int64_t>((n_rows + rows_per_block - 1) / rows_per_block, (int64_t)sm_count * std::max(occ, 1));
  for (int c0 = 0; c0 < C; c0 += 32)
    for (int w = 0; w < n_win; ++w) {
      const int32_t* rp = win_rowptr + (int64_t)w * (n_rows + 1);
      if (w == 0)
        kern<<<(unsigned)blocks, THREADS, 0, st>>>(rp, col, val, src + c0, ld, dst + c0, ld, n_rows, std::min(32, C - c0),
                                                   ScatterParam<float, MODE>{});
      else
        rest<<<(unsigned)blocks, THREADS, 0, st>>>(rp, col, val, src + c0, ld, dst + c0, ld, n_rows, std::min(32, C - c0),
                                                   ScatterParam<float, MODE_REST>{});
    }
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

// one windowed hop: every (128-byte chunk, window) launch of `variant`; 0 on success
extern "C" int probe_window_hop(int variant, const int32_t* win_rowptr, int n_win, const int32_t* col, const float* val,
                                const float* src, int ld, float* dst, int n_rows, int C, int sm_count, void* stream) {
  if (C % 8 || ld % 8 || C > ld) return -1;
  const cudaStream_t st = (cudaStream_t)stream;
  if (variant == 0) return launch<3, EPI_SCATTER>(win_rowptr, n_win, col, val, src, ld, dst, n_rows, C, sm_count, st);
  if (variant == 1) return launch<7, EPI_SCATTER>(win_rowptr, n_win, col, val, src, ld, dst, n_rows, C, sm_count, st);
  if (variant == 2) return launch<3, EPI_NONE>(win_rowptr, n_win, col, val, src, ld, dst, n_rows, C, sm_count, st);
  if (variant == 3) return launch<3, EPI_NONE, EPI_ACCUM>(win_rowptr, n_win, col, val, src, ld, dst, n_rows, C, sm_count, st);
  return -1;
}
