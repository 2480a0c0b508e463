// One graph shift ("hop") of the LSIGF path:  dst[r, :] = sum_j A[r, j] * src[j, :]
// with A a CSR gather operator (S_e^T for the forward x·S of reference graphML.py:159, S_e for backward)
// and src/dst node-major [rows, ld] feature matrices.  This replaces the reference's dense broadcast-batched
// GEMM torch.matmul(x, S) and is the HBM-bound kernel the roofline in bench.py is quoted on.
//
// Mapping (sm_90a, 132 SMs) — details in spmm_kernels.cuh:
//   * rows of more than 128 bytes: one warp per (row, column chunk), chunk-major grid-stride order (keeps the gathered
//     column slab L2-resident when it fits), L lanes x 16-byte vectors per neighbour row, 32/L neighbours per LDG.128,
//     U loads in flight per lane, col/val read once per row and broadcast by SHFL, 48 resident warps per SM,
//     L2 evict_last policy on the gathered rows;
//   * narrower rows: several rows per warp (spmm_hop_multirow_kernel);
//   * operators with a window-major copy (million-node graphs): one launch per (128-byte column chunk, source window),
//     each adding its window's sums into dst (launch_windows);
//   * optional epilogue: the computed row slice is also stored over NVLink into a peer's buffer (b200gf_hop_scatter).
#include <cstdlib>
#include <cstring>

#include "common.cuh"
#include "spmm_kernels.cuh"

// L2 policy of the gathered rows in the v2 kernel (spmm_kernels.cuh HINT codes)
#ifndef B200GF_HOP_L2_HINT
#define B200GF_HOP_L2_HINT 3
#endif
#ifndef B200GF_HOP_L2_FRAC
#define B200GF_HOP_L2_FRAC 1.0f
#endif
// geometry and L2 policy of the windowed hop (launch_windows), for tools/hop_window_bench.py's sweep
#ifndef B200GF_HOP_WIN_GS
#define B200GF_HOP_WIN_GS 4
#endif
#ifndef B200GF_HOP_WIN_U
#define B200GF_HOP_WIN_U 4
#endif
#ifndef B200GF_HOP_WIN_HINT
#define B200GF_HOP_WIN_HINT 3
#endif

namespace b200gf {

template <typename T>
static ScatterArgs<T> make_scatter(const ScatterHost* sh) {
  ScatterArgs<T> sc{};
  if (sh && sh->n_peers > 0) {
    for (int i = 0; i < sh->n_peers; ++i) sc.peer[i] = reinterpret_cast<T*>(sh->peer[i]);
    sc.rows_per_peer = sh->rows_per_peer; sc.out_ld = sh->out_ld; sc.out_col = sh->out_col;
    sc.stride_b = sh->stride_b; sc.gl = sh->gl; sc.n_peers = sh->n_peers;
  }
  return sc;
}

template <typename T>
static BcastArgs<T> make_bcast(const BcastHost* bh) {
  BcastArgs<T> bc{};
  for (int i = 0; i < bh->n_peers; ++i) bc.peer[i] = reinterpret_cast<T*>(bh->peer[i]);
  bc.mc = reinterpret_cast<T*>(bh->mc);
  bc.row0 = bh->row0; bc.out_ld = bh->out_ld; bc.n_peers = bh->n_peers;
  return bc;
}

// Library configuration (tools/spmm_sweep.cu explores the alternatives): 256 threads, registers capped for 6 resident
// blocks/SM (48 warps: the kernel is latency-bound below that), gathered rows loaded with an L2 evict_last policy and no
// L1 allocation (a sticky subset of the gathered slab stays in L2), no next-row prefetch (it costs registers).
template <typename T, int VEC, int L, int U>
static int launch_one(int sm_count, const CsrDev& A, int64_t n_rows, const T* src, int64_t src_ld, T* dst,
                      int64_t dst_ld, int C, cudaStream_t st, const ScatterHost* sh) {
  constexpr int THREADS = 256, MINB = sizeof(T) == 4 ? 6 : 4, HINT = 3;
  constexpr bool PF = false;
  auto kern = spmm_hop_kernel<T, VEC, L, U, THREADS, MINB, HINT, PF>;
  const int n_chunks = (C + L * VEC - 1) / (L * VEC);
  const int64_t n_items = n_rows * n_chunks;
  if (n_items == 0) return B200GF_OK;
  const int wpb = THREADS / 32;
  int occ = 0;
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, THREADS, 0));
  if (occ < 1) occ = 1;
  int64_t blocks = (n_items + wpb - 1) / wpb;
  const int64_t cap = (int64_t)sm_count * occ;  // one resident wave: persistent warps stride over the items
  if (blocks > cap) blocks = cap;
  kern<<<(unsigned)blocks, THREADS, 0, st>>>(A.rowptr, A.col, reinterpret_cast<const T*>(A.val), src, src_ld, dst,
                                             dst_ld, n_rows, C, n_chunks, 1.0f, make_scatter<T>(sh));
  LAUNCH_CHECK();
  return B200GF_OK;
}

// narrow rows (<= 128 bytes): several rows per warp (spmm_hop_multirow_kernel), geometry from the small-C sweep of
// tools/spmm_sweep.cu
template <typename T, int VEC, int L, int GS, int U, int MINB>
static int launch_multirow(int sm_count, const CsrDev& A, int64_t n_rows, const T* src, int64_t src_ld, T* dst,
                           int64_t dst_ld, int C, cudaStream_t st, const ScatterHost* sh) {
  constexpr int THREADS = 256, HINT = 3;
  auto kern = spmm_hop_multirow_kernel<T, VEC, L, GS, U, THREADS, MINB, HINT>;
  if (n_rows == 0) return B200GF_OK;
  constexpr int rows_per_block = (THREADS / 32) * (32 / GS);
  int occ = 0;
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, THREADS, 0));
  if (occ < 1) occ = 1;
  int64_t blocks = (n_rows + rows_per_block - 1) / rows_per_block;
  const int64_t cap = (int64_t)sm_count * occ;
  if (blocks > cap) blocks = cap;
  kern<<<(unsigned)blocks, THREADS, 0, st>>>(A.rowptr, A.col, reinterpret_cast<const T*>(A.val), src, src_ld, dst,
                                             dst_ld, n_rows, C, make_scatter<T>(sh));
  LAUNCH_CHECK();
  return B200GF_OK;
}

// Round-2 kernel (spmm_kernels.cuh: spmm_hop_v2_kernel): 32-byte lanes loaded as two 16-byte halves, 32-bit index
// arithmetic.  L lanes x 32 bytes cover a row chunk: the lanes' first halves its first L*16 bytes, their second halves the
// rest (LaneMap; the NVLink epilogues keep a lane's 32 bytes adjacent), so every LDG.128 / STG.128 of a lane group covers
// whole 32-byte sectors; 32/L neighbours per warp-wide load, U loads in flight per lane; 4 blocks of 256 threads per SM
// (64 registers); column chunks on blockIdx.y.
template <typename T, int L, int SCATTER>
static int launch_v2(int sm_count, const CsrDev& A, int64_t n_rows, const T* src, int64_t src_ld, T* dst, int64_t dst_ld,
                     int C, cudaStream_t st, const ScatterHost* sh, const BcastHost* bh) {
  constexpr int VEC = 32 / sizeof(T), U = 4, THREADS = 256, MINB = sizeof(T) == 4 ? 4 : 3, HINT = B200GF_HOP_L2_HINT;
  // streaming stores (SH = 1): the result rows are read by the next launch, not by this one, so at normal priority they
  // only displace gathered lines from the L2 (2.74 against 2.78 ms per hop at N = 1M, 64 fp32 columns)
  auto kern = spmm_hop_v2_kernel<T, int32_t, VEC, L, U, THREADS, MINB, HINT, SCATTER, 1>;
  if (n_rows == 0) return B200GF_OK;
  const int n_chunks = (C + L * VEC - 1) / (L * VEC);
  if (n_chunks > 65535) return B200GF_EUNSUPPORTED;
  const int wpb = THREADS / 32;
  int occ = 0;
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, THREADS, 0));
  if (occ < 1) occ = 1;
  int64_t blocks = (n_rows + wpb - 1) / wpb;
  // one resident wave per chunk when there is a single chunk; with several chunks each chunk gets its own wave-sized
  // slice of the grid so that the block scheduler runs them chunk-major
  const int64_t cap = (int64_t)sm_count * occ;
  if (blocks > cap) blocks = cap;
  ScatterParam<T, SCATTER> sp{};
  if constexpr (SCATTER == EPI_SCATTER) sp.a = make_scatter<T>(sh);
  if constexpr (SCATTER == EPI_BCAST) sp.a = make_bcast<T>(bh);
  if constexpr (SCATTER == EPI_GRID) { sp.s = make_scatter<T>(sh); sp.a = make_bcast<T>(bh); }
  kern<<<dim3((unsigned)blocks, (unsigned)n_chunks), THREADS, 0, st>>>(A.rowptr32, A.col, reinterpret_cast<const T*>(A.val),
                                                                      src, (int)src_ld, dst, (int)dst_ld, (int)n_rows, C,
                                                                      B200GF_HOP_L2_FRAC, sp);
  LAUNCH_CHECK();
  return B200GF_OK;
}

template <typename T, int L>
static int launch_v2_sc(int sm_count, const CsrDev& A, int64_t n_rows, const T* src, int64_t src_ld, T* dst,
                        int64_t dst_ld, int C, cudaStream_t st, const ScatterHost* sh, const BcastHost* bh) {
  if (bh && sh) return launch_v2<T, L, EPI_GRID>(sm_count, A, n_rows, src, src_ld, dst, dst_ld, C, st, sh, bh);
  if (bh) return launch_v2<T, L, EPI_BCAST>(sm_count, A, n_rows, src, src_ld, dst, dst_ld, C, st, nullptr, bh);
  if (sh && sh->n_peers > 0) {
    // the feature-sharded scatter sizes its chunks by row width alone (hop_chunk_lanes without an L2 budget), so L >= 8:
    // no 4-lane scatter kernel is compiled
    if constexpr (L >= 8) return launch_v2<T, L, EPI_SCATTER>(sm_count, A, n_rows, src, src_ld, dst, dst_ld, C, st, sh, nullptr);
    else return B200GF_EUNSUPPORTED;
  }
  return launch_v2<T, L, EPI_NONE>(sm_count, A, n_rows, src, src_ld, dst, dst_ld, C, st, nullptr, nullptr);
}

// 64-byte rows (C = 16 floats / 8 doubles) with 32-byte lanes: two lanes per neighbour row, 8-lane row groups, two loads in
// flight per lane; rows of C = 8 stay on spmm_hop_multirow_kernel.
template <typename T, int SCATTER>
static int launch_multirow_v2(int sm_count, const CsrDev& A, int64_t n_rows, const T* src, int64_t src_ld, T* dst,
                              int64_t dst_ld, int C, cudaStream_t st, const ScatterHost* sh, const BcastHost* bh = nullptr) {
  constexpr int VEC = 32 / sizeof(T), L = 2, GS = 8, U = 2, THREADS = 256, MINB = sizeof(T) == 4 ? 4 : 3, HINT = 3;
  auto kern = spmm_hop_multirow_v2_kernel<T, int32_t, VEC, L, GS, U, THREADS, MINB, HINT, SCATTER>;
  if (n_rows == 0) return B200GF_OK;
  constexpr int rows_per_block = (THREADS / 32) * (32 / GS);
  int occ = 0;
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, THREADS, 0));
  if (occ < 1) occ = 1;
  int64_t blocks = (n_rows + rows_per_block - 1) / rows_per_block;
  const int64_t cap = (int64_t)sm_count * occ;
  if (blocks > cap) blocks = cap;
  ScatterParam<T, SCATTER> sp{};
  if constexpr (SCATTER == EPI_SCATTER) sp.a = make_scatter<T>(sh);
  if constexpr (SCATTER == EPI_GRID) { sp.s = make_scatter<T>(sh); sp.a = make_bcast<T>(bh); }
  kern<<<(unsigned)blocks, THREADS, 0, st>>>(A.rowptr32, A.col, reinterpret_cast<const T*>(A.val), src, (int)src_ld, dst,
                                             (int)dst_ld, (int)n_rows, C, sp);
  LAUNCH_CHECK();
  return B200GF_OK;
}

// Lane count L (chunk = L x 32 bytes of each row) of spmm_hop_v2_kernel for rows of nw 32-byte vectors.  The kernel runs
// the chunks chunk-major, so what the resident warps gather from at any time is one chunk of every source row, n_src * L
// * 32 bytes.  By default the row width alone sets L (at most 32 lanes, 1 KB chunks).  When that chunk does not fit the
// L2, the widest narrower chunk (L = 16, 8 or 4) that fits is used: every extra chunk re-reads col/val once, far fewer
// bytes than gathering rows that miss the L2 from HBM.  L >= 4 keeps a chunk whole 128-byte L2 lines.  When not even
// L = 4 fits, the default stays.
// The budget is the whole L2: on an H100 (50 MB L2) chunks of 51.2 MB ran as fast as chunks of 25.6 MB (N = 100k,
// 2048 fp32 columns) or faster (N = 200k, 1024 fp32 columns: 3.51 against 3.58 ms per hop), while 102 MB chunks were
// 11 % slower.
// When not even L = 4 fits, two 128-byte chunks of a 256-byte row still raise the share of gathers that hit the L2 if
// the gathers spread over the whole source (`spread`) and a chunk is at most 3x the L2: 2.69 against 2.74 ms per hop
// at N = 1M with 64 fp32 columns (128 MB chunks).  They cost time at 5x the L2 (N = 2M: 6.16 against 5.92 ms), on a
// graph numbered community by community, whose gathers stay near the diagonal (2.19 against 2.17 ms), and as four
// chunks of a 512-byte row (64 fp64 columns: 5.80 against 5.70 ms), which read col/val four times.
static int hop_chunk_lanes(int64_t n_src, int nw, int64_t l2_bytes, bool spread) {
  const int L0 = nw <= 8 ? 8 : nw <= 16 ? 16 : 32;
  const auto fits = [&](int L) { return n_src * 32 * (L < nw ? L : nw) <= l2_bytes; };
  if (fits(L0)) return L0;
  for (int L = L0 / 2; L >= 4; L /= 2)
    if (fits(L)) return L;
  if (spread && nw > 4 && nw <= 8 && n_src * 32 * 4 <= 3 * l2_bytes) return 4;
  return L0;
}

// Windowed hop over rows of at least 128 bytes (CsrDev::win_*): one launch per (128-byte column chunk, source window),
// chunk-major then window-major on the stream, so that the gathers of a launch read one window's rows of one chunk, an
// L2-sized range.  Window 0 stores its sums, every later window adds its sums into dst (EPI_ACCUM: fp32 with L2 vector
// reductions, fp64 by read-add-write).  Four 32-byte lanes
// own a row's chunk and a warp works on 32 / GS rows (spmm_hop_multirow_v2_kernel); a window holds few entries per row,
// so that with GS = 4 a row needs no cross-lane fold.  Written columns: [0, padded(C)), as the plain hop.
template <typename T, int MODE>
static int launch_window(int sm_count, const int32_t* rowptr, const CsrDev& A, int64_t n_rows, const T* src,
                         int64_t src_ld, T* dst, int64_t dst_ld, int C, cudaStream_t st) {
  constexpr int VEC = 32 / sizeof(T), L = 4, GS = B200GF_HOP_WIN_GS, U = B200GF_HOP_WIN_U, THREADS = 256;
  constexpr int MINB = sizeof(T) == 4 ? 4 : 3, HINT = B200GF_HOP_WIN_HINT;
  auto kern = spmm_hop_multirow_v2_kernel<T, int32_t, VEC, L, GS, U, THREADS, MINB, HINT, MODE>;
  constexpr int rows_per_block = (THREADS / 32) * (32 / GS);
  int occ = 0;
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, THREADS, 0));
  if (occ < 1) occ = 1;
  const int64_t blocks = std::min<int64_t>((n_rows + rows_per_block - 1) / rows_per_block, (int64_t)sm_count * occ);
  kern<<<(unsigned)blocks, THREADS, 0, st>>>(rowptr, A.win_col, reinterpret_cast<const T*>(A.win_val), src, (int)src_ld,
                                             dst, (int)dst_ld, (int)n_rows, C, ScatterParam<T, MODE>{});
  LAUNCH_CHECK();
  return B200GF_OK;
}

template <typename T>
static int launch_windows(int sm_count, const CsrDev& A, int64_t n_rows, const T* src, int64_t src_ld, T* dst,
                          int64_t dst_ld, int C, cudaStream_t st) {
  if (n_rows == 0) return B200GF_OK;
  constexpr int CW = 128 / sizeof(T);   // columns per chunk
  for (int c0 = 0; c0 < C; c0 += CW) {
    const int Cc = std::min(CW, C - c0);
    for (int w = 0; w < A.n_win; ++w) {
      const int32_t* rp = A.win_rowptr32 + (int64_t)w * (n_rows + 1);
      const int rc = w == 0 ? launch_window<T, EPI_NONE>(sm_count, rp, A, n_rows, src + c0, src_ld, dst + c0, dst_ld, Cc, st)
                            : launch_window<T, EPI_ACCUM>(sm_count, rp, A, n_rows, src + c0, src_ld, dst + c0, dst_ld, Cc, st);
      if (rc) return rc;
    }
  }
  return B200GF_OK;
}

// Rows R per source window of the default window-major operator copy (b200gf_plan_create), 0 for none: only when not
// even a 128-byte chunk of the source fits the L2 (hop_chunk_lanes has no chunk left to narrow), the gathers spread over
// the whole source, and the source splits into at most 8 windows.  Windows of 5/8 of the L2 (256 000 rows, 32.8 MB on an
// H100): 250k-row windows ran the N = 1M, 64-column fp32 hop in 2.43 against 2.56 ms, 200k and 333k rows in 2.47 and
// 2.44, 125k rows (16 MB) in 2.65.  Every window after the first re-reads and re-writes the destination and the window
// offsets, so the gain shrinks as windows are added: W = 4 (N = 1M) gained 5 % per hop, W = 8 (N = 2M) 1.4 % (5.67
// against 5.60 ms); more windows were not measured and are not taken.  Re-measured once fp32 windows added in the L2
// instead of reading dst back: R = 250k still ran er1m fastest (1.81 ms; 200k 1.88, 333k 1.96, 125k 2.38).  At N = 2M
// 333k-row windows (W = 6) ran 5.19 against 5.49 ms, with read-add-write as well (5.27 against 5.51), but they lose at
// N = 1M, so the rule stays.
int64_t hop_window_rows(int64_t n_src, int64_t l2_bytes, bool spread) {
  if (!spread || l2_bytes <= 0 || n_src * 128 <= l2_bytes) return 0;
  const int64_t R = l2_bytes * 5 / 8 / 128;
  return R > 0 && n_src <= 8 * R ? R : 0;
}

template <typename T>
static int launch_typed(int sm_count, int64_t l2_bytes, const CsrDev& A, int64_t n_rows, const void* src_, int64_t src_ld,
                        void* dst_, int64_t dst_ld, int C, cudaStream_t st, const ScatterHost* sh, const BcastHost* bh) {
  constexpr int VEC = 16 / sizeof(T);
  const T* src = reinterpret_cast<const T*>(src_);
  T* dst = reinterpret_cast<T*>(dst_);
  if (bh) {
    // fused all-gather epilogue (EPI_BCAST), or all-gather + scatter (EPI_GRID, when `sh` is given too): v2 kernels only
    // (32-byte aligned rows on every side, 32-bit offsets, rows of at least 64 bytes)
    constexpr int VWb = 32 / sizeof(T);
    const int Cwb = (C + VWb - 1) / VWb * VWb;
    const bool grid = sh && sh->n_peers > 0;
    bool ok = A.rowptr32 != nullptr && src_ld % VWb == 0 && Cwb <= src_ld && (reinterpret_cast<uintptr_t>(src) & 31) == 0 &&
              src_ld <= INT32_MAX && n_rows <= INT32_MAX && Cwb >= 2 * VWb;
    if (bh->n_peers > 0) ok = ok && Cwb <= bh->out_ld && bh->out_ld % VWb == 0;
    for (int i = 0; i < bh->n_peers; ++i) ok = ok && (reinterpret_cast<uintptr_t>(bh->peer[i]) & 31) == 0;
    ok = ok && (reinterpret_cast<uintptr_t>(bh->mc) & 31) == 0;
    if (grid) ok = ok && sh->gl % VWb == 0 && sh->out_ld % VWb == 0 && sh->out_col % VWb == 0 && sh->stride_b % VWb == 0;
    if (!grid && bh->n_peers <= 0) ok = false;
    if (dst_) ok = ok && dst_ld % VWb == 0 && Cwb <= dst_ld && (reinterpret_cast<uintptr_t>(dst_) & 31) == 0 && dst_ld <= INT32_MAX;
    if (!ok) return B200GF_EUNSUPPORTED;
    const int nwb = Cwb / VWb;
    if (nwb == 2) {
      if (!grid) return B200GF_EUNSUPPORTED;        // 64-byte rows: only the grid epilogue is instantiated for the multi-row kernel
      return launch_multirow_v2<T, EPI_GRID>(sm_count, A, n_rows, src, src_ld, dst, dst_ld, C, st, sh, bh);
    }
    if (nwb <= 4) return launch_v2_sc<T, 4>(sm_count, A, n_rows, src, src_ld, dst, dst_ld, C, st, grid ? sh : nullptr, bh);
    if (nwb <= 8) return launch_v2_sc<T, 8>(sm_count, A, n_rows, src, src_ld, dst, dst_ld, C, st, grid ? sh : nullptr, bh);
    if (nwb <= 16) return launch_v2_sc<T, 16>(sm_count, A, n_rows, src, src_ld, dst, dst_ld, C, st, grid ? sh : nullptr, bh);
    return launch_v2_sc<T, 32>(sm_count, A, n_rows, src, src_ld, dst, dst_ld, C, st, grid ? sh : nullptr, bh);
  }
  const int Cv = (C + VEC - 1) / VEC * VEC;
  const bool vec_ok = (src_ld % VEC == 0) && (dst_ld % VEC == 0) && (Cv <= src_ld) && (Cv <= dst_ld) &&
                      ((reinterpret_cast<uintptr_t>(src) & 15) == 0) && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0);
  if (!vec_ok) {
    if (sh && sh->n_peers > 0) return B200GF_EUNSUPPORTED;  // the fused scatter needs the 16-byte vector path
    return launch_one<T, 1, 32, 4>(sm_count, A, n_rows, src, src_ld, dst, dst_ld, C, st, nullptr);
  }
  if (sh && sh->n_peers > 0 && (sh->gl % VEC != 0 || sh->out_ld % VEC != 0 || sh->out_col % VEC != 0 || sh->stride_b % VEC != 0))
    return B200GF_EUNSUPPORTED;
  const int nv = Cv / VEC;  // 16-byte vectors per row
  constexpr int MB = sizeof(T) == 4 ? 6 : 4;
  {
    // exactly-64-byte rows: the 32-byte-lane multi-row kernel when its preconditions hold
    constexpr int VW2 = 32 / sizeof(T);
    bool w2 = nv > 2 && nv <= 4 && A.rowptr32 != nullptr && src_ld % VW2 == 0 && dst_ld % VW2 == 0 && 2 * VW2 <= src_ld &&
              2 * VW2 <= dst_ld && (reinterpret_cast<uintptr_t>(src) & 31) == 0 && (reinterpret_cast<uintptr_t>(dst) & 31) == 0 &&
              src_ld <= INT32_MAX && dst_ld <= INT32_MAX && n_rows <= INT32_MAX;
    if (sh && sh->n_peers > 0)
      w2 = w2 && sh->gl % VW2 == 0 && sh->out_ld % VW2 == 0 && sh->out_col % VW2 == 0 && sh->stride_b % VW2 == 0;
    if (w2) {
      if (sh && sh->n_peers > 0) return launch_multirow_v2<T, EPI_SCATTER>(sm_count, A, n_rows, src, src_ld, dst, dst_ld, C, st, sh);
      return launch_multirow_v2<T, EPI_NONE>(sm_count, A, n_rows, src, src_ld, dst, dst_ld, C, st, nullptr);
    }
  }
  // rows of at least 128 bytes of an operator with a window-major copy: the windowed hop (32-byte aligned rows, 32-bit
  // offsets), unless the plan's L2 size is 0 or the scatter epilogue is fused
  if (A.n_win > 0 && nv >= 8 && l2_bytes > 0 && !(sh && sh->n_peers > 0)) {
    constexpr int VW = 32 / sizeof(T);
    const int Cw = (C + VW - 1) / VW * VW;
    if (src_ld % VW == 0 && dst_ld % VW == 0 && Cw <= src_ld && Cw <= dst_ld && (reinterpret_cast<uintptr_t>(src) & 31) == 0 &&
        (reinterpret_cast<uintptr_t>(dst) & 31) == 0 && src_ld <= INT32_MAX && dst_ld <= INT32_MAX && n_rows <= INT32_MAX)
      return launch_windows<T>(sm_count, A, n_rows, src, src_ld, dst, dst_ld, C, st);
  }
  if (nv <= 1) return launch_multirow<T, VEC, 1, 8, 1, MB>(sm_count, A, n_rows, src, src_ld, dst, dst_ld, C, st, sh);
  if (nv <= 2) return launch_multirow<T, VEC, 2, 8, 2, MB>(sm_count, A, n_rows, src, src_ld, dst, dst_ld, C, st, sh);
  if (nv <= 4) return launch_multirow<T, VEC, 4, 16, 2, sizeof(T) == 4 ? 8 : 4>(sm_count, A, n_rows, src, src_ld, dst, dst_ld, C, st, sh);
  if (nv <= 8) return launch_multirow<T, VEC, 8, 32, 4, MB>(sm_count, A, n_rows, src, src_ld, dst, dst_ld, C, st, sh);
  // rows wider than 128 bytes: the v2 kernel when its preconditions hold (32-byte aligned rows, 32-bit offsets)
  constexpr int VW = 32 / sizeof(T);
  const int Cw = (C + VW - 1) / VW * VW;
  bool wide_ok = A.rowptr32 != nullptr && (src_ld % VW == 0) && (dst_ld % VW == 0) && (Cw <= src_ld) && (Cw <= dst_ld) &&
                 ((reinterpret_cast<uintptr_t>(src) & 31) == 0) && ((reinterpret_cast<uintptr_t>(dst) & 31) == 0) &&
                 src_ld <= INT32_MAX && dst_ld <= INT32_MAX && n_rows <= INT32_MAX;
  if (sh && sh->n_peers > 0)
    wide_ok = wide_ok && sh->gl % VW == 0 && sh->out_ld % VW == 0 && sh->out_col % VW == 0 && sh->stride_b % VW == 0;
  if (wide_ok) {
    const int nw = Cw / VW;  // 32-byte vectors per row
    // the feature-sharded scatter keeps the chunk width of its row width
    const int L = hop_chunk_lanes(n_rows, nw, sh && sh->n_peers > 0 ? 0 : l2_bytes, A.spread);
    if (L == 4) return launch_v2_sc<T, 4>(sm_count, A, n_rows, src, src_ld, dst, dst_ld, C, st, sh, nullptr);
    if (L == 8) return launch_v2_sc<T, 8>(sm_count, A, n_rows, src, src_ld, dst, dst_ld, C, st, sh, nullptr);
    if (L == 16) return launch_v2_sc<T, 16>(sm_count, A, n_rows, src, src_ld, dst, dst_ld, C, st, sh, nullptr);
    return launch_v2_sc<T, 32>(sm_count, A, n_rows, src, src_ld, dst, dst_ld, C, st, sh, nullptr);
  }
  if (nv <= 16) return launch_one<T, VEC, 16, 4>(sm_count, A, n_rows, src, src_ld, dst, dst_ld, C, st, sh);
  return launch_one<T, VEC, 32, 4>(sm_count, A, n_rows, src, src_ld, dst, dst_ld, C, st, sh);
}

int launch_hop(int dtype, int sm_count, int64_t l2_bytes, const CsrDev& A, int64_t n_rows, const void* src,
               int64_t src_ld, void* dst, int64_t dst_ld, int C, cudaStream_t st, const ScatterHost* sh, const BcastHost* bh) {
  if (C <= 0 || src_ld < C || (!bh && dst_ld < C)) return B200GF_EINVAL;
  if (sh && (sh->n_peers < 0 || sh->n_peers > MAX_PEERS)) return B200GF_EINVAL;
  if (bh && (bh->n_peers < 0 || bh->n_peers > MAX_PEERS || (bh->n_peers > 0 && bh->out_ld < C))) return B200GF_EINVAL;
  if (bh && bh->n_peers == 0 && !(sh && sh->n_peers > 0)) return B200GF_EINVAL;   // no all-gather only in the grid epilogue
  return with_dtype(dtype, [&](auto tag) {
    return launch_typed<decltype(tag)>(sm_count, l2_bytes, A, n_rows, src, src_ld, dst, dst_ld, C, st, sh, bh);
  });
}

// all-gather of an existing node-major row block (the k = 0 term x): every rank's full-height matrix gets these rows
template <typename T, int VEC>
__global__ void bcast_rows_kernel(const T* __restrict__ src, int64_t src_ld, int64_t n_rows, int C, const BcastArgs<T> bc) {
  const int vpr = C / VEC;
  const int64_t total = n_rows * vpr;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / vpr;
    const int cbase = (int)(i - row * vpr) * VEC;
    const Acc<T, VEC> a = load_vec<T, VEC, 0>(src + row * src_ld + cbase, 0);
    bcast_store<T, VEC>(bc, row, cbase, a);
  }
}

int launch_bcast_rows(int dtype, const void* src, int64_t src_ld, int64_t n_rows, int C, cudaStream_t st,
                      const BcastHost* bh) {
  if (!src || !bh || bh->n_peers <= 0 || bh->n_peers > MAX_PEERS || C <= 0 || src_ld < C || bh->out_ld < C) return B200GF_EINVAL;
  if (n_rows == 0) return B200GF_OK;
  const int blocks = 132 * 8;
  if ((reinterpret_cast<uintptr_t>(src) & 15) || (reinterpret_cast<uintptr_t>(bh->mc) & 15)) return B200GF_EUNSUPPORTED;
  for (int i = 0; i < bh->n_peers; ++i)   // 16-byte vector stores into every peer
    if (reinterpret_cast<uintptr_t>(bh->peer[i]) & 15) return B200GF_EUNSUPPORTED;
  if (dtype == B200GF_F32) {
    if (C % 4 || src_ld % 4 || bh->out_ld % 4) return B200GF_EUNSUPPORTED;
    bcast_rows_kernel<float, 4><<<blocks, 256, 0, st>>>((const float*)src, src_ld, n_rows, C, make_bcast<float>(bh));
  } else if (dtype == B200GF_F64) {
    if (C % 2 || src_ld % 2 || bh->out_ld % 2) return B200GF_EUNSUPPORTED;
    bcast_rows_kernel<double, 2><<<blocks, 256, 0, st>>>((const double*)src, src_ld, n_rows, C, make_bcast<double>(bh));
  } else {
    return B200GF_EUNSUPPORTED;
  }
  LAUNCH_CHECK();
  return B200GF_OK;
}

// copy-scatter of an existing node-major matrix (the k = 0 term, x itself) into the peers' row-local operands
template <typename T, int VEC>
__global__ void scatter_rows_kernel(const T* __restrict__ src, int64_t src_ld, int64_t n_rows, int C,
                                    const ScatterArgs<T> sc) {
  const int vpr = C / VEC;
  const int64_t total = n_rows * vpr;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / vpr;
    const int cbase = (int)(i - row * vpr) * VEC;
    const Acc<T, VEC> a = load_vec<T, VEC, 0>(src + row * src_ld + cbase, 0);
    scatter_store<T, VEC>(sc, row, cbase, a);
  }
}

int launch_scatter_rows(int dtype, const void* src, int64_t src_ld, int64_t n_rows, int C, cudaStream_t st,
                        const ScatterHost* sh) {
  if (!src || !sh || sh->n_peers <= 0 || sh->n_peers > MAX_PEERS || C <= 0 || src_ld < C) return B200GF_EINVAL;
  if (n_rows == 0) return B200GF_OK;
  const int blocks = 132 * 8;
  if (reinterpret_cast<uintptr_t>(src) & 15) return B200GF_EUNSUPPORTED;   // 16-byte vector loads
  if (dtype == B200GF_F32) {
    if (C % 4 || src_ld % 4 || sh->gl % 4 || sh->out_ld % 4 || sh->out_col % 4 || sh->stride_b % 4) return B200GF_EUNSUPPORTED;
    scatter_rows_kernel<float, 4><<<blocks, 256, 0, st>>>((const float*)src, src_ld, n_rows, C, make_scatter<float>(sh));
  } else if (dtype == B200GF_F64) {
    if (C % 2 || src_ld % 2 || sh->gl % 2 || sh->out_ld % 2 || sh->out_col % 2 || sh->stride_b % 2) return B200GF_EUNSUPPORTED;
    scatter_rows_kernel<double, 2><<<blocks, 256, 0, st>>>((const double*)src, src_ld, n_rows, C, make_scatter<double>(sh));
  } else {
    return B200GF_EUNSUPPORTED;
  }
  LAUNCH_CHECK();
  return B200GF_OK;
}

}  // namespace b200gf

extern "C" int b200gf_hop(const b200gf_plan* plan, int e, int direction, const void* src, int64_t src_ld,
                          void* dst, int64_t dst_ld, int C, void* stream) {
  if (!plan || !src || !dst || e < 0 || e >= plan->E) return B200GF_EINVAL;
  if (direction != B200GF_HOP_FWD && direction != B200GF_HOP_BWD) return B200GF_EINVAL;
  if (direction == B200GF_HOP_BWD && !plan->has_bwd) return B200GF_EINVAL;
  const b200gf::CsrDev& A = direction == B200GF_HOP_FWD ? plan->fwd[e] : plan->bwd[e];
  return b200gf::plan_hop(plan, A, src, src_ld, dst, dst_ld, C, (cudaStream_t)stream, nullptr);
}

// ---------------------------------------------------------------------------------------------------
// fused hop + NVLink scatter, and the symmetric (IPC) buffers it writes into
// ---------------------------------------------------------------------------------------------------
static int fill_scatter(b200gf::ScatterHost& sh, const void* const* peers, int n_peers, int64_t rows_per_peer,
                        int64_t out_ld, int64_t out_col, int gl, int64_t stride_b) {
  if (!peers || n_peers <= 0 || n_peers > b200gf::MAX_PEERS || rows_per_peer <= 0 || gl <= 0) return B200GF_EINVAL;
  for (int i = 0; i < n_peers; ++i) {
    if (!peers[i] || (reinterpret_cast<uintptr_t>(peers[i]) & 15)) return B200GF_EINVAL;
    sh.peer[i] = const_cast<void*>(peers[i]);
  }
  sh.n_peers = n_peers; sh.rows_per_peer = rows_per_peer; sh.out_ld = out_ld; sh.out_col = out_col; sh.gl = gl;
  sh.stride_b = stride_b;
  return B200GF_OK;
}

extern "C" int b200gf_hop_scatter(const b200gf_plan* plan, int e, int direction, const void* src, int64_t src_ld,
                                  void* dst, int64_t dst_ld, int C, const void* const* peers, int n_peers,
                                  int64_t rows_per_peer, int64_t out_ld, int64_t out_col, int gl, int64_t stride_b,
                                  void* stream) {
  if (!plan || !src || !dst || e < 0 || e >= plan->E) return B200GF_EINVAL;
  if (direction != B200GF_HOP_FWD && direction != B200GF_HOP_BWD) return B200GF_EINVAL;
  if (direction == B200GF_HOP_BWD && !plan->has_bwd) return B200GF_EINVAL;
  b200gf::ScatterHost sh{};
  int rc = fill_scatter(sh, peers, n_peers, rows_per_peer, out_ld, out_col, gl, stride_b);
  if (rc) return rc;
  if (plan->n_rows > rows_per_peer * n_peers || C % gl != 0) return B200GF_EINVAL;
  const b200gf::CsrDev& A = direction == B200GF_HOP_FWD ? plan->fwd[e] : plan->bwd[e];
  return b200gf::plan_hop(plan, A, src, src_ld, dst, dst_ld, C, (cudaStream_t)stream, &sh);
}

extern "C" int b200gf_scatter_rows(int dtype, const void* src, int64_t src_ld, int64_t n_rows, int C,
                                   const void* const* peers, int n_peers, int64_t rows_per_peer, int64_t out_ld,
                                   int64_t out_col, int gl, int64_t stride_b, void* stream) {
  b200gf::ScatterHost sh{};
  int rc = fill_scatter(sh, peers, n_peers, rows_per_peer, out_ld, out_col, gl, stride_b);
  if (rc) return rc;
  if (n_rows > rows_per_peer * n_peers || C % gl != 0) return B200GF_EINVAL;
  return b200gf::launch_scatter_rows(dtype, src, src_ld, n_rows, C, (cudaStream_t)stream, &sh);
}

static int fill_bcast(b200gf::BcastHost& bh, const void* const* peers, int n_peers, const void* mc, int64_t row0, int64_t out_ld) {
  if (!peers || n_peers <= 0 || n_peers > b200gf::MAX_PEERS || row0 < 0 || out_ld <= 0) return B200GF_EINVAL;
  for (int i = 0; i < n_peers; ++i) {
    if (!peers[i]) return B200GF_EINVAL;
    bh.peer[i] = const_cast<void*>(peers[i]);
  }
  bh.mc = const_cast<void*>(mc);
  bh.n_peers = n_peers; bh.row0 = row0; bh.out_ld = out_ld;
  return B200GF_OK;
}

extern "C" int b200gf_hop_bcast(const b200gf_plan* plan, int e, int direction, const void* src, int64_t src_ld, int C,
                                const void* const* peers, int n_peers, const void* mc, int64_t row0, int64_t out_ld,
                                void* stream) {
  if (!plan || !src || e < 0 || e >= plan->E) return B200GF_EINVAL;
  if (direction != B200GF_HOP_FWD && direction != B200GF_HOP_BWD) return B200GF_EINVAL;
  if (direction == B200GF_HOP_BWD && !plan->has_bwd) return B200GF_EINVAL;
  b200gf::BcastHost bh{};
  int rc = fill_bcast(bh, peers, n_peers, mc, row0, out_ld);
  if (rc) return rc;
  const b200gf::CsrDev& A = direction == B200GF_HOP_FWD ? plan->fwd[e] : plan->bwd[e];
  return b200gf::plan_hop(plan, A, src, src_ld, nullptr, 0, C, (cudaStream_t)stream, nullptr, &bh);
}

extern "C" int b200gf_hop_grid(const b200gf_plan* plan, int e, int direction, const void* src, int64_t src_ld, int C,
                               const void* const* bc_peers, int n_bc, int64_t row0, int64_t bc_ld,
                               const void* const* sc_peers, int n_sc, int64_t rows_per_peer, int64_t out_ld, int64_t out_col,
                               int gl, int64_t stride_b, void* stream) {
  if (!plan || !src || e < 0 || e >= plan->E) return B200GF_EINVAL;
  if (direction != B200GF_HOP_FWD && direction != B200GF_HOP_BWD) return B200GF_EINVAL;
  if (direction == B200GF_HOP_BWD && !plan->has_bwd) return B200GF_EINVAL;
  b200gf::BcastHost bh{};
  if (n_bc > 0) {
    int rc = fill_bcast(bh, bc_peers, n_bc, nullptr, row0, bc_ld);
    if (rc) return rc;
  } else {
    bh.n_peers = 0; bh.mc = nullptr; bh.row0 = 0; bh.out_ld = 0;
  }
  b200gf::ScatterHost sh{};
  int rc = fill_scatter(sh, sc_peers, n_sc, rows_per_peer, out_ld, out_col, gl, stride_b);
  if (rc) return rc;
  if (plan->n_rows > rows_per_peer * n_sc || C % gl != 0) return B200GF_EINVAL;
  const b200gf::CsrDev& A = direction == B200GF_HOP_FWD ? plan->fwd[e] : plan->bwd[e];
  return b200gf::plan_hop(plan, A, src, src_ld, nullptr, 0, C, (cudaStream_t)stream, &sh, &bh);
}

extern "C" int b200gf_bcast_rows(int dtype, const void* src, int64_t src_ld, int64_t n_rows, int C,
                                 const void* const* peers, int n_peers, const void* mc, int64_t row0, int64_t out_ld,
                                 void* stream) {
  b200gf::BcastHost bh{};
  int rc = fill_bcast(bh, peers, n_peers, mc, row0, out_ld);
  if (rc) return rc;
  return b200gf::launch_bcast_rows(dtype, src, src_ld, n_rows, C, (cudaStream_t)stream, &bh);
}

extern "C" int b200gf_symm_alloc(void** ptr, size_t bytes) {
  if (!ptr || bytes == 0) return B200GF_EINVAL;
  *ptr = nullptr;
  if (cudaMalloc(ptr, bytes) != cudaSuccess) { (void)cudaGetLastError(); return B200GF_ENOMEM; }
  CUDA_TRY(cudaMemset(*ptr, 0, bytes));
  return B200GF_OK;
}
extern "C" int b200gf_symm_free(void* ptr) {
  if (ptr) CUDA_TRY(cudaFree(ptr));
  return B200GF_OK;
}
extern "C" int b200gf_symm_export(void* ptr, void* handle64) {
  if (!ptr || !handle64) return B200GF_EINVAL;
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  CUDA_TRY(cudaIpcGetMemHandle(reinterpret_cast<cudaIpcMemHandle_t*>(handle64), ptr));
  return B200GF_OK;
}
extern "C" int b200gf_symm_import(const void* handle64, void** ptr) {
  if (!ptr || !handle64) return B200GF_EINVAL;
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, sizeof(h));
  CUDA_TRY(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return B200GF_OK;
}
extern "C" int b200gf_symm_close(void* ptr) {
  if (ptr) CUDA_TRY(cudaIpcCloseMemHandle(ptr));
  return B200GF_OK;
}

// ---------------------------------------------------------------------------------------------------
// Peer fence without NCCL: monotone step counters in symmetric memory.
//   signal: step = ++(*local_step); make every earlier peer store of this GPU visible (system-scope fence), then write
//           `step` into slot `my_rank` of every peer's flag array;
//   wait  : spin until all n_peers slots of MY flag array are >= *local_step.
// All arguments are fixed addresses, so both kernels can be captured in a CUDA graph and replayed every step.
// ---------------------------------------------------------------------------------------------------
namespace b200gf {

struct FlagPeers {
  unsigned long long* flags[MAX_PEERS];
};

__global__ void peer_signal_kernel(FlagPeers fp, int n_peers, int my_rank, unsigned long long* local_step) {
  __shared__ unsigned long long step;
  if (threadIdx.x == 0) {
    step = *local_step + 1ull;
    *local_step = step;
    __threadfence_system();  // orders this GPU's earlier (previous-kernel) peer stores before the flag stores below
  }
  __syncthreads();
  if ((int)threadIdx.x < n_peers) {
    unsigned long long* dst = fp.flags[threadIdx.x] + my_rank;
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(dst), "l"(step) : "memory");
  }
}

__global__ void peer_wait_kernel(const unsigned long long* my_flags, int n_peers, const unsigned long long* local_step) {
  if ((int)threadIdx.x >= n_peers) return;
  const unsigned long long want = *local_step;
  unsigned long long seen = 0;
  unsigned long long spins = 0;
  while (true) {
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(my_flags + threadIdx.x) : "memory");
    if (seen >= want) break;
    if (++spins > (1ull << 31)) __trap();  // a peer died: fail loudly instead of hanging the GPU
    __nanosleep(100);
  }
}

}  // namespace b200gf

extern "C" int b200gf_peer_signal(const void* const* peer_flags, int n_peers, int my_rank, void* local_step, void* stream) {
  if (!peer_flags || n_peers <= 0 || n_peers > b200gf::MAX_PEERS || my_rank < 0 || my_rank >= n_peers || !local_step)
    return B200GF_EINVAL;
  b200gf::FlagPeers fp{};
  for (int i = 0; i < n_peers; ++i) {
    if (!peer_flags[i]) return B200GF_EINVAL;
    fp.flags[i] = reinterpret_cast<unsigned long long*>(const_cast<void*>(peer_flags[i]));
  }
  b200gf::peer_signal_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(fp, n_peers, my_rank, (unsigned long long*)local_step);
  LAUNCH_CHECK();
  return B200GF_OK;
}

extern "C" int b200gf_peer_wait(const void* my_flags, int n_peers, const void* local_step, void* stream) {
  if (!my_flags || n_peers <= 0 || n_peers > b200gf::MAX_PEERS || !local_step) return B200GF_EINVAL;
  b200gf::peer_wait_kernel<<<1, 32, 0, (cudaStream_t)stream>>>((const unsigned long long*)my_flags, n_peers,
                                                             (const unsigned long long*)local_step);
  LAUNCH_CHECK();
  return B200GF_OK;
}
