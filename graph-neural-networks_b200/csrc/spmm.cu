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
// route_hop picks a hop's kernel, or refuses the hop, before any CUDA call; launch_route turns that choice into the
// kernel's instantiation and launches it.
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

template <typename T, int EPI>
static ScatterParam<T, EPI> make_epilogue(const ScatterHost* sh, const BcastHost* bh) {
  ScatterParam<T, EPI> sp{};
  if constexpr (EPI == EPI_SCATTER) sp.a = make_scatter<T>(sh);
  if constexpr (EPI == EPI_BCAST) sp.a = make_bcast<T>(bh);
  if constexpr (EPI == EPI_GRID) { sp.s = make_scatter<T>(sh); sp.a = make_bcast<T>(bh); }
  return sp;
}

// one hop's operands; sh is null unless there are scatter peers, bh null without the all-gather epilogue
template <typename T>
struct HopArgs {
  int sm_count;
  const CsrDev& A;
  int64_t n_rows;
  const T* src;
  int64_t src_ld;
  T* dst;
  int64_t dst_ld;
  int C;
  cudaStream_t st;
  const ScatterHost* sh;
  const BcastHost* bh;
};

// Launches kern as a persistent grid over `units` work items, `per_block` to a block: at most one resident wave
// (sm_count x the kernel's occupancy), whose warps stride over the rest; chunks on blockIdx.y.
template <typename T, typename K, typename... Args>
static int launch_resident(K kern, int threads, const HopArgs<T>& h, int64_t units, int per_block, int chunks,
                           Args... args) {
  int occ = 0;
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, 0));
  const int64_t blocks = std::min<int64_t>((units + per_block - 1) / per_block, (int64_t)h.sm_count * std::max(occ, 1));
  kern<<<dim3((unsigned)blocks, (unsigned)chunks), threads, 0, h.st>>>(args...);
  LAUNCH_CHECK();
  return B200GF_OK;
}

// Library configuration (tools/spmm_sweep.cu explores the alternatives): 256 threads, registers capped for 6 resident
// blocks/SM (48 warps: the kernel is latency-bound below that), gathered rows loaded with an L2 evict_last policy and no
// L1 allocation (a sticky subset of the gathered slab stays in L2), no next-row prefetch (it costs registers).
template <typename T, int VEC, int L>
static int launch_one(const HopArgs<T>& h) {
  constexpr int U = 4, THREADS = 256, MINB = sizeof(T) == 4 ? 6 : 4, HINT = 3;
  constexpr bool PF = false;
  auto kern = spmm_hop_kernel<T, VEC, L, U, THREADS, MINB, HINT, PF>;
  const int n_chunks = (h.C + L * VEC - 1) / (L * VEC);
  return launch_resident(kern, THREADS, h, h.n_rows * n_chunks, THREADS / 32, 1, h.A.rowptr, h.A.col,
                         reinterpret_cast<const T*>(h.A.val), h.src, h.src_ld, h.dst, h.dst_ld, h.n_rows, h.C, n_chunks,
                         1.0f, make_scatter<T>(h.sh));
}

// narrow rows (<= 128 bytes): several rows per warp (spmm_hop_multirow_kernel), geometry from the small-C sweep of
// tools/spmm_sweep.cu
template <typename T, int L, int GS, int U, int MINB>
static int launch_multirow(const HopArgs<T>& h) {
  constexpr int VEC = 16 / sizeof(T), THREADS = 256, HINT = 3;
  auto kern = spmm_hop_multirow_kernel<T, VEC, L, GS, U, THREADS, MINB, HINT>;
  return launch_resident(kern, THREADS, h, h.n_rows, (THREADS / 32) * (32 / GS), 1, h.A.rowptr, h.A.col,
                         reinterpret_cast<const T*>(h.A.val), h.src, h.src_ld, h.dst, h.dst_ld, h.n_rows, h.C,
                         make_scatter<T>(h.sh));
}

// Round-2 kernel (spmm_kernels.cuh: spmm_hop_v2_kernel): 32-byte lanes loaded as two 16-byte halves, 32-bit index
// arithmetic.  L lanes x 32 bytes cover a row chunk: the lanes' first halves its first L*16 bytes, their second halves the
// rest (LaneMap; the NVLink epilogues keep a lane's 32 bytes adjacent), so every LDG.128 / STG.128 of a lane group covers
// whole 32-byte sectors; 32/L neighbours per warp-wide load, U loads in flight per lane; 4 blocks of 256 threads per SM
// (64 registers); column chunks on blockIdx.y.
template <typename T, int L, int EPI>
static int launch_v2(const HopArgs<T>& h) {
  constexpr int VEC = 32 / sizeof(T), U = 4, THREADS = 256, MINB = sizeof(T) == 4 ? 4 : 3, HINT = B200GF_HOP_L2_HINT;
  // streaming stores (SH = 1): the result rows are read by the next launch, not by this one, so at normal priority they
  // only displace gathered lines from the L2 (2.74 against 2.78 ms per hop at N = 1M, 64 fp32 columns)
  auto kern = spmm_hop_v2_kernel<T, int32_t, VEC, L, U, THREADS, MINB, HINT, EPI, 1>;
  const int n_chunks = (h.C + L * VEC - 1) / (L * VEC);
  if (n_chunks > 65535) return B200GF_EUNSUPPORTED;
  // one resident wave per chunk when there is a single chunk; with several chunks each chunk gets its own wave-sized
  // slice of the grid so that the block scheduler runs them chunk-major
  return launch_resident(kern, THREADS, h, h.n_rows, THREADS / 32, n_chunks, h.A.rowptr32, h.A.col,
                         reinterpret_cast<const T*>(h.A.val), h.src, (int)h.src_ld, h.dst, (int)h.dst_ld, (int)h.n_rows,
                         h.C, B200GF_HOP_L2_FRAC, make_epilogue<T, EPI>(h.sh, h.bh));
}

// 64-byte rows (C = 16 floats / 8 doubles) with 32-byte lanes: two lanes per neighbour row, 8-lane row groups, two loads in
// flight per lane; rows of C = 8 stay on spmm_hop_multirow_kernel.
template <typename T, int EPI>
static int launch_multirow_v2(const HopArgs<T>& h) {
  constexpr int VEC = 32 / sizeof(T), L = 2, GS = 8, U = 2, THREADS = 256, MINB = sizeof(T) == 4 ? 4 : 3, HINT = 3;
  auto kern = spmm_hop_multirow_v2_kernel<T, int32_t, VEC, L, GS, U, THREADS, MINB, HINT, EPI>;
  return launch_resident(kern, THREADS, h, h.n_rows, (THREADS / 32) * (32 / GS), 1, h.A.rowptr32, h.A.col,
                         reinterpret_cast<const T*>(h.A.val), h.src, (int)h.src_ld, h.dst, (int)h.dst_ld, (int)h.n_rows,
                         h.C, make_epilogue<T, EPI>(h.sh, h.bh));
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
static int launch_window(const HopArgs<T>& h, const int32_t* rowptr, int c0, int Cc) {
  constexpr int VEC = 32 / sizeof(T), L = 4, GS = B200GF_HOP_WIN_GS, U = B200GF_HOP_WIN_U, THREADS = 256;
  constexpr int MINB = sizeof(T) == 4 ? 4 : 3, HINT = B200GF_HOP_WIN_HINT;
  auto kern = spmm_hop_multirow_v2_kernel<T, int32_t, VEC, L, GS, U, THREADS, MINB, HINT, MODE>;
  return launch_resident(kern, THREADS, h, h.n_rows, (THREADS / 32) * (32 / GS), 1, rowptr, h.A.win_col,
                         reinterpret_cast<const T*>(h.A.win_val), h.src + c0, (int)h.src_ld, h.dst + c0, (int)h.dst_ld,
                         (int)h.n_rows, Cc, ScatterParam<T, MODE>{});
}

template <typename T>
static int launch_windows(const HopArgs<T>& h) {
  constexpr int CW = 128 / sizeof(T);   // columns per chunk
  for (int c0 = 0; c0 < h.C; c0 += CW) {
    const int Cc = std::min(CW, h.C - c0);
    for (int w = 0; w < h.A.n_win; ++w) {
      const int32_t* rp = h.A.win_rowptr32 + (int64_t)w * (h.n_rows + 1);
      const int rc = w == 0 ? launch_window<T, EPI_NONE>(h, rp, c0, Cc) : launch_window<T, EPI_ACCUM>(h, rp, c0, Cc);
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

static bool aligned(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

// The operands of 32-byte lanes (the v2 kernels and the windowed hop): 32-bit row offsets and row count; src, and dst
// when the hop stores one, 32-byte aligned, with strides of whole 32-byte vectors that hold the padded row and fit
// int32.
template <typename T>
static bool lanes32_ok(const HopArgs<T>& h) {
  constexpr int V32 = 32 / sizeof(T);
  const int64_t Cw = (h.C + V32 - 1) / V32 * V32;
  const auto rows_ok = [&](const void* p, int64_t ld) {
    return aligned(p, 32) && ld % V32 == 0 && Cw <= ld && ld <= INT32_MAX;
  };
  return h.A.rowptr32 != nullptr && h.n_rows <= INT32_MAX && rows_ok(h.src, h.src_ld) &&
         (!h.dst || rows_ok(h.dst, h.dst_ld));
}

// no scatter epilogue, or one whose column offsets and strides are whole vectors of q elements
static bool scatter_aligned(const ScatterHost* sh, int q) {
  return !sh || (sh->gl % q == 0 && sh->out_ld % q == 0 && sh->out_col % q == 0 && sh->stride_b % q == 0);
}

enum class HopKernel { scalar, v1, multirow, multirow_v2, v2, windowed };

struct HopRoute {
  HopKernel kernel;
  int L;     // lanes (v1, v2) or 16-byte vectors per row (multirow)
  int epi;   // EPI_*; the 16-byte-lane kernels take the scatter as ScatterArgs
};

// The hop's kernel, or B200GF_EUNSUPPORTED, decided before any CUDA call.  The order of the checks is the policy.
template <typename T>
static int route_hop(const HopArgs<T>& h, int64_t l2_bytes, HopRoute* r) {
  constexpr int V16 = 16 / sizeof(T), V32 = 32 / sizeof(T);
  const int nw = (h.C + V32 - 1) / V32;   // 32-byte vectors per row
  const bool lanes32 = lanes32_ok(h);
  if (h.bh) {
    // 1. fused all-gather (EPI_BCAST), or all-gather + scatter (EPI_GRID): 32-byte lanes into 32-byte aligned peers,
    //    rows of at least 64 bytes
    const BcastHost& b = *h.bh;
    bool ok = lanes32 && nw >= 2 && aligned(b.mc, 32) && scatter_aligned(h.sh, V32);
    if (b.n_peers > 0) ok = ok && (int64_t)nw * V32 <= b.out_ld && b.out_ld % V32 == 0;
    for (int i = 0; i < b.n_peers; ++i) ok = ok && aligned(b.peer[i], 32);
    // 64-byte rows take the multi-row kernel, which is compiled for the grid epilogue only
    if (!ok || (nw == 2 && !h.sh)) return B200GF_EUNSUPPORTED;
    *r = nw == 2 ? HopRoute{HopKernel::multirow_v2, 2, EPI_GRID}
                 : HopRoute{HopKernel::v2, nw <= 4 ? 4 : nw <= 8 ? 8 : nw <= 16 ? 16 : 32, h.sh ? EPI_GRID : EPI_BCAST};
    return B200GF_OK;
  }
  // 2. 16-byte vectors, else one element per lane (without the fused scatter, which needs the vectors)
  const int nv = (h.C + V16 - 1) / V16;   // 16-byte vectors per row
  const auto vec16 = [&](const void* p, int64_t ld) { return aligned(p, 16) && ld % V16 == 0 && nv * V16 <= ld; };
  if (!vec16(h.src, h.src_ld) || !vec16(h.dst, h.dst_ld)) {
    if (h.sh) return B200GF_EUNSUPPORTED;
    *r = {HopKernel::scalar, 32, EPI_NONE};
    return B200GF_OK;
  }
  // 3. scatter fields of whole 16-byte vectors
  if (!scatter_aligned(h.sh, V16)) return B200GF_EUNSUPPORTED;
  const bool v2_ok = lanes32 && scatter_aligned(h.sh, V32);
  const int epi = h.sh ? EPI_SCATTER : EPI_NONE;
  if (nv > 2 && nv <= 4 && v2_ok)
    *r = {HopKernel::multirow_v2, 2, epi};   // 4. 64-byte rows (C = 16 floats / 8 doubles) with 32-byte lanes
  else if (nv >= 8 && h.A.n_win > 0 && l2_bytes > 0 && !h.sh && lanes32)
    *r = {HopKernel::windowed, 4, EPI_NONE};   // 5. rows of at least 128 bytes of an operator with source windows
  else if (nv <= 8)
    *r = {HopKernel::multirow, nv <= 1 ? 1 : nv <= 2 ? 2 : nv <= 4 ? 4 : 8, epi};   // 6. rows of <= 128 bytes
  else if (v2_ok)   // 7. wider rows with 32-byte lanes; the scatter keeps the chunk width of its row width
    *r = {HopKernel::v2, hop_chunk_lanes(h.n_rows, nw, h.sh ? 0 : l2_bytes, h.A.spread), epi};
  else
    *r = {HopKernel::v1, nv <= 16 ? 16 : 32, epi};   // 8. wider rows with 16-byte lanes
  return B200GF_OK;
}

// f(std::integral_constant<int, V>{}) for the V of Vs equal to v
template <int... Vs, typename Fn>
static int with_const(int v, Fn&& f) {
  int rc = B200GF_EUNSUPPORTED;
  (void)((v == Vs && ((rc = f(std::integral_constant<int, Vs>{})), true)) || ...);
  return rc;
}

// the instantiation of a route
template <typename T>
static int launch_route(const HopArgs<T>& h, const HopRoute& r) {
  constexpr int V16 = 16 / sizeof(T), MB = sizeof(T) == 4 ? 6 : 4;
  const auto with_epi = [&](auto f) { return with_const<EPI_NONE, EPI_SCATTER, EPI_BCAST, EPI_GRID>(r.epi, f); };
  switch (r.kernel) {
    case HopKernel::scalar: return launch_one<T, 1, 32>(h);
    case HopKernel::v1: return r.L == 16 ? launch_one<T, V16, 16>(h) : launch_one<T, V16, 32>(h);
    case HopKernel::multirow:
      switch (r.L) {
        case 1: return launch_multirow<T, 1, 8, 1, MB>(h);
        case 2: return launch_multirow<T, 2, 8, 2, MB>(h);
        case 4: return launch_multirow<T, 4, 16, 2, sizeof(T) == 4 ? 8 : 4>(h);
        default: return launch_multirow<T, 8, 32, 4, MB>(h);
      }
    case HopKernel::multirow_v2:
      return with_epi([&](auto e) -> int {
        constexpr int EPI = decltype(e)::value;
        // the all-gather alone never takes 64-byte rows: no such multi-row kernel is compiled
        if constexpr (EPI == EPI_BCAST) return B200GF_EUNSUPPORTED;
        else return launch_multirow_v2<T, EPI>(h);
      });
    case HopKernel::v2:
      return with_const<4, 8, 16, 32>(r.L, [&](auto l) {
        return with_epi([&](auto e) -> int {
          constexpr int L = decltype(l)::value, EPI = decltype(e)::value;
          // the scatter alone sizes its chunks by row width (hop_chunk_lanes without an L2 budget), so L >= 8: no 4-lane
          // scatter kernel is compiled
          if constexpr (L == 4 && EPI == EPI_SCATTER) return B200GF_EUNSUPPORTED;
          else return launch_v2<T, L, EPI>(h);
        });
      });
    case HopKernel::windowed: return launch_windows<T>(h);
  }
  return B200GF_EUNSUPPORTED;
}

int launch_hop(int dtype, int sm_count, int64_t l2_bytes, const CsrDev& A, int64_t n_rows, const void* src,
               int64_t src_ld, void* dst, int64_t dst_ld, int C, cudaStream_t st, const ScatterHost* sh, const BcastHost* bh) {
  if (C <= 0 || src_ld < C || (!bh && dst_ld < C)) return B200GF_EINVAL;
  if (sh && (sh->n_peers < 0 || sh->n_peers > MAX_PEERS)) return B200GF_EINVAL;
  if (bh && (bh->n_peers < 0 || bh->n_peers > MAX_PEERS || (bh->n_peers > 0 && bh->out_ld < C))) return B200GF_EINVAL;
  if (bh && bh->n_peers == 0 && !(sh && sh->n_peers > 0)) return B200GF_EINVAL;   // no all-gather only in the grid epilogue
  return with_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    const HopArgs<T> h{sm_count, A, n_rows, reinterpret_cast<const T*>(src), src_ld, reinterpret_cast<T*>(dst), dst_ld, C, st,
                       sh && sh->n_peers > 0 ? sh : nullptr, bh};
    HopRoute r;
    if (int rc = route_hop(h, l2_bytes, &r)) return rc;
    return n_rows == 0 ? B200GF_OK : launch_route(h, r);
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
  return with_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    constexpr int VEC = 16 / sizeof(T);
    if (C % VEC || src_ld % VEC || bh->out_ld % VEC) return B200GF_EUNSUPPORTED;
    bcast_rows_kernel<T, VEC><<<blocks, 256, 0, st>>>((const T*)src, src_ld, n_rows, C, make_bcast<T>(bh));
    LAUNCH_CHECK();
    return B200GF_OK;
  });
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
  return with_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    constexpr int VEC = 16 / sizeof(T);
    if (C % VEC || src_ld % VEC || !scatter_aligned(sh, VEC)) return B200GF_EUNSUPPORTED;
    scatter_rows_kernel<T, VEC><<<blocks, 256, 0, st>>>((const T*)src, src_ld, n_rows, C, make_scatter<T>(sh));
    LAUNCH_CHECK();
    return B200GF_OK;
  });
}

}  // namespace b200gf

// the operator of (e, direction) of a plan, null for a null plan, an e out of range, an unknown direction, or the
// backward operator of a plan without one
static const b200gf::CsrDev* hop_operator(const b200gf_plan* plan, int e, int direction) {
  if (!plan || e < 0 || e >= plan->E) return nullptr;
  if (direction == B200GF_HOP_FWD) return &plan->fwd[e];
  if (direction == B200GF_HOP_BWD && plan->has_bwd) return &plan->bwd[e];
  return nullptr;
}

extern "C" int b200gf_hop(const b200gf_plan* plan, int e, int direction, const void* src, int64_t src_ld,
                          void* dst, int64_t dst_ld, int C, void* stream) {
  const b200gf::CsrDev* A = hop_operator(plan, e, direction);
  if (!A || !src || !dst) return B200GF_EINVAL;
  return b200gf::plan_hop(plan, *A, src, src_ld, dst, dst_ld, C, (cudaStream_t)stream, nullptr);
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
  const b200gf::CsrDev* A = hop_operator(plan, e, direction);
  if (!A || !src || !dst) return B200GF_EINVAL;
  b200gf::ScatterHost sh{};
  int rc = fill_scatter(sh, peers, n_peers, rows_per_peer, out_ld, out_col, gl, stride_b);
  if (rc) return rc;
  if (plan->n_rows > rows_per_peer * n_peers || C % gl != 0) return B200GF_EINVAL;
  return b200gf::plan_hop(plan, *A, src, src_ld, dst, dst_ld, C, (cudaStream_t)stream, &sh);
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
  const b200gf::CsrDev* A = hop_operator(plan, e, direction);
  if (!A || !src) return B200GF_EINVAL;
  b200gf::BcastHost bh{};
  int rc = fill_bcast(bh, peers, n_peers, mc, row0, out_ld);
  if (rc) return rc;
  return b200gf::plan_hop(plan, *A, src, src_ld, nullptr, 0, C, (cudaStream_t)stream, nullptr, &bh);
}

extern "C" int b200gf_hop_grid(const b200gf_plan* plan, int e, int direction, const void* src, int64_t src_ld, int C,
                               const void* const* bc_peers, int n_bc, int64_t row0, int64_t bc_ld,
                               const void* const* sc_peers, int n_sc, int64_t rows_per_peer, int64_t out_ld, int64_t out_col,
                               int gl, int64_t stride_b, void* stream) {
  const b200gf::CsrDev* A = hop_operator(plan, e, direction);
  if (!A || !src) return B200GF_EINVAL;
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
  return b200gf::plan_hop(plan, *A, src, src_ld, nullptr, 0, C, (cudaStream_t)stream, &sh, &bh);
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
