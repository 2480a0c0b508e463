// Kernels of the graph shift ("hop"); included by spmm.cu (the library) and tools/spmm_sweep.cu (tuning sweeps).
//
//   dst[r, :] = sum_j A[r, j] * src[j, :]        A = CSR gather operator, src/dst node-major [rows, ld]
//
// Mapping (sm_90a, 132 SMs):
//   * one warp per (row, column chunk) work item, grid-stride over items in chunk-major order, so that at any
//     time all resident warps gather from the same column slab (keeps it L2-resident when N * chunk_bytes fits);
//   * L lanes cover the chunk of a neighbour row; the 32/L lane groups each take a different neighbour, so one
//     warp-wide load fetches 32/L neighbour rows;
//   * the wide-row kernels (v2) give each lane 32 bytes as two 16-byte halves (sm_90 has no 256-bit load).  The first
//     halves of a group's L lanes are the chunk's first L*16 bytes and the second halves the rest (LaneMap), so each
//     warp-wide LDG.128 or STG.128 covers whole 32-byte sectors;
//   * U independent loads per lane are in flight before the FMAs (memory-level parallelism);
//   * col/val of a row are read once, coalesced (lane i holds entry i), and broadcast with SHFL;
//   * PF (template flag, off in the library): prefetch of the next row's col/val and of the rowptr pair after it while
//     the current row is gathered — it costs registers and issue slots; kept for the sweep tool.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>

// EPI_ACCUM with fp32 32-byte lanes (the windowed hop's windows after the first): 1 adds into dst with L2 vector
// reductions, 0 reads, adds and stores (tools/hop_window_bench.py --variants builds both)
#ifndef B200GF_HOP_WIN_RED
#define B200GF_HOP_WIN_RED 1
#endif

namespace b200gf {

template <typename T, int VEC>
struct Acc {
  T v[VEC];
  __device__ __forceinline__ void zero() {
#pragma unroll
    for (int i = 0; i < VEC; ++i) v[i] = T(0);
  }
};

// L2 cache policy: `frac` of the touched lines (chosen by address hash) get evict_last priority, the rest stay
// evict_unchanged.  With the gathered feature matrix larger than the L2, a sticky subset that fits turns an LRU
// thrash into hits on that subset.
__device__ __forceinline__ uint64_t evict_last_policy(float frac) {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, %1;" : "=l"(pol) : "f"(frac));
  return pol;
}

// HINT 0: ld.global.nc (default policy)   1: + L1::no_allocate (gathered rows have no L1 reuse)
// HINT >= 2: L1::no_allocate + the L2 policy in `pol` on the gathered rows (fight for L2 residency of the feature slab)
template <typename T, int VEC, int HINT>
__device__ __forceinline__ Acc<T, VEC> load_vec(const T* p, uint64_t pol) {
  Acc<T, VEC> a;
  if constexpr (VEC == 4 && sizeof(T) == 4) {
    float4 t;
    if constexpr (HINT == 0) {
      t = __ldg(reinterpret_cast<const float4*>(p));
    } else if constexpr (HINT == 1) {
      asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                   : "=f"(t.x), "=f"(t.y), "=f"(t.z), "=f"(t.w) : "l"(p));
    } else {
      asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;"
                   : "=f"(t.x), "=f"(t.y), "=f"(t.z), "=f"(t.w) : "l"(p), "l"(pol));
    }
    a.v[0] = t.x; a.v[1] = t.y; a.v[2] = t.z; a.v[3] = t.w;
  } else if constexpr (VEC == 2) {
    double2 t;
    if constexpr (HINT == 0) {
      t = __ldg(reinterpret_cast<const double2*>(p));
    } else if constexpr (HINT == 1) {
      asm volatile("ld.global.nc.L1::no_allocate.v2.f64 {%0,%1}, [%2];" : "=d"(t.x), "=d"(t.y) : "l"(p));
    } else {
      asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.f64 {%0,%1}, [%2], %3;"
                   : "=d"(t.x), "=d"(t.y) : "l"(p), "l"(pol));
    }
    a.v[0] = t.x; a.v[1] = t.y;
  } else {
    a.v[0] = __ldg(p);
  }
  return a;
}

// SH 0: default store   1: st.global.cs (streaming: the result row is not re-read by this kernel)
template <typename T, int VEC, int SH>
__device__ __forceinline__ void store_vec(T* p, const Acc<T, VEC>& a) {
  if constexpr (VEC * sizeof(T) == 32) {
    // 32-byte lane: two adjacent 16-byte stores
    Acc<T, VEC / 2> lo, hi;
#pragma unroll
    for (int i = 0; i < VEC / 2; ++i) { lo.v[i] = a.v[i]; hi.v[i] = a.v[VEC / 2 + i]; }
    store_vec<T, VEC / 2, SH>(p, lo);
    store_vec<T, VEC / 2, SH>(p + VEC / 2, hi);
  } else if constexpr (VEC == 4) {
    if constexpr (SH == 1) __stcs(reinterpret_cast<float4*>(p), make_float4(a.v[0], a.v[1], a.v[2], a.v[3]));
    else *reinterpret_cast<float4*>(p) = make_float4(a.v[0], a.v[1], a.v[2], a.v[3]);
  } else if constexpr (VEC == 2) {
    if constexpr (SH == 1) __stcs(reinterpret_cast<double2*>(p), make_double2(a.v[0], a.v[1]));
    else *reinterpret_cast<double2*>(p) = make_double2(a.v[0], a.v[1]);
  } else {
    p[0] = a.v[0];
  }
}

// streaming reads of the CSR arrays (each entry is used once per hop)
template <typename V>
__device__ __forceinline__ V ld_stream(const V* p) { return __ldcs(p); }

// streaming (ld.global.cs) 16-byte read: one half of a 32-byte lane, or a whole 16-byte lane
template <typename T, int H>
__device__ __forceinline__ Acc<T, H> load_stream_16(const T* p) {
  static_assert(H * sizeof(T) == 16, "16-byte reads only");
  Acc<T, H> a;
  if constexpr (sizeof(T) == 4) {
    const float4 t = __ldcs(reinterpret_cast<const float4*>(p));
    a.v[0] = t.x; a.v[1] = t.y; a.v[2] = t.z; a.v[3] = t.w;
  } else {
    const double2 t = __ldcs(reinterpret_cast<const double2*>(p));
    a.v[0] = t.x; a.v[1] = t.y;
  }
  return a;
}

// *p += a for one 16-byte fp32 half, as a reduction in the L2 (red.add.v4.f32) with L2 policy `pol`.  The sum is
// p[i] + a[i], the operands of the read-add-write it replaces and so the same bits, except that the reduction flushes
// subnormal operands and results to zero.  Two adds to one address in a launch would land in either order, so the bits
// would vary from run to run: each caller's address belongs to its lane alone, and the stream orders the launches.
__device__ __forceinline__ void red_add_16(float* p, const Acc<float, 4>& a, uint64_t pol) {
  asm volatile("red.relaxed.gpu.global.add.L2::cache_hint.v4.f32 [%0], {%1,%2,%3,%4}, %5;"
               :: "l"(p), "f"(a.v[0]), "f"(a.v[1]), "f"(a.v[2]), "f"(a.v[3]), "l"(pol) : "memory");
}

constexpr unsigned FULL = 0xffffffffu;

// Fused hop + collective (feature-sharded multi-GPU path): besides the local result row, each computed row slice is
// stored straight into the row-local contraction operand of the rank that owns that node row, through NVLink peer
// pointers (st.global on IPC-mapped memory).  Row r goes to peer r / rows_per_peer, local row r % rows_per_peer;
// local column (b, g) = b*gl + g lands at b*stride_b + out_col + g.  n_peers == 0 turns it off.
constexpr int MAX_PEERS = 16;
template <typename T>
struct ScatterArgs {
  T* peer[MAX_PEERS];
  int64_t rows_per_peer;
  int64_t out_ld;
  int64_t out_col;
  int64_t stride_b;
  int gl;
  int n_peers;
};

template <typename T, int VEC>
__device__ __forceinline__ void scatter_store(const ScatterArgs<T>& sc, int64_t row, int cbase, const Acc<T, VEC>& acc) {
  const int64_t q = row / sc.rows_per_peer;
  const int64_t lr = row - q * sc.rows_per_peer;
  const int b = cbase / sc.gl;
  const int g = cbase - b * sc.gl;
  T* o = sc.peer[q] + lr * sc.out_ld + (int64_t)b * sc.stride_b + sc.out_col + g;
  store_vec<T, VEC, 0>(o, acc);
}

template <typename T, int VEC, int L, int U, int THREADS, int MINB, int HINT, bool PF, int SH = 0>
__global__ void __launch_bounds__(THREADS, MINB)
spmm_hop_kernel(const int64_t* __restrict__ rowptr, const int32_t* __restrict__ col,
                const T* __restrict__ val, const T* __restrict__ src, int64_t src_ld,
                T* __restrict__ dst, int64_t dst_ld, int64_t n_rows, int C, int n_chunks, float l2_frac,
                const ScatterArgs<T> sc) {
  uint64_t pol = 0;
  if constexpr (HINT == 2) pol = evict_last_policy(l2_frac);
  if constexpr (HINT == 3) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  if constexpr (HINT == 4) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 0.5;" : "=l"(pol));
  if constexpr (HINT == 5) asm volatile("createpolicy.fractional.L2::evict_last.L2::evict_first.b64 %0, 0.5;" : "=l"(pol));
  constexpr int S = 32 / L;  // neighbours gathered concurrently by one warp
  const int lane = threadIdx.x & 31;
  const int sub = lane / L;
  const int cl = lane % L;
  const int64_t n_warps = (int64_t)gridDim.x * (THREADS >> 5);
  const int64_t n_items = n_rows * n_chunks;
  int64_t item = (int64_t)blockIdx.x * (THREADS >> 5) + (threadIdx.x >> 5);
  if (item >= n_items) return;

  // software pipeline state: current row (beg, end, c, v), next row (nbeg, nend)
  int64_t row = item % n_rows;
  int64_t beg = __ldg(rowptr + row), end = __ldg(rowptr + row + 1);
  int32_t c = 0;
  T v = T(0);
  if (beg + lane < end) { c = ld_stream(col + beg + lane); v = ld_stream(val + beg + lane); }
  int64_t nbeg = 0, nend = 0;
  if (PF && item + n_warps < n_items) {
    const int64_t nrow = (item + n_warps) % n_rows;
    nbeg = __ldg(rowptr + nrow); nend = __ldg(rowptr + nrow + 1);
  }

  while (true) {
    const int chunk = (int)(item / n_rows);
    row = item - (int64_t)chunk * n_rows;
    const int cbase = chunk * (L * VEC) + cl * VEC;
    const bool col_ok = cbase < C;
    const T* __restrict__ srcc = src + cbase;

    // prefetch: next row's first 32 (col, val), and the rowptr pair of the row after that
    const int64_t next = item + n_warps;
    const bool has_next = next < n_items;
    int32_t nc = 0;
    T nv = T(0);
    int64_t nnbeg = 0, nnend = 0;
    if (PF) {
      if (has_next && nbeg + lane < nend) { nc = ld_stream(col + nbeg + lane); nv = ld_stream(val + nbeg + lane); }
      if (next + n_warps < n_items) {
        const int64_t nnrow = (next + n_warps) % n_rows;
        nnbeg = __ldg(rowptr + nnrow); nnend = __ldg(rowptr + nnrow + 1);
      }
    }

    Acc<T, VEC> acc;
    acc.zero();
    for (int64_t base = beg; base < end; base += 32) {
      if (base != beg) {  // rows longer than 32: fetch the following entries (not prefetched)
        c = 0; v = T(0);
        if (base + lane < end) { c = ld_stream(col + base + lane); v = ld_stream(val + base + lane); }
      }
      const int cnt = (int)((end - base) < 32 ? (end - base) : 32);
#pragma unroll 1
      for (int j = 0; j < cnt; j += S * U) {
        Acc<T, VEC> buf[U];
        T w[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int jj = j + u * S + sub;
          const int32_t cc = __shfl_sync(FULL, c, jj & 31);
          const T ww = __shfl_sync(FULL, v, jj & 31);
          const bool ok = (jj < cnt) && col_ok;
          w[u] = ok ? ww : T(0);
          if (ok) buf[u] = load_vec<T, VEC, HINT>(srcc + (int64_t)cc * src_ld, pol);
          else buf[u].zero();
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
#pragma unroll
          for (int i = 0; i < VEC; ++i) acc.v[i] = fma(w[u], buf[u].v[i], acc.v[i]);
        }
      }
    }
    // fold the S neighbour groups together
#pragma unroll
    for (int off = L; off < 32; off <<= 1) {
#pragma unroll
      for (int i = 0; i < VEC; ++i) acc.v[i] += __shfl_xor_sync(FULL, acc.v[i], off);
    }
    if (sub == 0 && col_ok) {
      store_vec<T, VEC, SH>(dst + row * dst_ld + cbase, acc);
      if (sc.n_peers > 0 && cbase < C) scatter_store<T, VEC>(sc, row, cbase, acc);
    }

    if (!has_next) break;
    item = next;
    if (PF) {
      beg = nbeg; end = nend; c = nc; v = nv;
      nbeg = nnbeg; nend = nnend;
    } else {
      row = item % n_rows;
      beg = __ldg(rowptr + row); end = __ldg(rowptr + row + 1);
      c = 0; v = T(0);
      if (beg + lane < end) { c = ld_stream(col + beg + lane); v = ld_stream(val + beg + lane); }
    }
  }
}


// ---------------------------------------------------------------------------------------------------
// Round-2 hop kernels.
//
// (1) spmm_hop_v2_kernel: the register-path (LDG.128) kernel above with the register pressure removed, so that the
//     40-register / 48-warp configuration no longer spills: 32-bit row and offset arithmetic (IDX = int32 rowptr when
//     nnz < 2^31), leading dimensions as 32-bit (IMAD.WIDE forms the 64-bit address), chunk loop outside the
//     grid-stride row loop (no 64-bit item / n_rows division), and the NVLink scatter arguments compiled out of the
//     plain instantiation (SCATTER = false carries an empty struct).
//
// (2) A variant that stages the gathered rows in shared memory with cp.async and software-pipelines the index chain three
//     units deep was built and was slower than (1); it lives
//     with the sweep tool (tools/spmm_async_variant.cuh), not in the library.
// ---------------------------------------------------------------------------------------------------
// Fused hop + all-gather (node-sharded multi-GPU path): the rank computes rows [row0, row0 + n_rows) of the next hop's
// source matrix and every finished row is written into the full-height matrix of EVERY rank while the gather of the
// following rows is still in flight — either with one multimem.st through the NVSwitch multicast address `mc`
// (egress n_rows*C*s per hop) or, without multicast, with one NVLink peer store per rank (egress (P-1)/P*N*C*s).
template <typename T>
struct BcastArgs {
  T* peer[MAX_PEERS];     // full-height destination [n_total, out_ld] of every rank (own one included)
  T* mc;                  // multicast alias of the same buffer, or nullptr
  int64_t row0;           // global index of this rank's first row
  int64_t out_ld;
  int n_peers;
};

template <int VEC>
__device__ __forceinline__ void multimem_store(float* p, const Acc<float, VEC>& a) {
#pragma unroll
  for (int i = 0; i < VEC; i += 4)
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p + i), "f"(a.v[i]), "f"(a.v[i + 1]),
                 "f"(a.v[i + 2]), "f"(a.v[i + 3]) : "memory");
}
template <int VEC>
__device__ __forceinline__ void multimem_store(double* p, const Acc<double, VEC>& a) {
  // multimem.st has no f64 vector form; a store moves bits, so two doubles travel as one .v4.f32
#pragma unroll
  for (int i = 0; i < VEC; i += 2)
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p + i),
                 "f"(__int_as_float(__double2loint(a.v[i]))), "f"(__int_as_float(__double2hiint(a.v[i]))),
                 "f"(__int_as_float(__double2loint(a.v[i + 1]))), "f"(__int_as_float(__double2hiint(a.v[i + 1]))) : "memory");
}

template <typename T, int VEC>
__device__ __forceinline__ void bcast_store(const BcastArgs<T>& bc, int64_t row, int cbase, const Acc<T, VEC>& acc) {
  const int64_t off = (bc.row0 + row) * bc.out_ld + cbase;
  if (bc.mc != nullptr) {
    multimem_store<VEC>(bc.mc + off, acc);
  } else {
    for (int q = 0; q < bc.n_peers; ++q) store_vec<T, VEC, 0>(bc.peer[q] + off, acc);
  }
}

// epilogue of the v2 / async kernels.  MODE 0: plain hop; 1: feature-sharded scatter (ScatterArgs); 2: row broadcast.
//                               3 (2-D process grid): both — the row is all-gathered inside the rank's column group AND its
//                               slice is delivered to the row's contraction owner inside the rank's row group.
//                               4: the row slice is added into dst (source windows after the first of a windowed hop).
constexpr int EPI_NONE = 0, EPI_SCATTER = 1, EPI_BCAST = 2, EPI_GRID = 3, EPI_ACCUM = 4;
template <typename T, int MODE>
struct ScatterParam {};
template <typename T>
struct ScatterParam<T, EPI_SCATTER> { ScatterArgs<T> a; };
template <typename T>
struct ScatterParam<T, EPI_BCAST> { BcastArgs<T> a; };
template <typename T>
struct ScatterParam<T, EPI_GRID> { ScatterArgs<T> s; BcastArgs<T> a; };

// Columns of the two 16-byte halves (H = VEC/2 columns each) of lane cl's 32-byte accumulator in a row chunk of L
// lanes, relative to the chunk's first column: the first half starts at lo(cl), the second HI columns after it.
//   SPLIT (the local epilogues, EPI_NONE and EPI_ACCUM): lane cl owns [cl*H, +H) and [L*H + cl*H, +H).  In each of a
//     lane's two 16-byte loads and stores the L lanes of a group cover L*16 contiguous bytes: whole 32-byte sectors
//     (whole 128-byte lines for L >= 8);
//   otherwise (the NVLink epilogues, which store a lane's 32 bytes as one piece): lane cl owns [cl*VEC, +VEC), HI = H.
// Either way a column is summed by the same lane group over the same neighbours in the same order, so both mappings give
// bit-identical sums.  A half is live when it starts below the padded width (C rounded up to VEC): columns
// [0, padded(C)) are written, nothing past them.
template <int VEC, int L, bool SPLIT>
struct LaneMap {
  static constexpr int H = VEC / 2;
  static constexpr int HI = SPLIT ? L * H : H;
  __host__ __device__ static constexpr int lo(int cl) { return SPLIT ? cl * H : cl * VEC; }
};
template <int MODE>
constexpr bool split_lanes = MODE == EPI_NONE || MODE == EPI_ACCUM;
// The v2 kernels take 32-byte lanes (the library) or 16-byte lanes (variants of tools/spmm_sweep.cu).  A 16-byte lane is
// one load and one store, already whole sectors for every two lanes, so it keeps the adjacent map: lane cl owns
// [cl*VEC, +VEC).
template <typename T, int VEC>
constexpr bool wide_lane = VEC * sizeof(T) == 32;
template <typename T, int VEC, int L, int MODE>
using LaneMapOf = LaneMap<VEC, L, wide_lane<T, VEC> && split_lanes<MODE>>;

// a 32-byte lane's two 16-byte halves, at p and p + HI (a half that is not live reads nothing and holds zeros), or a
// 16-byte lane's one load (when lo_ok)
template <typename T, int VEC, int HINT, int HI>
__device__ __forceinline__ Acc<T, VEC> load_lane(const T* p, bool lo_ok, bool hi_ok, uint64_t pol) {
  static_assert(VEC * sizeof(T) == 16 || VEC * sizeof(T) == 32, "16- or 32-byte lanes only");
  if constexpr (!wide_lane<T, VEC>) {
    Acc<T, VEC> a;
    if (lo_ok) a = load_vec<T, VEC, HINT>(p, pol); else a.zero();
    return a;
  }
  constexpr int H = VEC / 2;
  Acc<T, H> lo, hi;
  if (lo_ok) lo = load_vec<T, H, HINT>(p, pol); else lo.zero();
  if (hi_ok) hi = load_vec<T, H, HINT>(p + HI, pol); else hi.zero();
  Acc<T, VEC> a;
#pragma unroll
  for (int i = 0; i < H; ++i) { a.v[i] = lo.v[i]; a.v[H + i] = hi.v[i]; }
  return a;
}

// shared epilogue of the v2 kernels; called for lanes whose first half is live (the peer epilogues: the whole lane)
template <typename T, int VEC, int L, int MODE, int SH>
__device__ __forceinline__ void hop_epilogue(const ScatterParam<T, MODE>& sp, T* __restrict__ dst, int dst_ld, int row, int cbase,
                                             bool hi_ok, const Acc<T, VEC>& acc) {
  static_assert(VEC * sizeof(T) == 16 || VEC * sizeof(T) == 32, "16- or 32-byte lanes only");
  constexpr int H = VEC / 2, HI = LaneMapOf<T, VEC, L, MODE>::HI;
  if constexpr (MODE == EPI_BCAST) {
    bcast_store<T, VEC>(sp.a, row, cbase, acc);              // the rank's own copy is one of the destinations
  } else if constexpr (MODE == EPI_GRID) {
    if (sp.a.n_peers > 0) bcast_store<T, VEC>(sp.a, row, cbase, acc);   // n_peers == 0: last hop of a chain, no all-gather
    else if (dst != nullptr) store_vec<T, VEC, SH>(dst + (int64_t)row * dst_ld + cbase, acc);
    scatter_store<T, VEC>(sp.s, row, cbase, acc);
  } else if constexpr (MODE == EPI_SCATTER) {
    store_vec<T, VEC, SH>(dst + (int64_t)row * dst_ld + cbase, acc);
    if (sp.a.n_peers > 0) scatter_store<T, VEC>(sp.a, row, cbase, acc);
  } else if constexpr (!wide_lane<T, VEC>) {
    // 16-byte lane: one read (EPI_ACCUM) and one store
    T* p = dst + (int64_t)row * dst_ld + cbase;
    Acc<T, VEC> a = acc;
    if constexpr (MODE == EPI_ACCUM) {
      const Acc<T, VEC> d = load_stream_16<T, VEC>(p);
#pragma unroll
      for (int i = 0; i < VEC; ++i) a.v[i] = d.v[i] + a.v[i];
    }
    store_vec<T, VEC, MODE == EPI_ACCUM ? 1 : SH>(p, a);
  } else {
    T* p = dst + (int64_t)row * dst_ld + cbase;
    Acc<T, H> a0, a1;
#pragma unroll
    for (int i = 0; i < H; ++i) { a0.v[i] = acc.v[i]; a1.v[i] = acc.v[H + i]; }
    if constexpr (MODE == EPI_ACCUM && sizeof(T) == 4 && B200GF_HOP_WIN_RED) {
      // fp32: the L2 adds each half into dst and returns nothing, so dst is not read back to the SM, whose warps keep
      // hiding the gathers' latency.  The evict-first policy matches the streaming stores below.  (There is no vector
      // fp64 reduction.)
      uint64_t pol;
      asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
      red_add_16(p, a0, pol);
      if (hi_ok) red_add_16(p + HI, a1, pol);
    } else {
      if constexpr (MODE == EPI_ACCUM) {
        // dst is read and written once per window: streaming (evict-first) accesses keep the gathered window in the L2.
        // Both halves are read before either is written, so that the two reads are in flight together.
        Acc<T, H> d0 = load_stream_16<T, H>(p), d1;
        if (hi_ok) d1 = load_stream_16<T, H>(p + HI); else d1.zero();
#pragma unroll
        for (int i = 0; i < H; ++i) { a0.v[i] = d0.v[i] + a0.v[i]; a1.v[i] = d1.v[i] + a1.v[i]; }
      }
      constexpr int SHs = MODE == EPI_ACCUM ? 1 : SH;
      store_vec<T, H, SHs>(p, a0);
      if (hi_ok) store_vec<T, H, SHs>(p + HI, a1);
    }
  }
}

// HINT: 0/1 no L2 policy; 3 evict_last on every gathered line; 2 evict_last on the fraction l2_frac of the lines (by
// address hash), the rest unchanged; 6 the same with evict_first on the rest.  SH = 1: streaming stores of the result.
template <typename T, typename IDX, int VEC, int L, int U, int THREADS, int MINB, int HINT, int SCATTER, int SH = 0>
__global__ void __launch_bounds__(THREADS, MINB)
spmm_hop_v2_kernel(const IDX* __restrict__ rowptr, const int32_t* __restrict__ col, const T* __restrict__ val,
                   const T* __restrict__ src, int src_ld, T* __restrict__ dst, int dst_ld, int n_rows, int C,
                   float l2_frac, const ScatterParam<T, SCATTER> sp) {
  uint64_t pol = 0;
  if constexpr (HINT == 3) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  if constexpr (HINT == 2) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, %1;" : "=l"(pol) : "f"(l2_frac));
  if constexpr (HINT == 6)
    asm volatile("createpolicy.fractional.L2::evict_last.L2::evict_first.b64 %0, %1;" : "=l"(pol) : "f"(l2_frac));
  constexpr int S = 32 / L;
  using Map = LaneMapOf<T, VEC, L, SCATTER>;
  const int lane = threadIdx.x & 31;
  const int sub = lane / L;
  const int cl = lane % L;
  const int warp0 = blockIdx.x * (THREADS >> 5) + (threadIdx.x >> 5);
  {
    // column chunk = blockIdx.y: the block scheduler hands out all CTAs of chunk 0 first, so the resident warps gather
    // from one column slab at a time (chunk-major order) without a chunk loop in the kernel
    const int cbase = (int)blockIdx.y * (L * VEC) + Map::lo(cl);
    const int Cp = (C + VEC - 1) / VEC * VEC;
    const bool lo_ok = cbase < Cp, hi_ok = cbase + Map::HI < Cp;
    const T* __restrict__ srcc = src + cbase;
    for (int row = warp0; row < n_rows;) {
      IDX p = __ldg(rowptr + row);
      const IDX end = __ldg(rowptr + row + 1);
      Acc<T, VEC> acc;
      acc.zero();
      for (; p < end; p += 32) {
        int32_t c = 0;
        T v = T(0);
        const int cnt = (int)min((IDX)32, end - p);
        if (lane < cnt) { c = ld_stream(col + p + lane); v = ld_stream(val + p + lane); }
#pragma unroll 1
        for (int j = 0; j < cnt; j += S * U) {
          Acc<T, VEC> buf[U];
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const int jj = j + u * S + sub;
            const int32_t cc = __shfl_sync(FULL, c, jj & 31);
            if (jj < cnt) buf[u] = load_lane<T, VEC, HINT, Map::HI>(srcc + (int64_t)cc * src_ld, lo_ok, hi_ok, pol);
            else buf[u].zero();
          }
#pragma unroll
          for (int u = 0; u < U; ++u) {   // weights are shuffled after the loads are in flight (saves U registers)
            const int jj = j + u * S + sub;
            const T ww = __shfl_sync(FULL, v, jj & 31);
            const T w = jj < cnt ? ww : T(0);
#pragma unroll
            for (int i = 0; i < VEC; ++i) acc.v[i] = fma(w, buf[u].v[i], acc.v[i]);
          }
        }
      }
#pragma unroll
      for (int off = L; off < 32; off <<= 1) {
#pragma unroll
        for (int i = 0; i < VEC; ++i) acc.v[i] += __shfl_xor_sync(FULL, acc.v[i], off);
      }
      // lane id and grid size are re-read here (volatile) so that the compiler does not park the loop-invariant store
      // predicate and row stride in local memory to fit the 40-register budget (it did: 24-byte "spill")
      unsigned ln, gdx;
      asm volatile("mov.u32 %0, %%laneid;" : "=r"(ln));
      asm volatile("mov.u32 %0, %%nctaid.x;" : "=r"(gdx));
      if (ln < (unsigned)L && lo_ok) hop_epilogue<T, VEC, L, SCATTER, SH>(sp, dst, dst_ld, row, cbase, hi_ok, acc);
      row += (int)gdx * (THREADS >> 5);
    }
  }
}

// Narrow rows with the v2 treatment (32-bit index math, 32-byte lanes, epilogue selected at compile time): a warp works on
// RPW = 32/GS consecutive rows at once, each group of GS lanes owns one row and its S = GS/L sub-groups of L lanes gather S
// neighbours per load.  C = 8 floats: L = 1 — one lane fetches a whole 32-byte neighbour row.
template <typename T, typename IDX, int VEC, int L, int GS, int U, int THREADS, int MINB, int HINT, int SCATTER>
__global__ void __launch_bounds__(THREADS, MINB)
spmm_hop_multirow_v2_kernel(const IDX* __restrict__ rowptr, const int32_t* __restrict__ col, const T* __restrict__ val,
                            const T* __restrict__ src, int src_ld, T* __restrict__ dst, int dst_ld, int n_rows, int C,
                            const ScatterParam<T, SCATTER> sp) {
  static_assert(GS % L == 0 && GS <= 32 && (GS / L) * U <= GS, "bad multirow geometry");
  constexpr int RPW = 32 / GS;
  constexpr int S = GS / L;
  using Map = LaneMapOf<T, VEC, L, SCATTER>;
  uint64_t pol = 0;
  if constexpr (HINT >= 2) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  const int lane = threadIdx.x & 31;
  const int grp = lane / GS, gl = lane % GS;
  const int sub = gl / L, cl = gl % L;
  const int cbase = Map::lo(cl);
  const int Cp = (C + VEC - 1) / VEC * VEC;
  const bool lo_ok = cbase < Cp, hi_ok = cbase + Map::HI < Cp;
  const T* __restrict__ srcc = src + cbase;
  const int n_warps = gridDim.x * (THREADS >> 5);
  for (int row0 = (blockIdx.x * (THREADS >> 5) + (threadIdx.x >> 5)) * RPW; row0 < n_rows; row0 += n_warps * RPW) {
    const int row = row0 + grp;
    const bool row_ok = row < n_rows;
    const IDX beg = row_ok ? __ldg(rowptr + row) : 0;
    const int len = row_ok ? (int)(__ldg(rowptr + row + 1) - beg) : 0;
    int maxlen = len;  // warp-uniform trip count: the longest of the RPW rows
#pragma unroll
    for (int off = GS; off < 32; off <<= 1) maxlen = max(maxlen, __shfl_xor_sync(FULL, maxlen, off));
    Acc<T, VEC> acc;
    acc.zero();
    for (int b0 = 0; b0 < maxlen; b0 += GS) {
      int32_t c = 0;
      T v = T(0);
      if (b0 + gl < len) { c = ld_stream(col + beg + b0 + gl); v = ld_stream(val + beg + b0 + gl); }
      const int cnt = len - b0;           // entries of my row left in this chunk (may be <= 0)
      const int maxcnt = maxlen - b0;
#pragma unroll
      for (int j = 0; j < GS; j += S * U) {
        if (j >= maxcnt) break;           // warp-uniform
        Acc<T, VEC> buf[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int jj = j + u * S + sub;
          const int32_t cc = __shfl_sync(FULL, c, jj, GS);
          if (jj < cnt) buf[u] = load_lane<T, VEC, HINT, Map::HI>(srcc + (int64_t)cc * src_ld, lo_ok, hi_ok, pol);
          else buf[u].zero();
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int jj = j + u * S + sub;
          const T ww = __shfl_sync(FULL, v, jj, GS);
          const T w = jj < cnt ? ww : T(0);
#pragma unroll
          for (int i = 0; i < VEC; ++i) acc.v[i] = fma(w, buf[u].v[i], acc.v[i]);
        }
      }
    }
#pragma unroll
    for (int off = L; off < GS; off <<= 1) {
#pragma unroll
      for (int i = 0; i < VEC; ++i) acc.v[i] += __shfl_xor_sync(FULL, acc.v[i], off);
    }
    // a row with no entries in a source window after the first leaves its partial sums as they are
    const bool add_ok = SCATTER != EPI_ACCUM || len > 0;
    if (sub == 0 && lo_ok && row_ok && add_ok) hop_epilogue<T, VEC, L, SCATTER, 0>(sp, dst, dst_ld, row, cbase, hi_ok, acc);
  }
}

// Narrow feature rows (C * sizeof(T) <= 128 bytes): one warp per row leaves most lanes idle and the kernel
// latency-bound on the rowptr -> col/val -> gather dependency chain.  Here a warp works on RPW = 32/GS consecutive rows at once: each group of GS lanes owns one row, reads
// its col/val GS entries at a time, and its S = GS/L sub-groups of L lanes gather S neighbours per load.
template <typename T, int VEC, int L, int GS, int U, int THREADS, int MINB, int HINT>
__global__ void __launch_bounds__(THREADS, MINB)
spmm_hop_multirow_kernel(const int64_t* __restrict__ rowptr, const int32_t* __restrict__ col,
                         const T* __restrict__ val, const T* __restrict__ src, int64_t src_ld,
                         T* __restrict__ dst, int64_t dst_ld, int64_t n_rows, int C, const ScatterArgs<T> sc) {
  static_assert(GS % L == 0 && GS <= 32 && (GS / L) * U <= GS, "bad multirow geometry");
  constexpr int RPW = 32 / GS;
  constexpr int S = GS / L;
  uint64_t pol = 0;
  if constexpr (HINT >= 2) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  const int lane = threadIdx.x & 31;
  const int grp = lane / GS, gl = lane % GS;
  const int sub = gl / L, cl = gl % L;
  const int cbase = cl * VEC;
  const bool col_ok = cbase < C;
  const T* __restrict__ srcc = src + cbase;
  const int64_t n_warps = (int64_t)gridDim.x * (THREADS >> 5);
  const int64_t warp_global = (int64_t)blockIdx.x * (THREADS >> 5) + (threadIdx.x >> 5);
  for (int64_t row0 = warp_global * RPW; row0 < n_rows; row0 += n_warps * RPW) {
    const int64_t row = row0 + grp;
    const bool row_ok = row < n_rows;
    const int64_t beg = row_ok ? __ldg(rowptr + row) : 0;
    const int len = row_ok ? (int)(__ldg(rowptr + row + 1) - beg) : 0;
    int maxlen = len;  // warp-uniform trip count: the longest of the RPW rows
#pragma unroll
    for (int off = GS; off < 32; off <<= 1) maxlen = max(maxlen, __shfl_xor_sync(FULL, maxlen, off));
    Acc<T, VEC> acc;
    acc.zero();
    for (int b0 = 0; b0 < maxlen; b0 += GS) {
      int32_t c = 0;
      T v = T(0);
      if (b0 + gl < len) { c = ld_stream(col + beg + b0 + gl); v = ld_stream(val + beg + b0 + gl); }
      const int cnt = len - b0;           // entries of my row left in this chunk (may be <= 0)
      const int maxcnt = maxlen - b0;
#pragma unroll
      for (int j = 0; j < GS; j += S * U) {
        if (j >= maxcnt) break;           // warp-uniform
        Acc<T, VEC> buf[U];
        T w[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int jj = j + u * S + sub;
          const int32_t cc = __shfl_sync(FULL, c, jj, GS);
          const T ww = __shfl_sync(FULL, v, jj, GS);
          const bool ok = (jj < cnt) && col_ok;
          w[u] = ok ? ww : T(0);
          if (ok) buf[u] = load_vec<T, VEC, HINT>(srcc + (int64_t)cc * src_ld, pol);
          else buf[u].zero();
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
#pragma unroll
          for (int i = 0; i < VEC; ++i) acc.v[i] = fma(w[u], buf[u].v[i], acc.v[i]);
        }
      }
    }
#pragma unroll
    for (int off = L; off < GS; off <<= 1) {
#pragma unroll
      for (int i = 0; i < VEC; ++i) acc.v[i] += __shfl_xor_sync(FULL, acc.v[i], off);
    }
    if (sub == 0 && col_ok && row_ok) {
      store_vec<T, VEC, 0>(dst + row * dst_ld + cbase, acc);
      if (sc.n_peers > 0) scatter_store<T, VEC>(sc, row, cbase, acc);
    }
  }
}

}  // namespace b200gf
