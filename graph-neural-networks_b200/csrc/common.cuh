// Internal helpers shared by the b200gf translation units (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include <algorithm>
#include <atomic>
#include <type_traits>
#include <vector>

#include "../../include/b200gf.h"

#define B200GF_VERSION 100

#define CUDA_TRY(expr)                                               \
  do {                                                               \
    cudaError_t _e = (expr);                                         \
    if (_e != cudaSuccess) return B200GF_ECUDA - (int)_e;            \
  } while (0)

// after every kernel launch (or group of n launches): error check + the library's launch counter (b200gf_launch_count)
#define LAUNCH_CHECK_N(n)                                            \
  do {                                                               \
    cudaError_t _e = cudaGetLastError();                             \
    if (_e != cudaSuccess) return B200GF_ECUDA - (int)_e;            \
    b200gf::g_launch_count.fetch_add((n), std::memory_order_relaxed); \
  } while (0)
#define LAUNCH_CHECK() LAUNCH_CHECK_N(1)

namespace b200gf {

extern std::atomic<long long> g_launch_count;  // kernels launched by this library in this process (plan.cu)

struct CsrDev {
  int64_t* rowptr = nullptr;  // [n_rows + 1]
  int32_t* rowptr32 = nullptr;  // the same offsets as int32 when nnz < 2^31 (hop kernel v2: 32-bit index math), else null
  int32_t* col = nullptr;     // [nnz]
  void* val = nullptr;        // [nnz] of dtype
  int64_t nnz = 0;
  bool owned = true;          // false when it aliases the other direction (symmetric GSO)
  // most non-zeros lie far from the diagonal, so a hop's gathers spread over the whole source (hop_chunk_lanes);
  // set by b200gf_plan_create, which sees the host CSR
  bool spread = false;
  // window-major copy of the operator (b200gf_plan_set_hop_windows): window w holds the entries whose column lies in
  // [w * win_rows, (w + 1) * win_rows), as a full-height CSR with offsets win_rowptr32[w * (n_rows + 1) ..] into the
  // shared win_col / win_val (window 0's entries first).  Columns stay global.  win_rows == 0: no copy.
  int64_t win_rows = 0;
  int n_win = 0;
  int32_t* win_rowptr32 = nullptr;  // [n_win * (n_rows + 1)]
  int32_t* win_col = nullptr;       // [nnz]
  void* win_val = nullptr;          // [nnz] of dtype
};

inline size_t dtype_size(int dtype) { return dtype == B200GF_F64 ? 8 : 4; }
__host__ __device__ inline int64_t imin64(int64_t a, int64_t b) { return a < b ? a : b; }
inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// padded node-major row length (elements): rows start 16-byte aligned and cover whole 32-byte sectors
inline int64_t padded_ld(int64_t C, int dtype) {
  const int64_t q = 32 / (int64_t)dtype_size(dtype);
  return (C + q - 1) / q * q;
}

// f(float{}) or f(double{}) for the dtype, B200GF_EUNSUPPORTED for any other; f names its type as decltype(tag)
template <typename Fn>
int with_dtype(int dtype, Fn&& f) {
  if (dtype == B200GF_F32) return f(float{});
  if (dtype == B200GF_F64) return f(double{});
  return B200GF_EUNSUPPORTED;
}

// blocks of `threads` for a grid-stride loop over `total` items: one item per thread, at most `cap` blocks, at least one
inline int grid_for(int64_t total, int threads, int64_t cap) {
  return (int)std::max<int64_t>(1, std::min<int64_t>((total + threads - 1) / threads, cap));
}

// rows per piece of the deterministic two-pass sums: about 1024 pieces, at least 32 rows each
inline int64_t piece_rows(int64_t N) { return std::max<int64_t>(32, (N + 1023) / 1024); }

// consecutive 256-byte aligned slices of the caller's workspace; with a null base it only adds up the bytes (off)
struct Carver {
  char* base;
  size_t off = 0;
  explicit Carver(void* p) : base((char*)p) {}
  void* take(size_t bytes) {
    void* r = base ? base + off : nullptr;
    off += align_up(bytes, 256);
    return r;
  }
};

// the caller's workspace: EINVAL when not 256-byte aligned, EWORKSPACE when null although `required` or `need` > 0,
// EWORKSPACE when smaller than `need`
inline int check_workspace(const void* ws, size_t need, size_t have, bool required) {
  if (ws && ((uintptr_t)ws & 255) != 0) return B200GF_EINVAL;
  if (!ws && (required || need > 0)) return B200GF_EWORKSPACE;
  return need > have ? B200GF_EWORKSPACE : B200GF_OK;
}

// type-erased description of the fused NVLink scatter epilogue (spmm_kernels.cuh: ScatterArgs)
struct ScatterHost {
  void* peer[16];
  int64_t rows_per_peer, out_ld, out_col, stride_b;
  int gl, n_peers;
};

// type-erased description of the fused all-gather epilogue (spmm_kernels.cuh: BcastArgs)
struct BcastHost {
  void* peer[16];
  void* mc;
  int64_t row0, out_ld;
  int n_peers;
};

// internal launchers (defined across the .cu files) -------------------------------------------------
// l2_bytes: L2 size the plain hop's column chunks are sized against (hop_chunk_lanes), 0 = row width alone decides
int launch_hop(int dtype, int sm_count, int64_t l2_bytes, const CsrDev& A, int64_t n_rows, const void* src,
               int64_t src_ld, void* dst, int64_t dst_ld, int C, cudaStream_t st, const ScatterHost* sh = nullptr,
               const BcastHost* bh = nullptr);
// rows per source window of the default window-major operator copy, 0 for none (spmm.cu)
int64_t hop_window_rows(int64_t n_src, int64_t l2_bytes, bool spread);
int launch_scatter_rows(int dtype, const void* src, int64_t src_ld, int64_t n_rows, int C, cudaStream_t st,
                        const ScatterHost* sh);
int launch_bcast_rows(int dtype, const void* src, int64_t src_ld, int64_t n_rows, int C, cudaStream_t st,
                      const BcastHost* bh);

struct TermList {            // passed by value to kernels: up to MAX_TERMS (pointer, ld) pairs
  static constexpr int MAX_TERMS = 48;
  const void* ptr[MAX_TERMS];
  int64_t ld[MAX_TERMS];
};

// the first n terms of the arrays zs / z_ld (n <= MAX_TERMS)
inline TermList make_terms(const void* const* zs, const int64_t* z_ld, int n) {
  TermList tl;
  for (int i = 0; i < n; ++i) {
    tl.ptr[i] = zs[i];
    tl.ld[i] = z_ld[i];
  }
  return tl;
}

int launch_tap_contract(int dtype, int64_t n_rows, int B, int P, int Q, int T, const void* const* zs,
                        const int64_t* z_ld, const void* W, const void* bias, int bias_per_node,
                        void* out, int64_t out_ld, int accumulate, cudaStream_t st, int act = 0);

// out_mode 0: dW[t][p][q];  out_mode 1: taps layout dh[F=Q, E, K, G=P] with t=0 broadcast to every e (k=0)
int launch_tap_grad(int dtype, int64_t n_rows, int B, int P, int Q, int T, const void* A, int64_t a_ld,
                    const void* const* vs, const int64_t* v_ld, void* dW, int out_mode, int E, int K,
                    void* scratch, size_t scratch_bytes, cudaStream_t st);
size_t tap_grad_scratch_bytes(int dtype, int64_t n_rows, int B, int P, int Q, int T);

int launch_bias_grad(int dtype, int64_t n_rows, int B, int F, const void* dy, int64_t dy_ld, void* dbias,
                     int bias_per_node, void* scratch, size_t scratch_bytes, cudaStream_t st);
size_t bias_grad_scratch_bytes(int dtype, int64_t n_rows, int B, int F);

// tensor-core (wgmma, 3xTF32) contraction, tc_contract.cu
size_t tc_contract_scratch_bytes(int T, int P, int Q);
bool tc_contract_eligible(int dtype, int64_t n_rows, int B, int P, int Q, int T, const void* const* zs,
                          const int64_t* z_ld, const void* out, int64_t out_ld, int accumulate);
int launch_pack_taps_split(const void* h, void* whi_wlo, int F, int E, int K, int G, int to_input, cudaStream_t st);
int launch_split_w(const void* W, void* whi_wlo, int T, int P, int Q, cudaStream_t st);
int launch_tc_contract(int sm_count, int64_t n_rows, int B, int P, int Q, int T, const void* const* zs,
                       const void* whi_wlo, const void* bias, int bias_per_node, void* out, int64_t out_ld,
                       cudaStream_t st, int act = 0);

// FP64 contraction on DMMA (mma.sync.m8n8k4.f64), dmma_contract.cu; W is the plain [T][P][Q] packing
bool dmma_contract_eligible(int dtype, int64_t n_rows, int B, int P, int Q, int T, const void* const* zs,
                            const int64_t* z_ld, const void* out, int64_t out_ld, int accumulate);
int launch_dmma_contract(int sm_count, int64_t n_rows, int B, int P, int Q, int T, const void* const* zs,
                         const int64_t* z_ld, const void* W, const void* bias, int bias_per_node, void* out,
                         int64_t out_ld, cudaStream_t st, int act);

int launch_pack_taps(int dtype, const void* h, void* W, int F, int E, int K, int G, int transpose_taps,
                     cudaStream_t st);
int launch_to_node_major(int dtype, const void* src, void* dst, int64_t dst_ld, int64_t N, int C,
                         cudaStream_t st);
int launch_to_feature_major(int dtype, const void* src, int64_t src_ld, void* dst, int64_t N, int C,
                            cudaStream_t st);

}  // namespace b200gf

struct b200gf_plan {
  int device = 0;
  int dtype = B200GF_F32;
  int64_t n_rows = 0, n_cols = 0;
  int E = 0;
  int sm_count = 132;
  int64_t l2_bytes = 0;   // device L2 size the hops size their column chunks against (b200gf_plan_set_l2_bytes)
  bool symmetric = false;
  bool has_bwd = false;
  bool from_gso = false;      // built by b200gf_plan_create: the only plans that take window-major operator copies
  std::vector<b200gf::CsrDev> fwd;  // CSR of S_e^T rows: forward shift gather operator
  std::vector<b200gf::CsrDev> bwd;  // CSR of S_e rows  : backward shift gather operator
  // measurement hook (b200gf_profile_hops): event pairs around hop launches
  mutable std::vector<cudaEvent_t> prof_start, prof_stop;
  mutable int prof_used = 0;
};

namespace b200gf {
// hop launch of forward/backward, bracketed with events when profiling is on
int plan_hop(const b200gf_plan* p, const CsrDev& A, const void* src, int64_t src_ld, void* dst, int64_t dst_ld, int C,
             cudaStream_t st, const ScatterHost* sh = nullptr, const BcastHost* bh = nullptr);
// the hop chains z_{e,0} = src, z_{e,k} = z_{e,k-1} · op_e (k = 1 .. K-1) of every edge feature e, ops = plan->fwd or
// plan->bwd.  Hop output t = 1 + e(K-1) + k-1 is written to slot t-1 of buf (n_rows x ld elements per slot); zs / zld
// receive the T = 1 + E(K-1) terms (pointer, ld), zs[0] = src.
int hop_chain(const b200gf_plan* p, const std::vector<CsrDev>& ops, const void* src, int64_t src_ld, void* buf, int64_t ld,
              int C, int K, std::vector<const void*>& zs, std::vector<int64_t>& zld, cudaStream_t st);
}
