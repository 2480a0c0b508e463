// Internal helpers shared by the b200gf translation units (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
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
};

inline size_t dtype_size(int dtype) { return dtype == B200GF_F64 ? 8 : 4; }
__host__ __device__ inline int64_t imin64(int64_t a, int64_t b) { return a < b ? a : b; }
inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// padded node-major row length (elements): rows start 16-byte aligned and cover whole 32-byte sectors
inline int64_t padded_ld(int64_t C, int dtype) {
  const int64_t q = 32 / (int64_t)dtype_size(dtype);
  return (C + q - 1) / q * q;
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
int launch_scatter_rows(int dtype, const void* src, int64_t src_ld, int64_t n_rows, int C, cudaStream_t st,
                        const ScatterHost* sh);
int launch_bcast_rows(int dtype, const void* src, int64_t src_ld, int64_t n_rows, int C, cudaStream_t st,
                      const BcastHost* bh);

struct TermList {            // passed by value to kernels: up to MAX_TERMS (pointer, ld) pairs
  static constexpr int MAX_TERMS = 48;
  const void* ptr[MAX_TERMS];
  int64_t ld[MAX_TERMS];
};

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
}
