// Edge-gated graph recurrent layer (EdgeGatedHiddenState, alegnn/utils/graphML.py:4033-4209), sparse execution.
//
// The reference builds two dense B*T x N x N attention GSOs per forward (learnAttentionGSO, graphML.py:640-737) and
// shifts every sample against every sample's gated GSO before keeping the diagonal (graphML.py:1425-1431, :1492-1498).
// Everything it needs lives on the non-zeros of S + I, so the kernels here work per non-zero:
//
//   attention  alpha[q, b] = softmax over the mask row i of  LeakyReLU_0.2(a1 s[j, b] + a2 s[i, b]),   q = (i, j)
//              (the graph attention layers, attention.py, score the two ends with two arrays and the mixer (1, 1):
//               LeakyReLU_0.2(s_src[j, b] + s_dst[i, b]), b200gf_attention_forward / _backward)
//              mask = |S + I| > 1e-9 (graphML.py:692, :726-728), a = the gate's mixer, s = W z_gate (one scalar per
//              node and sample).  The FIRST mixer half multiplies the COLUMN node j (graphML.py:706-712).
//   gated hop  dst[j, (b, c)] = sum_i S_ij alpha[b, p(i, j)] src[i, (b, c)]         row-vector shift u S~, S~ = alpha (.) S
//              over the CSR of S^T; p(i, j) = position of (i, j) in the mask CSR, -1 when it is outside the mask.
//
// Layouts: s, dsig1, dsig2 [N, Bs] and alpha, dalpha, dlogit [nnz_mask, Bs] have the sample index innermost, so one
// index / value load of the pattern is shared by the adjacent lanes of a warp and every data access of a row is
// coalesced (as in ev.cu).  The hop's gate pointer takes a sample and a non-zero stride, so the input filter (all B*T
// samples) and the hidden filter at step t (the B samples of one time slab) read one gate buffer without copies.
// Node-major signals: [rows, ld], column b*C + c.
//
// Every output element has exactly one writer and every sum runs in a fixed order: no atomics, bitwise reproducible.
#include "common.cuh"

namespace b200gf {
namespace egate {

template <typename T>
__device__ __forceinline__ T leaky(T v) { return v > T(0) ? v : T(0.2) * v; }
__device__ __forceinline__ float ex(float v) { return expf(v); }
__device__ __forceinline__ double ex(double v) { return exp(v); }

// one thread per (mask row i, sample b): three passes over the row (max, exp + sum, scale).  s_src is read at the
// column node j, s_dst at the row node i (edge gating passes its one score array as both; the graph attention layers
// pass the mixer (1, 1), so that their logit is s_src[j] + s_dst[i])
template <typename T>
__global__ __launch_bounds__(256) void egate_softmax_kernel(const int64_t* __restrict__ rowptr,
                                                            const int32_t* __restrict__ col,
                                                            const T* __restrict__ s_src, const T* __restrict__ s_dst,
                                                            const T* __restrict__ mixer, T* __restrict__ alpha, int Bs,
                                                            int64_t total /* N * Bs */) {
  const T a1 = mixer[0], a2 = mixer[1];
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(t % Bs);
    const int64_t i = t / Bs;
    const int64_t beg = rowptr[i], end = rowptr[i + 1];
    if (beg == end) continue;
    const T si = a2 * s_dst[i * Bs + b];
    T m = -INFINITY;
    for (int64_t q = beg; q < end; ++q) m = fmax(m, leaky(a1 * s_src[(int64_t)col[q] * Bs + b] + si));
    T sum = T(0);
    for (int64_t q = beg; q < end; ++q) {
      const T w = ex(leaky(a1 * s_src[(int64_t)col[q] * Bs + b] + si) - m);
      alpha[q * Bs + b] = w;
      sum += w;
    }
    const T inv = T(1) / sum;
    for (int64_t q = beg; q < end; ++q) alpha[q * Bs + b] *= inv;
  }
}

// softmax + LeakyReLU backward, one thread per (mask row i, sample b):
//   dlogit[q] = alpha[q] (dalpha[q] - sum_row alpha dalpha) * LeakyReLU'(e[q]);   dsig2[i] = sum_row dlogit
template <typename T>
__global__ __launch_bounds__(256) void egate_softmax_bwd_kernel(const int64_t* __restrict__ rowptr,
                                                                const int32_t* __restrict__ col,
                                                                const T* __restrict__ s_src, const T* __restrict__ s_dst,
                                                                const T* __restrict__ mixer, const T* __restrict__ alpha,
                                                                const T* __restrict__ dalpha, T* __restrict__ dlogit,
                                                                T* __restrict__ dsig2, int Bs, int64_t total) {
  const T a1 = mixer[0], a2 = mixer[1];
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(t % Bs);
    const int64_t i = t / Bs;
    const int64_t beg = rowptr[i], end = rowptr[i + 1];
    T dot = T(0);
    for (int64_t q = beg; q < end; ++q) dot = fma(alpha[q * Bs + b], dalpha[q * Bs + b], dot);
    const T si = a2 * s_dst[i * Bs + b];
    T acc = T(0);
    for (int64_t q = beg; q < end; ++q) {
      const T de = alpha[q * Bs + b] * (dalpha[q * Bs + b] - dot);
      const T dl = a1 * s_src[(int64_t)col[q] * Bs + b] + si > T(0) ? de : T(0.2) * de;
      dlogit[q * Bs + b] = dl;
      acc += dl;
    }
    dsig2[t] = acc;
  }
}

// dsig1[j, b] = sum over the mask entries (i, j) of column j of dlogit: a gather over the transposed mask pattern
template <typename T>
__global__ __launch_bounds__(256) void egate_colsum_kernel(const int64_t* __restrict__ rowptrT,
                                                           const int32_t* __restrict__ permT,
                                                           const T* __restrict__ dlogit, T* __restrict__ dsig1, int Bs,
                                                           int64_t total) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(t % Bs);
    const int64_t j = t / Bs;
    T acc = T(0);
    for (int64_t it = rowptrT[j]; it < rowptrT[j + 1]; ++it) acc += dlogit[(int64_t)permT[it] * Bs + b];
    dsig1[t] = acc;
  }
}

template <typename T, int V>
struct Vec {
  T v[V];
};
template <typename T, int V>
__device__ __forceinline__ Vec<T, V> vload(const T* p) {
  Vec<T, V> r;
  if constexpr (V == 4 && sizeof(T) == 4) {
    const float4 a = *reinterpret_cast<const float4*>(p);
    r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
  } else if constexpr (V == 2 && sizeof(T) == 8) {
    const double2 a = *reinterpret_cast<const double2*>(p);
    r.v[0] = a.x; r.v[1] = a.y;
  } else {
#pragma unroll
    for (int u = 0; u < V; ++u) r.v[u] = p[u];
  }
  return r;
}
template <typename T, int V>
__device__ __forceinline__ void vstore(T* p, const Vec<T, V>& a) {
  if constexpr (V == 4 && sizeof(T) == 4) {
    *reinterpret_cast<float4*>(p) = make_float4(a.v[0], a.v[1], a.v[2], a.v[3]);
  } else if constexpr (V == 2 && sizeof(T) == 8) {
    *reinterpret_cast<double2*>(p) = make_double2(a.v[0], a.v[1]);
  } else {
#pragma unroll
    for (int u = 0; u < V; ++u) p[u] = a.v[u];
  }
}

// dst[r, (b, c)] = sum_{it in row r} val[it] * gate[b, pos[it]] * src[col[it], (b, c)]
// One thread owns V consecutive columns of one sample (C % V == 0) of one row; the row's index, value and position
// loads are shared by the lanes of that row, the gate load by the lanes of one sample.
template <typename T, int V>
__global__ __launch_bounds__(256) void egate_hop_kernel(const int64_t* __restrict__ rowptr,
                                                        const int32_t* __restrict__ col, const T* __restrict__ val,
                                                        const int32_t* __restrict__ pos, const T* __restrict__ gate,
                                                        int64_t g_sb, int64_t g_sp, const T* __restrict__ src,
                                                        int64_t src_ld, T* __restrict__ dst, int64_t dst_ld, int C,
                                                        int64_t per_row /* Bs*C/V */, int64_t total) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t c0 = (t % per_row) * V;
    const int64_t r = t / per_row;
    const T* __restrict__ g = gate + (c0 / C) * g_sb;
    Vec<T, V> acc;
#pragma unroll
    for (int u = 0; u < V; ++u) acc.v[u] = T(0);
    const int64_t beg = rowptr[r], end = rowptr[r + 1];
    for (int64_t it = beg; it < end; ++it) {
      const int32_t p = pos[it];
      if (p < 0) continue;                                       // S entry outside the mask: gated to zero
      const T w = g[(int64_t)p * g_sp] * val[it];
      const Vec<T, V> x = vload<T, V>(src + (int64_t)col[it] * src_ld + c0);
#pragma unroll
      for (int u = 0; u < V; ++u) acc.v[u] = fma(w, x.v[u], acc.v[u]);
    }
    vstore<T, V>(dst + r * dst_ld + c0, acc);
  }
}

// dgate[b, q] = m_sval[q] * sum_c src[i, (b, c)] * ddst[j, (b, c)]  for every mask entry q = (i, j) (SDDMM on the mask;
// m_sval = S_ij, 0 where the mask has no S entry).  One thread per (mask row i, sample b).
template <typename T>
__global__ __launch_bounds__(256) void egate_sddmm_kernel(const int64_t* __restrict__ m_rowptr,
                                                          const int32_t* __restrict__ m_col,
                                                          const T* __restrict__ m_sval, const T* __restrict__ src,
                                                          int64_t src_ld, const T* __restrict__ ddst, int64_t ddst_ld,
                                                          T* __restrict__ dgate, int64_t d_sb, int64_t d_sp, int Bs,
                                                          int C, int64_t total /* N * Bs */) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(t % Bs);
    const int64_t i = t / Bs;
    const T* __restrict__ si = src + i * src_ld + (int64_t)b * C;
    T* __restrict__ out = dgate + b * d_sb;
    for (int64_t q = m_rowptr[i]; q < m_rowptr[i + 1]; ++q) {
      const T sv = m_sval[q];
      T acc = T(0);
      if (sv != T(0)) {
        const T* __restrict__ dj = ddst + (int64_t)m_col[q] * ddst_ld + (int64_t)b * C;
        for (int c = 0; c < C; ++c) acc = fma(si[c], dj[c], acc);
      }
      out[q * d_sp] = sv * acc;
    }
  }
}

template <typename T>
int attention_forward_t(int64_t N, int Bs, const int64_t* rowptr, const int32_t* col, const T* s_src, const T* s_dst,
                        const T* mixer, T* alpha, cudaStream_t st) {
  const int64_t total = N * Bs;
  if (total == 0) return B200GF_OK;
  egate_softmax_kernel<T><<<grid_for(total, 256, 132 * 16), 256, 0, st>>>(rowptr, col, s_src, s_dst, mixer, alpha, Bs,
                                                                          total);
  LAUNCH_CHECK();
  return B200GF_OK;
}

template <typename T>
int attention_backward_t(int64_t N, int Bs, const int64_t* rowptr, const int32_t* col, const int64_t* rowptrT,
                         const int32_t* permT, const T* s_src, const T* s_dst, const T* mixer, const T* alpha,
                         const T* dalpha, T* dlogit, T* dsig1, T* dsig2, cudaStream_t st) {
  const int64_t total = N * Bs;
  if (total == 0) return B200GF_OK;
  const int grid = grid_for(total, 256, 132 * 16);
  egate_softmax_bwd_kernel<T><<<grid, 256, 0, st>>>(rowptr, col, s_src, s_dst, mixer, alpha, dalpha, dlogit, dsig2, Bs,
                                                    total);
  LAUNCH_CHECK();
  egate_colsum_kernel<T><<<grid, 256, 0, st>>>(rowptrT, permT, dlogit, dsig1, Bs, total);
  LAUNCH_CHECK();
  return B200GF_OK;
}

template <typename T, int V>
inline bool vec_ok(int C, int64_t a_ld, int64_t b_ld, const void* a, const void* b) {
  if (V == 1) return true;
  const uintptr_t bits = reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b);
  return C % V == 0 && a_ld % V == 0 && b_ld % V == 0 && (bits & 15) == 0;
}

template <typename T>
int hop_t(int64_t n_rows, int Bs, int C, const int64_t* rowptr, const int32_t* col, const T* val, const int32_t* pos,
          const T* gate, int64_t g_sb, int64_t g_sp, const T* src, int64_t src_ld, T* dst, int64_t dst_ld,
          cudaStream_t st) {
  const int64_t cols = (int64_t)Bs * C;
  if (n_rows == 0 || cols == 0) return B200GF_OK;
  constexpr int VV = sizeof(T) == 4 ? 4 : 2;                     // one 16-byte access per lane
  if (vec_ok<T, VV>(C, src_ld, dst_ld, src, dst)) {
    const int64_t per_row = cols / VV;
    egate_hop_kernel<T, VV><<<grid_for(n_rows * per_row, 256, 132 * 16), 256, 0, st>>>(
        rowptr, col, val, pos, gate, g_sb, g_sp, src, src_ld, dst, dst_ld, C, per_row, n_rows * per_row);
  } else {
    egate_hop_kernel<T, 1><<<grid_for(n_rows * cols, 256, 132 * 16), 256, 0, st>>>(
        rowptr, col, val, pos, gate, g_sb, g_sp, src, src_ld, dst, dst_ld, C, cols, n_rows * cols);
  }
  LAUNCH_CHECK();
  return B200GF_OK;
}

template <typename T>
int hop_backward_t(int64_t N, int Bs, int C, const int64_t* rowptr, const int32_t* col, const T* val,
                   const int32_t* pos, const int64_t* m_rowptr, const int32_t* m_col, const T* m_sval, const T* gate,
                   int64_t g_sb, int64_t g_sp, const T* src, int64_t src_ld, const T* ddst, int64_t ddst_ld, T* dsrc,
                   int64_t dsrc_ld, T* dgate, int64_t d_sb, int64_t d_sp, cudaStream_t st) {
  if (dsrc) {
    const int rc = hop_t<T>(N, Bs, C, rowptr, col, val, pos, gate, g_sb, g_sp, ddst, ddst_ld, dsrc, dsrc_ld, st);
    if (rc != B200GF_OK) return rc;
  }
  if (dgate && N * Bs > 0) {
    egate_sddmm_kernel<T><<<grid_for(N * Bs, 256, 132 * 16), 256, 0, st>>>(m_rowptr, m_col, m_sval, src, src_ld, ddst,
                                                                           ddst_ld, dgate, d_sb, d_sp, Bs, C, N * Bs);
    LAUNCH_CHECK();
  }
  return B200GF_OK;
}

}  // namespace egate
}  // namespace b200gf

extern "C" {

int b200gf_attention_forward(int dtype, int64_t N, int64_t nnz, int Bs, const int64_t* rowptr, const int32_t* col,
                             const void* s_src, const void* s_dst, const void* mixer, void* alpha, void* stream) {
  using namespace b200gf;
  if (N < 0 || nnz < 0 || Bs <= 0) return B200GF_EINVAL;
  if (!rowptr || !s_src || !s_dst || !mixer || (nnz > 0 && (!col || !alpha))) return B200GF_EINVAL;
  if (N > INT32_MAX || nnz > INT32_MAX) return B200GF_EUNSUPPORTED;
  return with_dtype(dtype, [&](auto tag) {
    using T = decltype(tag);
    return egate::attention_forward_t<T>(N, Bs, rowptr, col, (const T*)s_src, (const T*)s_dst, (const T*)mixer, (T*)alpha,
                                         (cudaStream_t)stream);
  });
}

int b200gf_attention_backward(int dtype, int64_t N, int64_t nnz, int Bs, const int64_t* rowptr, const int32_t* col,
                              const int64_t* rowptrT, const int32_t* permT, const void* s_src, const void* s_dst,
                              const void* mixer, const void* alpha, const void* dalpha, void* dlogit, void* dsig1, void* dsig2,
                              void* stream) {
  using namespace b200gf;
  if (N < 0 || nnz < 0 || Bs <= 0) return B200GF_EINVAL;
  if (!rowptr || !rowptrT || !s_src || !s_dst || !mixer || !dsig1 || !dsig2) return B200GF_EINVAL;
  if (nnz > 0 && (!col || !permT || !alpha || !dalpha || !dlogit)) return B200GF_EINVAL;
  if (N > INT32_MAX || nnz > INT32_MAX) return B200GF_EUNSUPPORTED;
  return with_dtype(dtype, [&](auto tag) {
    using T = decltype(tag);
    return egate::attention_backward_t<T>(N, Bs, rowptr, col, rowptrT, permT, (const T*)s_src, (const T*)s_dst,
                                          (const T*)mixer, (const T*)alpha, (const T*)dalpha, (T*)dlogit, (T*)dsig1,
                                          (T*)dsig2, (cudaStream_t)stream);
  });
}

// edge gating: the attention softmax with one score array s for both ends of an edge
int b200gf_egate_attention_forward(int dtype, int64_t N, int64_t nnz, int Bs, const int64_t* rowptr,
                                   const int32_t* col, const void* s, const void* mixer, void* alpha, void* stream) {
  return b200gf_attention_forward(dtype, N, nnz, Bs, rowptr, col, s, s, mixer, alpha, stream);
}

int b200gf_egate_attention_backward(int dtype, int64_t N, int64_t nnz, int Bs, const int64_t* rowptr,
                                    const int32_t* col, const int64_t* rowptrT, const int32_t* permT, const void* s,
                                    const void* mixer, const void* alpha, const void* dalpha, void* dlogit,
                                    void* dsig1, void* dsig2, void* stream) {
  return b200gf_attention_backward(dtype, N, nnz, Bs, rowptr, col, rowptrT, permT, s, s, mixer, alpha, dalpha, dlogit,
                                   dsig1, dsig2, stream);
}

int b200gf_gated_hop_forward(int dtype, int64_t N, int Bs, int C, const int64_t* rowptrT, const int32_t* colT,
                             const void* valT, const int32_t* posT, const void* gate, int64_t gate_sb, int64_t gate_sp,
                             const void* src, int64_t src_ld, void* dst, int64_t dst_ld, void* stream) {
  using namespace b200gf;
  if (N < 0 || Bs <= 0 || C <= 0) return B200GF_EINVAL;
  if (!rowptrT || !colT || !valT || !posT || !gate || !src || !dst) return B200GF_EINVAL;
  if (src_ld < (int64_t)Bs * C || dst_ld < (int64_t)Bs * C) return B200GF_EINVAL;
  if (N > INT32_MAX) return B200GF_EUNSUPPORTED;
  return with_dtype(dtype, [&](auto tag) {
    using T = decltype(tag);
    return egate::hop_t<T>(N, Bs, C, rowptrT, colT, (const T*)valT, posT, (const T*)gate, gate_sb, gate_sp, (const T*)src,
                           src_ld, (T*)dst, dst_ld, (cudaStream_t)stream);
  });
}

int b200gf_gated_hop_backward(int dtype, int64_t N, int Bs, int C, const int64_t* rowptr, const int32_t* col,
                              const void* val, const int32_t* pos, const int64_t* m_rowptr, const int32_t* m_col,
                              const void* m_sval, const void* gate, int64_t gate_sb, int64_t gate_sp, const void* src,
                              int64_t src_ld, const void* ddst, int64_t ddst_ld, void* dsrc, int64_t dsrc_ld,
                              void* dgate, int64_t dgate_sb, int64_t dgate_sp, void* stream) {
  using namespace b200gf;
  if (N < 0 || Bs <= 0 || C <= 0 || (!dsrc && !dgate) || !ddst) return B200GF_EINVAL;
  if (dsrc && (!rowptr || !col || !val || !pos || !gate || dsrc_ld < (int64_t)Bs * C)) return B200GF_EINVAL;
  if (dgate && (!m_rowptr || !m_col || !m_sval || !src || src_ld < (int64_t)Bs * C)) return B200GF_EINVAL;
  if (ddst_ld < (int64_t)Bs * C) return B200GF_EINVAL;
  if (N > INT32_MAX) return B200GF_EUNSUPPORTED;
  return with_dtype(dtype, [&](auto tag) {
    using T = decltype(tag);
    return egate::hop_backward_t<T>(N, Bs, C, rowptr, col, (const T*)val, pos, m_rowptr, m_col, (const T*)m_sval,
                                    (const T*)gate, gate_sb, gate_sp, (const T*)src, src_ld, (const T*)ddst, ddst_ld,
                                    (T*)dsrc, dsrc_ld, (T*)dgate, dgate_sb, dgate_sp, (cudaStream_t)stream);
  });
}

}  // extern "C"
