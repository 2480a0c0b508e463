// Edge-variant graph filter (EVGF), sparse execution — the variant row of the path (SURVEY.md §8 a-7).
//
// Reference: EVGF(S, x, b), alegnn/utils/graphML.py:389-488, called by EdgeVariantGF.forward (:2670-2698) with
// Phi = weightEV * sparsityPatternFull (:2676).  Per (f, e, g) it runs the chain
//     u_0 = Phi^(0) x_g ,  u_k = Phi^(k) u_{k-1}      (COLUMN convention Phi·x, graphML.py:464,475)
// and sums u_k over k, g, e.  The reference stores every Phi^(k)_{feg} as a dense N x N matrix; only the entries on
// the masked sparsity pattern of |S_e| + I are live (:2620-2663).  Here the live entries are stored per non-zero of
// one CSR pattern (rowptr, col) over a COMPACT node set A of NA nodes (for the hybrid layer: the M selected nodes and
// the nodes adjacent to them — every other row and column of Phi is identically zero), one call per edge feature e.
//
// Round-2 layout: the BATCH index is innermost everywhere,
//     w    [F, K, G, nnz]      Phi^(k) on the pattern
//     xT   [G, NA, B]          input restricted to A
//     U_k  [F*G, NA, B]        chain states u_k (kept for k < K-1: the weight gradient of step k+1 needs them)
//     Y    [F, NA, B]          sum_g sum_k u_k   (the caller sums over e and adds the bias)
// so that the B chains sharing one weight matrix Phi^(k)_{feg} sit in adjacent lanes: one weight / column index is read
// once per warp and broadcast, every state access is a coalesced B*s-byte row (the r1 kernels had the node index
// innermost: every lane read its own weights, states were gathered element-wise, and an extra [F,G,B,NA] running sum
// was read-modified-written once per k).  The sum over g happens in registers (one thread owns (f, i, b) and loops
// over g), so Y is written once per step.  `diag` (optional, int32 [NA]): position of the diagonal entry of row i in
// the pattern, -1 if it is not live — the layer's k = 0 mask is "identity on the selected nodes" (:2653-2663), so its
// first step is an element-wise product, not a sparse product; without `diag` (functional EVGF with arbitrary matrices)
// k = 0 runs like every other step.
#include "common.cuh"

namespace b200gf {
namespace ev {

// small fixed-size vector of VB batch elements (VB = 4: one 16-byte access when B % 4 == 0 and T = float; else VB = 1)
template <typename T, int VB>
struct BVec {
  T v[VB];
  __device__ __forceinline__ void zero() {
#pragma unroll
    for (int i = 0; i < VB; ++i) v[i] = T(0);
  }
};
template <typename T, int VB>
__device__ __forceinline__ BVec<T, VB> bload(const T* p) {
  BVec<T, VB> r;
  if constexpr (VB == 4 && sizeof(T) == 4) {
    const float4 t = *reinterpret_cast<const float4*>(p);
    r.v[0] = t.x; r.v[1] = t.y; r.v[2] = t.z; r.v[3] = t.w;
  } else {
#pragma unroll
    for (int i = 0; i < VB; ++i) r.v[i] = p[i];
  }
  return r;
}
template <typename T, int VB>
__device__ __forceinline__ void bstore(T* p, const BVec<T, VB>& a) {
  if constexpr (VB == 4 && sizeof(T) == 4) {
    *reinterpret_cast<float4*>(p) = make_float4(a.v[0], a.v[1], a.v[2], a.v[3]);
  } else {
#pragma unroll
    for (int i = 0; i < VB; ++i) p[i] = a.v[i];
  }
}

// step k of every chain (f, g, b) for one edge feature; one thread owns (f, i, VB consecutive b) and loops over g
template <typename T, int VB, int GB = 8>
__global__ void __launch_bounds__(256)
step_kernel(const int64_t* __restrict__ rowptr, const int32_t* __restrict__ col, const int32_t* __restrict__ diag,
            const T* __restrict__ w, const T* __restrict__ uprev, const T* __restrict__ xT, T* __restrict__ ucur,
            T* __restrict__ Y, int NA, int B, int G, int K, int k, int nnz, int64_t total /* F*NA*(B/VB) */) {
  const int BV = B / VB;
  const size_t plane = (size_t)NA * B;                       // one (f, g) state
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(t % BV) * VB;
    const int64_t fi = t / BV;
    const int i = (int)(fi % NA);
    const int f = (int)(fi / NA);
    const int beg = (int)rowptr[i], end = (int)rowptr[i + 1];
    const int32_t d = (k == 0 && diag) ? diag[i] : -2;        // -2: ordinary sparse step
    BVec<T, VB> ysum;
    ysum.zero();
    const T* __restrict__ wk = w + ((size_t)(f * K + k) * G) * nnz;                    // + g * nnz
    const T* __restrict__ up = (k == 0 ? xT : uprev + (size_t)f * G * plane) + b;      // + g * plane
    T* __restrict__ uc = ucur ? ucur + (size_t)f * G * plane + (size_t)i * B + b : nullptr;
    // GB input features at a time: their loads (one weight + one state row each per non-zero) are independent, so GB
    // requests are in flight per thread instead of one (the one-g-at-a-time loop stalls on each load in turn)
    for (int g0 = 0; g0 < G; g0 += GB) {
      BVec<T, VB> acc[GB];
#pragma unroll
      for (int q = 0; q < GB; ++q) acc[q].zero();
      if (d != -2) {
        if (d >= 0) {
#pragma unroll
          for (int q = 0; q < GB; ++q) {
            if (g0 + q < G) {
              const T wv = wk[(size_t)(g0 + q) * nnz + d];
              const BVec<T, VB> u = bload<T, VB>(up + (size_t)(g0 + q) * plane + (size_t)i * B);
#pragma unroll
              for (int r = 0; r < VB; ++r) acc[q].v[r] = wv * u.v[r];
            }
          }
        }
      } else {
        for (int idx = beg; idx < end; ++idx) {
          const size_t cb = (size_t)col[idx] * B;
#pragma unroll
          for (int q = 0; q < GB; ++q) {
            if (g0 + q < G) {
              const T wv = wk[(size_t)(g0 + q) * nnz + idx];
              const BVec<T, VB> u = bload<T, VB>(up + (size_t)(g0 + q) * plane + cb);
#pragma unroll
              for (int r = 0; r < VB; ++r) acc[q].v[r] = fma(wv, u.v[r], acc[q].v[r]);
            }
          }
        }
      }
#pragma unroll
      for (int q = 0; q < GB; ++q) {
        if (g0 + q < G) {
          if (uc) bstore<T, VB>(uc + (size_t)(g0 + q) * plane, acc[q]);
#pragma unroll
          for (int r = 0; r < VB; ++r) ysum.v[r] += acc[q].v[r];
        }
      }
    }
    T* __restrict__ y = Y + ((size_t)f * NA + i) * B + b;
    if (k != 0) {
      const BVec<T, VB> old = bload<T, VB>(y);
#pragma unroll
      for (int q = 0; q < VB; ++q) ysum.v[q] += old.v[q];
    }
    bstore<T, VB>(y, ysum);
  }
}

// lam_{K-1}[(f,g), i, b] = dY[f, i, b]
template <typename T>
__global__ void adjoint_init_kernel(const T* __restrict__ dY, T* __restrict__ lam, int64_t NA, int B, int G, int64_t total) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t ib = t % (NA * B);
    const int64_t f = (t / (NA * B)) / G;
    lam[t] = dY[f * NA * B + ib];
  }
}

// lam_{k-1}[(f,g), j, b] = dY[f, j, b] + sum_{it in rowT(j)} w_k[perm[it]] * lam_k[(f,g), colT[it], b]        (k >= 1)
template <typename T, int VB>
__global__ void __launch_bounds__(256)
adjoint_step_kernel(const int64_t* __restrict__ rowptrT, const int32_t* __restrict__ colT, const int64_t* __restrict__ perm,
                    const T* __restrict__ w, const T* __restrict__ dY, const T* __restrict__ lam_k, T* __restrict__ lam_km1,
                    int NA, int B, int G, int K, int k, int nnz, int64_t total /* F*G*NA*(B/VB) */) {
  const int BV = B / VB;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(t % BV) * VB;
    const int64_t cj = t / BV;
    const int j = (int)(cj % NA);
    const int fg = (int)(cj / NA);
    const int f = fg / G;
    const int g = fg - f * G;
    const T* __restrict__ wk = w + ((size_t)(f * K + k) * G + g) * nnz;
    const T* __restrict__ lk = lam_k + (size_t)fg * NA * B + b;
    BVec<T, VB> acc = bload<T, VB>(dY + ((size_t)f * NA + j) * B + b);
    const int beg = (int)rowptrT[j], end = (int)rowptrT[j + 1];
    for (int it = beg; it < end; it += 4) {                  // 4 entries per pass: their index and data loads overlap
      T wv[4];
      BVec<T, VB> l[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (it + u < end) {
          wv[u] = wk[perm[it + u]];
          l[u] = bload<T, VB>(lk + (size_t)colT[it + u] * B);
        } else {
          wv[u] = T(0);
          l[u].zero();
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int q = 0; q < VB; ++q) acc.v[q] = fma(wv[u], l[u].v[q], acc.v[q]);
    }
    bstore<T, VB>(lam_km1 + ((size_t)fg * NA + j) * B + b, acc);
  }
}

// dw_k[(f,g), idx(i, j)] = sum_b lam_k[(f,g), i, b] * prev[(f,g), j, b]      prev = u_{k-1}, or x_g for k = 0
// One warp per ((f,g), row i): lanes run over b (coalesced rows), the products are reduced with shuffles, lane (n % 32)
// keeps the result of the row's n-th entry so that the row's gradients leave in one coalesced store.
template <typename T>
__global__ void __launch_bounds__(256)
wgrad_kernel(const int64_t* __restrict__ rowptr, const int32_t* __restrict__ col, const int32_t* __restrict__ diag,
             const T* __restrict__ lam_k, const T* __restrict__ uprev, const T* __restrict__ xT, T* __restrict__ dw,
             int64_t NA, int B, int G, int K, int k, int64_t nnz, int64_t n_items /* F*G*NA */) {
  const int lane = threadIdx.x & 31;
  const int64_t n_warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t item = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); item < n_items; item += n_warps) {
    const int64_t i = item % NA;
    const int64_t fg = item / NA;
    const int64_t f = fg / G;
    const int g = (int)(fg - f * G);
    const int64_t beg = rowptr[i], end = rowptr[i + 1];
    const T* __restrict__ li = lam_k + (fg * NA + i) * B;
    const T* __restrict__ pv = k == 0 ? xT + (int64_t)g * NA * B : uprev + fg * NA * B;
    T* __restrict__ out = dw + ((f * K + k) * G + g) * nnz;
    const int32_t dg = (k == 0 && diag) ? diag[i] : -2;          // -2: general step
    T keep = T(0);
    for (int64_t idx = beg; idx < end; ++idx) {
      T part = T(0);
      if (dg == -2 || idx == dg) {
        const T* __restrict__ pj = pv + (int64_t)col[idx] * B;
        for (int b = lane; b < B; b += 32) part = fma(li[b], pj[b], part);
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) part += __shfl_xor_sync(0xffffffffu, part, off);
      }
      const int n = (int)(idx - beg);
      if ((n & 31) == lane) keep = part;
      if ((n & 31) == 31 || idx == end - 1) {                    // flush up to 32 results, coalesced
        const int64_t base = idx - (n & 31);
        if (base + lane <= idx) out[base + lane] = keep;
      }
    }
  }
}

// dxT[g, j, b] = sum_f sum_{it in rowT(j)} w_0[f, g, perm[it]] * lam_0[(f,g), colT[it], b]
template <typename T>
__global__ void __launch_bounds__(256)
xgrad_kernel(const int64_t* __restrict__ rowptrT, const int32_t* __restrict__ colT, const int64_t* __restrict__ perm,
             const int32_t* __restrict__ diag, const T* __restrict__ w, const T* __restrict__ lam0, T* __restrict__ dxT,
             int64_t NA, int B, int G, int F, int K, int64_t nnz, int64_t total /* G*NA*B */) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(t % B);
    const int64_t gj = t / B;
    const int64_t j = gj % NA;
    const int64_t g = gj / NA;
    T acc = T(0);
    for (int64_t f = 0; f < F; ++f) {
      const T* __restrict__ w0 = w + ((f * K + 0) * G + g) * nnz;
      const T* __restrict__ l0 = lam0 + (f * G + g) * NA * B + b;
      if (diag) {
        const int32_t d = diag[j];
        if (d >= 0) acc = fma(w0[d], l0[j * B], acc);
      } else {
        for (int64_t it = rowptrT[j]; it < rowptrT[j + 1]; ++it) acc = fma(w0[perm[it]], l0[(int64_t)colT[it] * B], acc);
      }
    }
    dxT[t] = acc;
  }
}

// 16-byte batch vectors: float data, B a multiple of 4, every operand 16-byte aligned (all row strides are multiples of B)
template <typename T>
inline bool vec4_ok(int B, const void* a, const void* b, const void* c, const void* d) {
  const uintptr_t bits = reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c) |
                         reinterpret_cast<uintptr_t>(d);
  return sizeof(T) == 4 && B % 4 == 0 && (bits & 15) == 0;
}

template <typename T>
int forward_t(int64_t NA, int B, int G, int F, int K, const int64_t* rowptr, const int32_t* col, const int32_t* diag,
              int64_t nnz, const T* w, const T* xT, T* states, int n_states, T* Y, cudaStream_t st) {
  const int64_t total = (int64_t)F * NA * B;
  const int64_t chain = (int64_t)F * G * NA * B;
  if (total == 0) return B200GF_OK;
  for (int k = 0; k < K; ++k) {
    // states: n_states buffers of F*G*NA*B.  n_states >= K-1: u_k kept in buffer k (training); n_states == 2: ping-pong
    // (inference); the last step's state is never needed and is not written.
    const T* prev = k > 0 ? states + (int64_t)((k - 1) % n_states) * chain : nullptr;
    T* cur = k < K - 1 ? states + (int64_t)(k % n_states) * chain : nullptr;
    if (vec4_ok<T>(B, w, xT, states, Y))
      step_kernel<T, 4><<<grid_for(total / 4, 256, 132 * 16), 256, 0, st>>>(rowptr, col, diag, w, prev, xT, cur, Y, (int)NA, B, G, K, k, (int)nnz, total / 4);
    else
      step_kernel<T, 1><<<grid_for(total, 256, 132 * 16), 256, 0, st>>>(rowptr, col, diag, w, prev, xT, cur, Y, (int)NA, B, G, K, k, (int)nnz, total);
    LAUNCH_CHECK();
  }
  return B200GF_OK;
}

template <typename T>
int backward_t(int64_t NA, int B, int G, int F, int K, const int64_t* rowptr, const int32_t* col, const int64_t* rowptrT,
               const int32_t* colT, const int64_t* perm, const int32_t* diag, int64_t nnz, const T* w, const T* xT,
               const T* states, const T* dY, T* lam /* 2 x [F*G, NA, B] */, T* dw, T* dxT, cudaStream_t st) {
  const int64_t chain = (int64_t)F * G * NA * B;
  if (chain == 0) return B200GF_OK;
  T* cur = lam;
  T* nxt = lam + chain;
  adjoint_init_kernel<T><<<grid_for(chain, 256, 132 * 16), 256, 0, st>>>(dY, cur, NA, B, G, chain);
  LAUNCH_CHECK();
  const int64_t items = (int64_t)F * G * NA;
  for (int k = K - 1; k >= 0; --k) {
    if (nnz > 0) {
      const int blocks = (int)imin64((items + 7) / 8, 132 * 16);
      wgrad_kernel<T><<<blocks, 256, 0, st>>>(rowptr, col, diag, cur, k > 0 ? states + (int64_t)(k - 1) * chain : nullptr, xT, dw,
                                              NA, B, G, K, k, nnz, items);
      LAUNCH_CHECK();
    }
    if (k == 0) break;
    if (vec4_ok<T>(B, dY, lam, lam, dY))
      adjoint_step_kernel<T, 4><<<grid_for(chain / 4, 256, 132 * 16), 256, 0, st>>>(rowptrT, colT, perm, w, dY, cur, nxt, (int)NA, B, G, K, k, (int)nnz, chain / 4);
    else
      adjoint_step_kernel<T, 1><<<grid_for(chain, 256, 132 * 16), 256, 0, st>>>(rowptrT, colT, perm, w, dY, cur, nxt, (int)NA, B, G, K, k, (int)nnz, chain);
    LAUNCH_CHECK();
    T* tmp = cur; cur = nxt; nxt = tmp;
  }
  const int64_t tx = (int64_t)G * NA * B;
  xgrad_kernel<T><<<grid_for(tx, 256, 132 * 16), 256, 0, st>>>(rowptrT, colT, perm, diag, w, cur, dxT, NA, B, G, F, K, nnz, tx);
  LAUNCH_CHECK();
  return B200GF_OK;
}

}  // namespace ev
}  // namespace b200gf

extern "C" {

int b200gf_ev_forward(int dtype, int64_t NA, int B, int G, int F, int K, const int64_t* rowptr, const int32_t* col,
                      const int32_t* diag, int64_t nnz, const void* w, const void* xT, void* states, int n_states, void* Y,
                      void* stream) {
  using namespace b200gf;
  if (NA < 0 || B <= 0 || G <= 0 || F <= 0 || K <= 0 || nnz < 0) return B200GF_EINVAL;
  if (!rowptr || !col || !xT || !Y || (nnz > 0 && !w)) return B200GF_EINVAL;
  if (NA > INT32_MAX || nnz > INT32_MAX) return B200GF_EUNSUPPORTED;
  if (K > 1 && (!states || n_states < 1 || (n_states < K - 1 && n_states != 2))) return B200GF_EINVAL;
  if (K > 2 && n_states == 1) return B200GF_EINVAL;
  return with_dtype(dtype, [&](auto tag) {
    using T = decltype(tag);
    return ev::forward_t<T>(NA, B, G, F, K, rowptr, col, diag, nnz, (const T*)w, (const T*)xT, (T*)states,
                            n_states < 1 ? 1 : n_states, (T*)Y, (cudaStream_t)stream);
  });
}

int b200gf_ev_backward(int dtype, int64_t NA, int B, int G, int F, int K, const int64_t* rowptr, const int32_t* col,
                       const int64_t* rowptrT, const int32_t* colT, const int64_t* perm, const int32_t* diag, int64_t nnz,
                       const void* w, const void* xT, const void* states, const void* dY, void* lam, void* dw, void* dxT,
                       void* stream) {
  using namespace b200gf;
  if (NA < 0 || B <= 0 || G <= 0 || F <= 0 || K <= 0 || nnz < 0) return B200GF_EINVAL;
  if (!rowptr || !col || !rowptrT || !colT || !perm || !xT || !dY || !lam || !dxT || (K > 1 && !states)) return B200GF_EINVAL;
  if (nnz > 0 && (!w || !dw)) return B200GF_EINVAL;
  if (NA > INT32_MAX || nnz > INT32_MAX) return B200GF_EUNSUPPORTED;
  return with_dtype(dtype, [&](auto tag) {
    using T = decltype(tag);
    return ev::backward_t<T>(NA, B, G, F, K, rowptr, col, rowptrT, colT, perm, diag, nnz, (const T*)w, (const T*)xT,
                             (const T*)states, (const T*)dY, (T*)lam, (T*)dw, (T*)dxT, (cudaStream_t)stream);
  });
}

}  // extern "C"
