// The steps either side of the filter inside one graph-convolutional layer of the reference's selection architectures
// (alegnn/modules/architectures.py:274-296:  GraphFilter -> nn.ReLU -> NoPool | MaxPoolLocal), on the node-major layout
// the filter produces — SURVEY.md §8 f-1.
//   * ReLU itself is the epilogue of the tap contraction (b200gf_forward_act; tc_contract.cu / taps.cu): no extra pass over
//     y.  Its backward needs only the layer output: dy_pre = dy * (y > 0)               -> relu_bwd_kernel
//   * MaxPoolLocal (alegnn/utils/graphML.py:1968-2019): out[i, c] = max_{j in nb(i)} x[j, c] over the K-hop neighbourhood
//     lists, i < n_out.  The reference repeats x maxNeighborhoodSize times and torch.gather's it ((maxNb + 2) N B F s
//     bytes); here it is one gather over the neighbourhood matrix reading node-major rows                -> maxpool_fwd_kernel
//     with the arg-max kept per output element for the backward scatter                  -> maxpool_bwd_kernel
//   * MaxLocalActivation / MedianLocalActivation (graphML.py:1535-1810): the same gather-select, run over ring-ordered
//     K-hop lists (graphtools_sparse.ring_neighborhoods) for every k at once, with the max or the lower median as the
//     selection and the combine y = w0 x + sum_k w_k agg_k fused in                          -> maxpool_fwd_kernel
//     and the scatter of w_k dy by every hop's choice                                         -> maxpool_bwd_kernel
//     The two kernels are generalised in place: runtime arguments describe the list format, the selection and the
//     weights, so MaxPoolLocal's padded-matrix launches run the code they always ran.
#include "common.cuh"

namespace b200gf {
namespace layer {

template <typename T>
__global__ void relu_bwd_kernel(const T* __restrict__ y, int64_t y_ld, const T* __restrict__ dy, int64_t dy_ld,
                                T* __restrict__ out, int64_t out_ld, int64_t n_rows, int C) {
  const int64_t total = n_rows * C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / C;
    const int c = (int)(i - r * C);
    out[r * out_ld + c] = y[r * y_ld + c] > T(0) ? dy[r * dy_ld + c] : T(0);
  }
}

// order-preserving unsigned key of a float / double: a < b  <=>  key(a) < key(b) (-0 sorts below +0)
__device__ __forceinline__ uint32_t order_key(float v) {
  const uint32_t u = __float_as_uint(v);
  return u ^ ((uint32_t)((int32_t)u >> 31) | 0x80000000u);
}
__device__ __forceinline__ uint64_t order_key(double v) {
  const uint64_t u = (uint64_t)__double_as_longlong(v);
  return u ^ ((uint64_t)((int64_t)u >> 63) | 0x8000000000000000ull);
}

// The (n - 1) / 2-th smallest of x[row[0 .. n), c] (the lower median, torch.median's), and the smallest node index
// holding that value.  Radix select on the order-preserving keys, 4-bit digits from the top, the 16 digit counts in
// registers: one pass over the list per digit, each counting only the entries that still match the selected prefix,
// stopping early once a single entry matches; one last pass picks the smallest node index among the matching entries.
template <typename T>
__device__ __forceinline__ void lower_median(const T* __restrict__ x, int64_t x_ld, const int32_t* __restrict__ row, int n,
                                             int c, T& val, int32_t& node) {
  using K = decltype(order_key(T{}));
  constexpr int BITS = 8 * (int)sizeof(K);
  int rank = (n - 1) / 2;
  K prefix = 0, mask = 0;
  for (int shift = BITS - 4; shift >= 0; shift -= 4) {
    int cnt[16];
#pragma unroll
    for (int b = 0; b < 16; ++b) cnt[b] = 0;
    for (int j = 0; j < n; ++j) {
      const K key = order_key(x[(int64_t)__ldg(row + j) * x_ld + c]);
      if ((key & mask) == prefix) {
        const int d = (int)(key >> shift) & 15;
#pragma unroll
        for (int b = 0; b < 16; ++b) cnt[b] += (d == b);
      }
    }
    int sel = 15, left = 0;
    bool found = false;
#pragma unroll
    for (int b = 0; b < 16; ++b) {
      if (!found) {
        if (rank < cnt[b]) { sel = b; left = cnt[b]; found = true; }
        else rank -= cnt[b];
      }
    }
    prefix |= (K)sel << shift;
    mask |= (K)15 << shift;
    if (left == 1) break;
  }
  node = INT32_MAX;
  for (int j = 0; j < n; ++j) {
    const int32_t m = __ldg(row + j);
    const T v = x[(int64_t)m * x_ld + c];
    if ((order_key(v) & mask) == prefix && m < node) { node = m; val = v; }
  }
}

// thread per output element; consecutive threads = consecutive columns of one output node (coalesced neighbour rows).
// Two list formats, told apart by rowptr:
//   rowptr null (MaxPoolLocal): row i is nb[i * max_nb, + max_nb), padded with one of its members; one selection, the
//     maximum, the first maximum of the list winning; out [n_out, out_ld], arg [n_out, C] (optional).
//   rowptr set (localized activations): row i is nb[rowptr[i] ..], ordered by hop distance (graphtools_sparse
//     .ring_neighborhoods), its k-hop neighbourhood the prefix of length ring_end[i * (K + 1) + k] >= 1.  For k = 1..K
//     selection k-1 goes to out[(k-1) n_out out_ld + i out_ld + c] and arg[(k-1) n_out C + i C + c]: the maximum of the
//     prefix (select 0; equal values: the smaller node index wins) or its lower median (select 1; the smallest node
//     index holding the median value).  y[i, c] = w[0] x[i, c] + w[1] out_1 + ... + w[K] out_K, k ascending.
template <typename T>
__global__ void maxpool_fwd_kernel(const T* __restrict__ x, int64_t x_ld, const int32_t* __restrict__ nb, int max_nb,
                                   T* __restrict__ out, int64_t out_ld, int32_t* __restrict__ arg, int64_t n_out, int C,
                                   const int64_t* __restrict__ rowptr, const int32_t* __restrict__ ring_end, int K,
                                   int select, const T* __restrict__ w, T* __restrict__ y, int64_t y_ld) {
  const int64_t total = n_out * C;
  if (rowptr == nullptr) {                          // the padded matrix: its own loop, as it was before the ring lists
    for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
      const int64_t i = idx / C;
      const int c = (int)(idx - i * C);
      const int32_t* __restrict__ row = nb + i * max_nb;
      int32_t best = __ldg(row);
      T vmax = x[(int64_t)best * x_ld + c];
      for (int j = 1; j < max_nb; ++j) {
        const int32_t n = __ldg(row + j);
        const T v = x[(int64_t)n * x_ld + c];
        if (v > vmax) { vmax = v; best = n; }       // strict: the first maximum of the list wins, like torch.max on the CPU
      }
      out[i * out_ld + c] = vmax;
      if (arg) arg[idx] = best;
    }
    return;
  }
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = idx / C;
    const int c = (int)(idx - i * C);
    const int32_t* __restrict__ row = nb + __ldg(rowptr + i);
    const int32_t* __restrict__ ends = ring_end + i * (K + 1);
    const T xi = x[i * x_ld + c];
    T acc = __ldg(w) * xi;
    int32_t best = __ldg(row);
    T vmax = x[(int64_t)best * x_ld + c];
    int j = 1;
    for (int k = 1; k <= K; ++k) {
      const int end = __ldg(ends + k);
      T v_k;
      int32_t a_k;
      if (select == 0) {                            // one running pass: the prefix maxima of every k
        for (; j < end; ++j) {
          const int32_t n = __ldg(row + j);
          const T v = x[(int64_t)n * x_ld + c];
          if (v > vmax || (v == vmax && n < best)) { vmax = v; best = n; }
        }
        v_k = vmax;
        a_k = best;
      } else {
        lower_median(x, x_ld, row, end, c, v_k, a_k);
      }
      out[(int64_t)(k - 1) * n_out * out_ld + i * out_ld + c] = v_k;
      arg[(int64_t)(k - 1) * total + idx] = a_k;
      acc += __ldg(w + k) * v_k;
    }
    y[i * y_ld + c] = acc;
  }
}

// the scatter of the selections' gradients.  arg set: for each of the K selections k (arg slice [k * n_out * C, ..)),
// dx[arg_k[i, c], c] += w[k + 1] dy[i, c] (dy itself when w is null), by atomicAdd: the order of the additions, and so
// the last bits, may change from run to run.  arg null: the identity selection, dx[i, c] = w[0] dy[i, c], plain stores
// (every element has one writer), which a scatter launch then adds to.
template <typename T>
__global__ void maxpool_bwd_kernel(const T* __restrict__ dy, int64_t dy_ld, const int32_t* __restrict__ arg,
                                   T* __restrict__ dx, int64_t dx_ld, int64_t n_out, int C, int K,
                                   const T* __restrict__ w) {
  const int64_t total = n_out * C;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = idx / C;
    const int c = (int)(idx - i * C);
    const T g = dy[i * dy_ld + c];
    if (arg == nullptr) {
      dx[i * dx_ld + c] = __ldg(w) * g;
      continue;
    }
    for (int k = 0; k < K; ++k)
      atomicAdd(dx + (int64_t)arg[(int64_t)k * total + idx] * dx_ld + c, w ? __ldg(w + k + 1) * g : g);
  }
}

}  // namespace layer
}  // namespace b200gf

using namespace b200gf;

extern "C" {

int b200gf_relu_backward(int dtype, const void* y, int64_t y_ld, const void* dy, int64_t dy_ld, void* out, int64_t out_ld,
                         int64_t n_rows, int C, void* stream) {
  if (!y || !dy || !out || n_rows < 0 || C <= 0 || y_ld < C || dy_ld < C || out_ld < C) return B200GF_EINVAL;
  if (n_rows == 0) return B200GF_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int g = grid_for(n_rows * C, 256, 132 * 16);
  return with_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    layer::relu_bwd_kernel<T><<<g, 256, 0, st>>>((const T*)y, y_ld, (const T*)dy, dy_ld, (T*)out, out_ld, n_rows, C);
    LAUNCH_CHECK();
    return B200GF_OK;
  });
}

int b200gf_maxpool_forward(int dtype, const void* x, int64_t x_ld, int64_t n_in, int C, const int32_t* nb, int64_t n_out,
                           int max_nb, void* out, int64_t out_ld, int32_t* argmax, void* stream) {
  if (!x || !nb || !out || n_in <= 0 || n_out < 0 || C <= 0 || max_nb <= 0 || x_ld < C || out_ld < C) return B200GF_EINVAL;
  if (n_in > INT32_MAX) return B200GF_EUNSUPPORTED;
  if (n_out == 0) return B200GF_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int g = grid_for(n_out * C, 256, 132 * 16);
  return with_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    layer::maxpool_fwd_kernel<T><<<g, 256, 0, st>>>((const T*)x, x_ld, nb, max_nb, (T*)out, out_ld, argmax, n_out, C,
                                                    nullptr, nullptr, 1, 0, nullptr, nullptr, 0);
    LAUNCH_CHECK();
    return B200GF_OK;
  });
}

int b200gf_maxpool_backward(int dtype, const void* dy, int64_t dy_ld, const int32_t* argmax, int64_t n_out, int C,
                            void* dx, int64_t dx_ld, int64_t n_in, void* stream) {
  if (!dy || !argmax || !dx || n_in <= 0 || n_out < 0 || C <= 0 || dy_ld < C || dx_ld < C) return B200GF_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  return with_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    CUDA_TRY(cudaMemsetAsync(dx, 0, (size_t)n_in * dx_ld * sizeof(T), st));
    if (n_out == 0) return B200GF_OK;
    layer::maxpool_bwd_kernel<T><<<grid_for(n_out * C, 256, 132 * 16), 256, 0, st>>>((const T*)dy, dy_ld, argmax, (T*)dx,
                                                                                     dx_ld, n_out, C, 1, nullptr);
    LAUNCH_CHECK();
    return B200GF_OK;
  });
}

int b200gf_local_activation_forward(int dtype, int select, const void* x, int64_t x_ld, int64_t N, int C,
                                    const int64_t* rowptr, const int32_t* col, const int32_t* ring_end, int K,
                                    const void* weight, void* y, int64_t y_ld, void* agg, int64_t agg_ld, int32_t* arg,
                                    void* stream) {
  if (!x || !rowptr || !col || !ring_end || !weight || !y || !agg || !arg || N < 0 || C <= 0 || K < 1 || x_ld < C ||
      y_ld < C || agg_ld < C)
    return B200GF_EINVAL;
  if (select != B200GF_LOCAL_MAX && select != B200GF_LOCAL_MEDIAN) return B200GF_EUNSUPPORTED;
  if (N > INT32_MAX) return B200GF_EUNSUPPORTED;
  if (N == 0) return B200GF_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int g = grid_for(N * C, 256, 132 * 16);
  return with_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    layer::maxpool_fwd_kernel<T><<<g, 256, 0, st>>>((const T*)x, x_ld, col, 0, (T*)agg, agg_ld, arg, N, C, rowptr,
                                                    ring_end, K, select, (const T*)weight, (T*)y, y_ld);
    LAUNCH_CHECK();
    return B200GF_OK;
  });
}

int b200gf_local_activation_backward(int dtype, const void* dy, int64_t dy_ld, const int32_t* arg, int64_t N, int C, int K,
                                     const void* weight, void* dx, int64_t dx_ld, void* stream) {
  if (!dy || !arg || !weight || !dx || N < 0 || C <= 0 || K < 1 || dy_ld < C || dx_ld < C) return B200GF_EINVAL;
  if (N > INT32_MAX) return B200GF_EUNSUPPORTED;
  if (N == 0) return B200GF_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int g = grid_for(N * C, 256, 132 * 16);
  return with_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    // dx = w0 dy first (no memset), then every hop's scatter adds to it
    layer::maxpool_bwd_kernel<T><<<g, 256, 0, st>>>((const T*)dy, dy_ld, nullptr, (T*)dx, dx_ld, N, C, 0,
                                                    (const T*)weight);
    LAUNCH_CHECK();
    layer::maxpool_bwd_kernel<T><<<g, 256, 0, st>>>((const T*)dy, dy_ld, arg, (T*)dx, dx_ld, N, C, K, (const T*)weight);
    LAUNCH_CHECK();
    return B200GF_OK;
  });
}

}  // extern "C"
