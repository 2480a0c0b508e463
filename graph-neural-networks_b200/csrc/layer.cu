// The steps either side of the filter inside one graph-convolutional layer of the reference's selection architectures
// (alegnn/modules/architectures.py:274-296:  GraphFilter -> nn.ReLU -> NoPool | MaxPoolLocal), on the node-major layout
// the filter produces — SURVEY.md §8 f-1.
//   * ReLU itself is the epilogue of the tap contraction (b200gf_forward_act; tc_contract.cu / taps.cu): no extra pass over
//     y.  Its backward needs only the layer output: dy_pre = dy * (y > 0)               -> relu_bwd_kernel
//   * MaxPoolLocal (alegnn/utils/graphML.py:1968-2019): out[i, c] = max_{j in nb(i)} x[j, c] over the K-hop neighbourhood
//     lists, i < n_out.  The reference repeats x maxNeighborhoodSize times and torch.gather's it ((maxNb + 2) N B F s
//     bytes); here it is one gather over the neighbourhood matrix reading node-major rows                -> maxpool_fwd_kernel
//     with the arg-max kept per output element for the backward scatter                  -> maxpool_bwd_kernel
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

// thread per output element; consecutive threads = consecutive columns of one output node (coalesced neighbour rows)
template <typename T>
__global__ void maxpool_fwd_kernel(const T* __restrict__ x, int64_t x_ld, const int32_t* __restrict__ nb, int max_nb,
                                   T* __restrict__ out, int64_t out_ld, int32_t* __restrict__ arg, int64_t n_out, int C) {
  const int64_t total = n_out * C;
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
}

template <typename T>
__global__ void maxpool_bwd_kernel(const T* __restrict__ dy, int64_t dy_ld, const int32_t* __restrict__ arg,
                                   T* __restrict__ dx, int64_t dx_ld, int64_t n_out, int C) {
  const int64_t total = n_out * C;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = idx / C;
    const int c = (int)(idx - i * C);
    atomicAdd(dx + (int64_t)arg[idx] * dx_ld + c, dy[i * dy_ld + c]);
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
    layer::maxpool_fwd_kernel<T><<<g, 256, 0, st>>>((const T*)x, x_ld, nb, max_nb, (T*)out, out_ld, argmax, n_out, C);
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
                                                                                     dx_ld, n_out, C);
    LAUNCH_CHECK();
    return B200GF_OK;
  });
}

}  // extern "C"
