// Layout conversion at the drop-in boundary.  The reference keeps activations as [B, G, N] with the node
// axis contiguous (graphML.py:108-109); the sparse shift needs one node's B*G features contiguous.
// [B, G, N] is a [C, N] matrix with C = B*G, so both directions are a tiled 2-D transpose through shared
// memory (coalesced 128-byte reads and writes, padded tile => no bank conflicts).
#include "common.cuh"

namespace b200gf {

// dst[n, c] = src[c, n];  columns c in [C, ld) of dst are zero-filled when fill_pad
template <typename T>
__global__ void __launch_bounds__(256)
transpose_kernel(const T* __restrict__ src, int64_t src_ld, T* __restrict__ dst, int64_t dst_ld, int64_t rows_src,
                 int64_t cols_src, int64_t dst_cols_total) {
  // src is [rows_src, cols_src] with row stride src_ld; dst is [cols_src, rows_src(+pad)] with row stride dst_ld
  __shared__ T tile[32][33];
  const int64_t c0 = (int64_t)blockIdx.x * 32;  // along src columns
  const int64_t r0 = (int64_t)blockIdx.y * 32;  // along src rows
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
#pragma unroll
  for (int i = 0; i < 32; i += 8) {
    const int64_t r = r0 + ty + i, c = c0 + tx;
    tile[ty + i][tx] = (r < rows_src && c < cols_src) ? src[r * src_ld + c] : T(0);
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 32; i += 8) {
    const int64_t c = c0 + ty + i, r = r0 + tx;  // dst row = c, dst col = r
    if (c < cols_src && r < dst_cols_total) dst[c * dst_ld + r] = tile[tx][ty + i];
  }
}

template <typename T>
static int run_transpose(const T* src, int64_t src_ld, T* dst, int64_t dst_ld, int64_t rows_src, int64_t cols_src,
                         int64_t dst_cols_total, cudaStream_t st) {
  if (rows_src <= 0 || cols_src <= 0) return B200GF_OK;
  const int64_t gx = (cols_src + 31) / 32, gy = (dst_cols_total + 31) / 32;
  if (gy > 65535) {
    // very wide source (many rows): loop over slabs of rows
    const int64_t slab = 65535LL * 32;
    for (int64_t r = 0; r < dst_cols_total; r += slab) {
      const int64_t nr = slab < dst_cols_total - r ? slab : dst_cols_total - r;
      int64_t src_rows_here = rows_src - r < nr ? rows_src - r : nr;
      if (src_rows_here < 0) src_rows_here = 0;
      dim3 grid((unsigned)gx, (unsigned)((nr + 31) / 32));
      transpose_kernel<T><<<grid, 256, 0, st>>>(src + r * src_ld, src_ld, dst + r, dst_ld, src_rows_here, cols_src, nr);
      LAUNCH_CHECK();
    }
    return B200GF_OK;
  }
  dim3 grid((unsigned)gx, (unsigned)gy);
  transpose_kernel<T><<<grid, 256, 0, st>>>(src, src_ld, dst, dst_ld, rows_src, cols_src, dst_cols_total);
  LAUNCH_CHECK();
  return B200GF_OK;
}

// [C, N] -> [N, ld]; pad columns [C, ld) are zero-filled so every later kernel may read whole padded rows
int launch_to_node_major(int dtype, const void* src, void* dst, int64_t dst_ld, int64_t N, int C, cudaStream_t st) {
  if (!src || !dst || N < 0 || C <= 0 || dst_ld < C) return B200GF_EINVAL;
  return with_dtype(dtype, [&](auto tag) {
    using T = decltype(tag);
    return run_transpose<T>((const T*)src, N, (T*)dst, dst_ld, C, N, dst_ld, st);
  });
}

// [N, ld] -> [C, N]
int launch_to_feature_major(int dtype, const void* src, int64_t src_ld, void* dst, int64_t N, int C, cudaStream_t st) {
  if (!src || !dst || N < 0 || C <= 0 || src_ld < C) return B200GF_EINVAL;
  return with_dtype(dtype, [&](auto tag) {
    using T = decltype(tag);
    return run_transpose<T>((const T*)src, src_ld, (T*)dst, N, N, C, N, st);
  });
}

}  // namespace b200gf

extern "C" {
int b200gf_to_node_major(int dtype, const void* src_cn, void* dst_nc, int64_t dst_ld, int64_t N, int C, void* stream) {
  return b200gf::launch_to_node_major(dtype, src_cn, dst_nc, dst_ld, N, C, (cudaStream_t)stream);
}
int b200gf_to_feature_major(int dtype, const void* src_nc, int64_t src_ld, void* dst_cn, int64_t N, int C, void* stream) {
  return b200gf::launch_to_feature_major(dtype, src_nc, src_ld, dst_cn, N, C, (cudaStream_t)stream);
}
}
