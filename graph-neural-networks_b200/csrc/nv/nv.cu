// Node-variant graph filter behind the C ABI (reference NVGF, alegnn/utils/graphML.py:293-387, and its autograd;
// NodeVariantGF :2317-2509).  Node-major only.  No allocation, no host synchronisation, one writer per output element
// and a fixed summation order everywhere, so a call is CUDA-graph capturable and bitwise reproducible.
//
//   W [M][T][G][F]  taps packed node-major (T = 1 + E(K-1); t = 0 merges the k = 0 taps of every e, as pack_taps does)
//   node_tap [N]    tap block of node n (the layer's copyNodes)
//
// Forward   Z_0 = x ; Z_{e,k} = Z_{e,k-1} · S_e      (E(K-1) hops, spmm.cu, unchanged)
//           y[n, b*F+f] = bias + sum_t sum_g Z_t[n, b*G+g] W[node_tap[n]][t][g][f]        (nv_contract_kernel)
// Backward  dz_t[n, b*G+g] = sum_f W[node_tap[n]][t][g][f] dy[n, b*F+f]                   (nv_contract_kernel, transposed)
//           dx = dz_0 + sum_e BWD(dz_{e,1} + BWD(dz_{e,2} + ... BWD(dz_{e,K-1})))            (Horner over the BWD hops)
//           dW[m][t][g][f] = sum_{n in nodes(m)} sum_b Z_t[n, b*G+g] dy[n, b*F+f]           (Z_t recomputed from x)
//           as a segmented two-pass reduction: the members of each tap are cut into pieces of `chunk` nodes, pass 1
//           writes one partial per piece, pass 2 sums a tap's pieces in order and unpacks to h's layout [F,E,K,G,M].
#include "../common.cuh"

using namespace b200gf;

namespace {

constexpr int NV_THREADS = 128;                  // contraction block
constexpr int NV_BT = 8;                         // batch lanes a contraction thread keeps in registers
constexpr size_t NV_SMEM = 48 * 1024;            // staged tap rows (the default dynamic shared-memory limit)
constexpr int NV_TG_THREADS = 256;               // tap-gradient block

// a tap shared by all N nodes is cut into pieces of piece_rows(N) nodes: sum_m ceil(cnt_m / chunk) < N / chunk + (number
// of non-empty taps)
int64_t nv_pieces_bound(int64_t N, int64_t M) { return N / piece_rows(N) + std::min(M, N) + 1; }

// ---------------------------------------------------------------------------------------------------------------
// pack: h [F][E][K][G][M] -> W [M][T][G][F]
// ---------------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void nv_pack_taps_kernel(const T* __restrict__ h, T* __restrict__ W, int F, int E, int K, int G, int64_t M) {
  const int Tn = 1 + E * (K - 1);
  const int64_t blk = (int64_t)Tn * G * F;
  const int64_t total = M * blk;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t m = i / blk;
    const int rem = (int)(i - m * blk);
    const int t = rem / (G * F);
    const int g = (rem / F) % G, f = rem % F;
    T val;
    if (t == 0) {
      val = T(0);
      for (int e = 0; e < E; ++e) val += h[((((int64_t)f * E + e) * K + 0) * G + g) * M + m];
    } else {
      const int e = (t - 1) / (K - 1), k = (t - 1) % (K - 1) + 1;
      val = h[((((int64_t)f * E + e) * K + k) * G + g) * M + m];
    }
    W[i] = val;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// per-node contraction
//   out[n, b*Q + q] = sum_{t, p} Z_t[n, b*P + p] Wn(t, p, q) (+ bias) (+ add[n, b*Q + q])
//   Wn = the tap block of node n, terms t_first .. t_first + T_terms - 1 of T_all:
//     forward    (P = G, Q = F): Wn(t, p, q) = W[m][t][p][q]
//     transposed (P = F, Q = G): Wn(t, p, q) = W[m][t][q][p]
// One block per node (grid-stride).  The node's tap rows (t, p) are staged in shared memory as [row][q]; threads run over
// (q, batch tile of NV_BT lanes) with the lanes' sums in registers.  STREAM = false: the whole block fits and is staged
// once per node.  STREAM = true: the block is larger than NV_SMEM, so it is staged `rows_fit` rows at a time.
// Each output is one fma chain over (t, p) in ascending order, then + bias, then + add.
// ---------------------------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ void nv_stage(T* __restrict__ sW, const T* __restrict__ Wn, int r0, int r1, int P, int Q,
                                         int transposed) {
  const int n_el = (r1 - r0) * Q;
  for (int i = threadIdx.x; i < n_el; i += blockDim.x) {
    const int r = r0 + i / Q, q = i % Q;
    const int tt = r / P, p = r - tt * P;
    sW[i] = transposed ? Wn[((int64_t)tt * Q + q) * P + p] : Wn[(int64_t)r * Q + q];
  }
}

template <typename T, bool STREAM>
__global__ void __launch_bounds__(NV_THREADS)
nv_contract_kernel(TermList z, int T_terms, int t_first, int T_all, int64_t n_rows, int B, int P, int Q, int transposed,
                   const T* __restrict__ W, const int32_t* __restrict__ node_tap, const T* __restrict__ bias,
                   int bias_per_node, const T* add, int64_t add_ld, T* out, int64_t out_ld, int rows_fit) {
  extern __shared__ __align__(16) unsigned char nv_smem[];
  T* sW = reinterpret_cast<T*>(nv_smem);
  const int nbt = (B + NV_BT - 1) / NV_BT;
  const int items = Q * nbt;
  const int R = T_terms * P;                           // tap rows (t, p)
  const int slab = STREAM ? rows_fit : R;
  for (int64_t n = blockIdx.x; n < n_rows; n += gridDim.x) {
    const int64_t m = node_tap[n];
    const T* __restrict__ Wn = W + (m * T_all + t_first) * (int64_t)P * Q;
    if (!STREAM) {
      __syncthreads();                                 // the previous node's reads are done
      nv_stage(sW, Wn, 0, R, P, Q, transposed);
      __syncthreads();
    }
    for (int i0 = 0; i0 < items; i0 += NV_THREADS) {
      const int it = i0 + threadIdx.x;
      const bool live = it < items;
      const int q = live ? it % Q : 0;
      const int b0 = live ? (it / Q) * NV_BT : 0;
      T acc[NV_BT];
#pragma unroll
      for (int j = 0; j < NV_BT; ++j) acc[j] = T(0);
      for (int r0 = 0; r0 < R; r0 += slab) {
        const int r1 = min(R, r0 + slab);
        if (STREAM) {
          __syncthreads();
          nv_stage(sW, Wn, r0, r1, P, Q, transposed);
          __syncthreads();
        }
        if (live) {
          int tt = r0 / P, p = r0 - tt * P;
          for (int r = r0; r < r1; ++r) {
            const T w = sW[(r - r0) * Q + q];
            const T* __restrict__ zr = reinterpret_cast<const T*>(z.ptr[tt]) + n * z.ld[tt] + (int64_t)b0 * P + p;
#pragma unroll
            for (int j = 0; j < NV_BT; ++j)
              if (b0 + j < B) acc[j] = fma(zr[(int64_t)j * P], w, acc[j]);
            if (++p == P) { p = 0; ++tt; }
          }
        }
      }
      if (live) {
        const T bv = bias ? (bias_per_node ? bias[(int64_t)q * n_rows + n] : bias[q]) : T(0);
#pragma unroll
        for (int j = 0; j < NV_BT; ++j) {
          const int b = b0 + j;
          if (b >= B) continue;
          T v = acc[j];
          if (bias) v += bv;
          if (add) v += add[n * add_ld + (int64_t)b * Q + q];
          out[n * out_ld + (int64_t)b * Q + q] = v;
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// tap gradient
// ---------------------------------------------------------------------------------------------------------------
// piece_ptr[m] = sum_{m' < m} ceil(cnt_m' / chunk), piece_ptr[M] = number of pieces.  One block of NV_SCAN_THREADS
// threads: each counts a contiguous range of taps, thread 0 scans the counts, every thread then writes its range.
constexpr int NV_SCAN_THREADS = 256;

__global__ void __launch_bounds__(NV_SCAN_THREADS)
nv_piece_scan_kernel(const int64_t* __restrict__ tap_rowptr, int64_t M, int64_t chunk, int64_t* __restrict__ piece_ptr) {
  __shared__ int64_t part[NV_SCAN_THREADS];
  const int64_t per = (M + NV_SCAN_THREADS - 1) / NV_SCAN_THREADS;
  const int64_t m0 = min(M, (int64_t)threadIdx.x * per), m1 = min(M, m0 + per);
  int64_t s = 0;
  for (int64_t m = m0; m < m1; ++m) s += (tap_rowptr[m + 1] - tap_rowptr[m] + chunk - 1) / chunk;
  part[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    int64_t run = 0;
    for (int i = 0; i < NV_SCAN_THREADS; ++i) {
      const int64_t c = part[i];
      part[i] = run;
      run += c;
    }
    piece_ptr[M] = run;
  }
  __syncthreads();
  int64_t run = part[threadIdx.x];
  for (int64_t m = m0; m < m1; ++m) {
    piece_ptr[m] = run;
    run += (tap_rowptr[m + 1] - tap_rowptr[m] + chunk - 1) / chunk;
  }
}

// pass 1: partial[piece][t][g][f] = sum over the piece's members n (ascending in tap_nodes), then b ascending, of
// Z_t[n, b*G + g] dy[n, b*F + f].  grid = (bound on the number of pieces, T); blocks past the last piece exit.
template <typename T>
__global__ void __launch_bounds__(NV_TG_THREADS)
nv_tap_grad_partial_kernel(TermList z, int T_all, int B, int G, int F, const T* __restrict__ dy, int64_t dy_ld,
                           const int64_t* __restrict__ tap_rowptr, const int32_t* __restrict__ tap_nodes,
                           const int64_t* __restrict__ piece_ptr, int64_t M, int64_t chunk, T* __restrict__ partial) {
  const int64_t piece = blockIdx.x;
  if (piece >= piece_ptr[M]) return;
  int64_t lo = 0, hi = M;                              // the tap m with piece_ptr[m] <= piece < piece_ptr[m + 1]
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) / 2;
    if (piece_ptr[mid] <= piece) lo = mid;
    else hi = mid;
  }
  const int64_t m = lo;
  const int64_t beg = tap_rowptr[m] + (piece - piece_ptr[m]) * chunk;
  const int64_t end = min(tap_rowptr[m + 1], beg + chunk);
  const int t = blockIdx.y;
  const T* __restrict__ Z = reinterpret_cast<const T*>(z.ptr[t]);
  const int64_t ld = z.ld[t];
  T* __restrict__ o = partial + (piece * T_all + t) * (int64_t)G * F;
  for (int idx = threadIdx.x; idx < G * F; idx += blockDim.x) {
    const int g = idx / F, f = idx - g * F;
    T acc = T(0);
    for (int64_t pos = beg; pos < end; ++pos) {
      const int64_t n = tap_nodes[pos];
      const T* __restrict__ zr = Z + n * ld + g;
      const T* __restrict__ dr = dy + n * dy_ld + f;
      for (int b = 0; b < B; ++b) acc = fma(zr[(int64_t)b * G], dr[(int64_t)b * F], acc);
    }
    o[idx] = acc;
  }
}

// pass 2: dh[f][e][k][g][m] = sum of tap m's pieces in order (k = 0: the merged t = 0 gradient, in every e); a tap
// without members sums nothing and is written as exactly 0.
template <typename T>
__global__ void nv_tap_grad_reduce_kernel(const T* __restrict__ partial, const int64_t* __restrict__ piece_ptr, int64_t M,
                                          int F, int E, int K, int G, T* __restrict__ dh) {
  const int T_all = 1 + E * (K - 1);
  const int64_t total = (int64_t)F * E * K * G * M;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t m = i % M;
    int64_t r = i / M;
    const int g = (int)(r % G);
    r /= G;
    const int k = (int)(r % K);
    r /= K;
    const int e = (int)(r % E);
    const int f = (int)(r / E);
    const int t = k == 0 ? 0 : 1 + e * (K - 1) + (k - 1);
    T s = T(0);
    for (int64_t p = piece_ptr[m]; p < piece_ptr[m + 1]; ++p) s += partial[((p * T_all + t) * G + g) * (int64_t)F + f];
    dh[i] = s;
  }
}

// dst[n, c] += src[n, c] for c < C (summing the E Horner chains)
template <typename T>
__global__ void nv_add_kernel(T* __restrict__ dst, int64_t dst_ld, const T* __restrict__ src, int64_t src_ld,
                              int64_t n_rows, int C) {
  const int64_t total = n_rows * C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t n = i / C;
    const int c = (int)(i - n * C);
    dst[n * dst_ld + c] += src[n * src_ld + c];
  }
}

int launch_nv_contract(int dt, int sm_count, const void* const* zs, const int64_t* z_ld, int T_terms, int t_first,
                       int T_all, int64_t n_rows, int B, int P, int Q, int transposed, const void* W,
                       const int32_t* node_tap, const void* bias, int bias_per_node, const void* add, int64_t add_ld,
                       void* out, int64_t out_ld, cudaStream_t st) {
  const TermList tl = make_terms(zs, z_ld, T_terms);
  const size_t es = dtype_size(dt);
  const int R = T_terms * P;
  const int rows_fit = (int)std::min<size_t>((size_t)R, NV_SMEM / ((size_t)Q * es));
  if (rows_fit < 1) return B200GF_EUNSUPPORTED;       // one tap row (Q elements) larger than NV_SMEM
  const bool stream_taps = rows_fit < R;
  const size_t smem = (size_t)rows_fit * Q * es;
  const int grid = (int)std::min<int64_t>(n_rows, (int64_t)sm_count * 8);
#define NV_CONTRACT(TY, S)                                                                                           \
  nv_contract_kernel<TY, S><<<grid, NV_THREADS, smem, st>>>(tl, T_terms, t_first, T_all, n_rows, B, P, Q, transposed,  \
                                                             (const TY*)W, node_tap, (const TY*)bias, bias_per_node,  \
                                                             (const TY*)add, add_ld, (TY*)out, out_ld, rows_fit)
  if (dt == B200GF_F32) {
    if (stream_taps) NV_CONTRACT(float, true);
    else NV_CONTRACT(float, false);
  } else {
    if (stream_taps) NV_CONTRACT(double, true);
    else NV_CONTRACT(double, false);
  }
#undef NV_CONTRACT
  LAUNCH_CHECK();
  return B200GF_OK;
}

int launch_nv_add(int dt, int sm_count, void* dst, int64_t dst_ld, const void* src, int64_t src_ld, int64_t n_rows, int C,
                  cudaStream_t st) {
  const int grid = grid_for(n_rows * C, 256, sm_count * 8);
  return with_dtype(dt, [&](auto tag) -> int {
    using T = decltype(tag);
    nv_add_kernel<T><<<grid, 256, 0, st>>>((T*)dst, dst_ld, (const T*)src, src_ld, n_rows, C);
    LAUNCH_CHECK();
    return B200GF_OK;
  });
}

struct NvWs {
  void* z = nullptr;        // E(K-1) hop outputs Z_{e,k}, each [N, ldc]
  void* hb[2] = {nullptr, nullptr};  // Horner ping-pong [N, ldc]        (backward, K > 1)
  void* sum = nullptr;      // sum over e of the chains [N, ldc]         (backward, K > 1)
  void* tmp = nullptr;      // chain e >= 1 before it is added [N, ldc]  (backward, K > 1, E > 1)
  int64_t* piece_ptr = nullptr;  // [M + 1]                             (backward)
  void* partial = nullptr;  // [pieces][T][G][F]                         (backward)
  void* bg = nullptr;       // bias-grad partials                        (backward)
  size_t bg_bytes = 0;
  size_t bytes = 0;
};

NvWs carve_nv(const b200gf_plan* p, void* ws, int B, int G, int F, int K, int64_t M, bool backward) {
  const size_t es = dtype_size(p->dtype);
  const int64_t N = p->n_rows;
  const int64_t ldc = padded_ld((int64_t)B * G, p->dtype);
  const int E = p->E;
  const int T = 1 + E * (K - 1);
  const size_t buf = (size_t)N * ldc * es;
  Carver c(ws);
  NvWs w;
  w.z = c.take((size_t)E * (K - 1) * buf);
  if (backward) {
    if (K > 1) {
      w.hb[0] = c.take(buf);
      w.hb[1] = c.take(buf);
      w.sum = c.take(buf);
      if (E > 1) w.tmp = c.take(buf);
    }
    w.piece_ptr = (int64_t*)c.take((size_t)(M + 1) * sizeof(int64_t));
    w.partial = c.take((size_t)nv_pieces_bound(N, M) * T * G * F * es);
    w.bg_bytes = bias_grad_scratch_bytes(p->dtype, N, B, F);
    w.bg = c.take(w.bg_bytes);
  }
  w.bytes = c.off;
  return w;
}

bool nv_bad_dims(const b200gf_plan* plan, int B, int G, int F, int K, int64_t M) {
  if (!plan || B <= 0 || G <= 0 || F <= 0 || K <= 0 || M <= 0) return true;
  return plan->n_rows != plan->n_cols;                 // partitioned plans are not supported here
}

}  // namespace

extern "C" {

int b200gf_nv_pack_taps(int dtype, const void* h, void* W, int F, int E, int K, int G, int64_t M, void* stream) {
  if (!h || !W || F <= 0 || E <= 0 || K <= 0 || G <= 0 || M <= 0) return B200GF_EINVAL;
  const int64_t total = M * (1 + E * (K - 1)) * (int64_t)G * F;
  const int grid = grid_for(total, 256, 132 * 8);
  return with_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    nv_pack_taps_kernel<T><<<grid, 256, 0, (cudaStream_t)stream>>>((const T*)h, (T*)W, F, E, K, G, M);
    LAUNCH_CHECK();
    return B200GF_OK;
  });
}

size_t b200gf_nv_workspace_bytes(const b200gf_plan* plan, int B, int G, int F, int K, int64_t M, int backward) {
  if (nv_bad_dims(plan, B, G, F, K, M)) return 0;
  return carve_nv(plan, nullptr, B, G, F, K, M, backward != 0).bytes + 256;
}

int b200gf_nv_forward(const b200gf_plan* plan, const void* x, int64_t x_ld, const void* W, const int32_t* node_tap,
                      int64_t M, const void* bias, int bias_per_node, void* y, int64_t y_ld, void* workspace,
                      size_t workspace_bytes, int B, int G, int F, int K, void* stream) {
  if (nv_bad_dims(plan, B, G, F, K, M) || !x || !W || !node_tap || !y) return B200GF_EINVAL;
  if (bias_per_node != 0 && bias_per_node != 1) return B200GF_EINVAL;
  const int64_t N = plan->n_rows;
  const int64_t C = (int64_t)B * G, CF = (int64_t)B * F;
  if (x_ld < C || y_ld < CF) return B200GF_EINVAL;
  if (C > INT32_MAX || CF > INT32_MAX) return B200GF_EUNSUPPORTED;
  const int T = 1 + plan->E * (K - 1);
  if (T > TermList::MAX_TERMS) return B200GF_EUNSUPPORTED;
  NvWs w = carve_nv(plan, workspace, B, G, F, K, M, false);
  int rc;
  if ((rc = check_workspace(workspace, w.bytes, workspace_bytes, false))) return rc;
  if (N == 0) return B200GF_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int dt = plan->dtype;
  std::vector<const void*> zs;
  std::vector<int64_t> zld;
  if ((rc = hop_chain(plan, plan->fwd, x, x_ld, w.z, padded_ld(C, dt), (int)C, K, zs, zld, st))) return rc;
  return launch_nv_contract(dt, plan->sm_count, zs.data(), zld.data(), T, 0, T, N, B, G, F, 0, W, node_tap, bias,
                            bias_per_node, nullptr, 0, y, y_ld, st);
}

int b200gf_nv_backward(const b200gf_plan* plan, const void* dy, int64_t dy_ld, const void* x, int64_t x_ld,
                       const void* W, const int32_t* node_tap, int64_t M, const int64_t* tap_rowptr,
                       const int32_t* tap_nodes, void* dx, int64_t dx_ld, void* dh, void* dbias, int bias_per_node,
                       void* workspace, size_t workspace_bytes, int B, int G, int F, int K, void* stream) {
  if (nv_bad_dims(plan, B, G, F, K, M) || !plan->has_bwd) return B200GF_EINVAL;
  if (!dy || !x || !W || !node_tap || !tap_rowptr || !tap_nodes || !dh) return B200GF_EINVAL;
  if (bias_per_node != 0 && bias_per_node != 1) return B200GF_EINVAL;
  const int64_t N = plan->n_rows;
  const int64_t C = (int64_t)B * G, CF = (int64_t)B * F;
  if (dy_ld < CF || x_ld < C || (dx && dx_ld < C)) return B200GF_EINVAL;
  if (C > INT32_MAX || CF > INT32_MAX) return B200GF_EUNSUPPORTED;
  const int E = plan->E;
  const int T = 1 + E * (K - 1);
  if (T > TermList::MAX_TERMS) return B200GF_EUNSUPPORTED;
  NvWs w = carve_nv(plan, workspace, B, G, F, K, M, true);
  int rc;
  if ((rc = check_workspace(workspace, w.bytes, workspace_bytes, true))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int dt = plan->dtype;
  const size_t es = dtype_size(dt);
  const int sms = plan->sm_count;
  if (N == 0) {
    CUDA_TRY(cudaMemsetAsync(dh, 0, (size_t)F * E * K * G * M * es, st));
    if (dbias && !bias_per_node) CUDA_TRY(cudaMemsetAsync(dbias, 0, (size_t)F * es, st));
    return B200GF_OK;
  }
  const int64_t ldc = padded_ld(C, dt);

  // dh: Z_t recomputed from x, segmented two-pass reduction over the members of each tap
  std::vector<const void*> zs;
  std::vector<int64_t> zld;
  if ((rc = hop_chain(plan, plan->fwd, x, x_ld, w.z, ldc, (int)C, K, zs, zld, st))) return rc;
  const int64_t chunk = piece_rows(N);
  nv_piece_scan_kernel<<<1, NV_SCAN_THREADS, 0, st>>>(tap_rowptr, M, chunk, w.piece_ptr);
  LAUNCH_CHECK();
  const TermList tl = make_terms(zs.data(), zld.data(), T);
  const dim3 pgrid((unsigned)nv_pieces_bound(N, M), (unsigned)T);
  const int rgrid = grid_for((int64_t)F * E * K * G * M, 256, sms * 8);
  rc = with_dtype(dt, [&](auto tag) -> int {
    using Ty = decltype(tag);
    nv_tap_grad_partial_kernel<Ty><<<pgrid, NV_TG_THREADS, 0, st>>>(tl, T, B, G, F, (const Ty*)dy, dy_ld, tap_rowptr,
                                                                   tap_nodes, w.piece_ptr, M, chunk, (Ty*)w.partial);
    nv_tap_grad_reduce_kernel<Ty><<<rgrid, 256, 0, st>>>((const Ty*)w.partial, w.piece_ptr, M, F, E, K, G, (Ty*)dh);
    LAUNCH_CHECK_N(2);
    return B200GF_OK;
  });
  if (rc) return rc;

  // dx by Horner: per e, buf = dz_{e,K-1}; buf = dz_{e,k} + BWD(buf) for k = K-2 .. 1; chain_e = BWD(buf)
  if (dx) {
    const void* dys[1] = {dy};
    const int64_t dyl[1] = {dy_ld};
    for (int e = 0; e < E && K > 1; ++e) {
      int cur = 0;
      if ((rc = launch_nv_contract(dt, sms, dys, dyl, 1, 1 + e * (K - 1) + (K - 2), T, N, B, F, G, 1, W, node_tap,
                                   nullptr, 0, nullptr, 0, w.hb[0], ldc, st)))
        return rc;
      for (int k = K - 2; k >= 1; --k) {
        if ((rc = plan_hop(plan, plan->bwd[e], w.hb[cur], ldc, w.hb[1 - cur], ldc, (int)C, st))) return rc;
        cur = 1 - cur;
        if ((rc = launch_nv_contract(dt, sms, dys, dyl, 1, 1 + e * (K - 1) + (k - 1), T, N, B, F, G, 1, W, node_tap,
                                     nullptr, 0, w.hb[cur], ldc, w.hb[cur], ldc, st)))
          return rc;
      }
      void* chain = e == 0 ? w.sum : w.tmp;
      if ((rc = plan_hop(plan, plan->bwd[e], w.hb[cur], ldc, chain, ldc, (int)C, st))) return rc;
      if (e > 0 && (rc = launch_nv_add(dt, sms, w.sum, ldc, w.tmp, ldc, N, (int)C, st))) return rc;
    }
    if ((rc = launch_nv_contract(dt, sms, dys, dyl, 1, 0, T, N, B, F, G, 1, W, node_tap, nullptr, 0,
                                 K > 1 ? w.sum : nullptr, ldc, dx, dx_ld, st)))
      return rc;
  }
  if (dbias)
    if ((rc = launch_bias_grad(dt, N, B, F, dy, dy_ld, dbias, bias_per_node, w.bg, w.bg_bytes, st))) return rc;
  return B200GF_OK;
}

}  // extern "C"
