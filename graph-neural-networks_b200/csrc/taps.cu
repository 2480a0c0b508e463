// Filter-tap side of the LSIGF path (FP32/FP64 FMA implementation, any shape):
//   tap_contract : y = sum_t Z_t · W_t (+ bias)      — reference graphML.py:170-175 (the [B,N,EKG] x [EKG,F] GEMM + bias)
//   tap_grad     : dW_t = A^T · V_t                    — autograd of the above w.r.t. h (SURVEY.md §8 a-8)
//   bias_grad    : db = column sums of dy
//   pack_taps    : h[F,E,K,G] -> W[t][G][F] (t = 0 merges the k = 0 taps of every e, graphML.py:154)
// The wgmma (3xTF32) contraction in tc_contract.cu takes over for the FP32 shapes it supports; these
// kernels are the general path and the FP64 path.
#include "common.cuh"

namespace b200gf {

// ---------------------------------------------------------------------------------------------------
// pack taps
// ---------------------------------------------------------------------------------------------------
template <typename T>
__global__ void pack_taps_kernel(const T* __restrict__ h, T* __restrict__ W, int F, int E, int K, int G,
                                 int transpose_taps) {
  const int Tn = 1 + E * (K - 1);
  const int64_t total = (int64_t)Tn * G * F;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i / ((int64_t)G * F));
    const int rem = (int)(i - (int64_t)t * G * F);
    int g, f;
    if (transpose_taps) { f = rem / G; g = rem % G; }  // W[t][f][g]
    else { g = rem / F; f = rem % F; }                  // W[t][g][f]
    T val;
    if (t == 0) {
      val = T(0);
      for (int e = 0; e < E; ++e) val += h[(((int64_t)f * E + e) * K + 0) * G + g];
    } else {
      const int e = (t - 1) / (K - 1), k = (t - 1) % (K - 1) + 1;
      val = h[(((int64_t)f * E + e) * K + k) * G + g];
    }
    W[i] = val;
  }
}

int launch_pack_taps(int dtype, const void* h, void* W, int F, int E, int K, int G, int transpose_taps,
                     cudaStream_t st) {
  if (!h || !W || F <= 0 || E <= 0 || K <= 0 || G <= 0) return B200GF_EINVAL;
  const int64_t total = (int64_t)(1 + E * (K - 1)) * G * F;
  return with_dtype(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    pack_taps_kernel<T><<<grid_for(total, 256, 132 * 8), 256, 0, st>>>((const T*)h, (T*)W, F, E, K, G, transpose_taps);
    LAUNCH_CHECK();
    return B200GF_OK;
  });
}

// ---------------------------------------------------------------------------------------------------
// tap contraction: out[(n,b), q] (+)= bias + sum_t sum_p Z_t[(n,b), p] W[t][p][q]
// 64 x 64 output tile per 256-thread block, 4 x 4 micro-tile per thread, K-step 16.
// ---------------------------------------------------------------------------------------------------
constexpr int TC_BM = 64, TC_BN = 64, TC_BK = 16;

template <typename T>
__global__ void __launch_bounds__(256)
tap_contract_kernel(TermList terms, int T_terms, const T* __restrict__ W, const T* __restrict__ bias,
                    int bias_per_node, T* __restrict__ out, int64_t out_ld, int64_t n_rows, int B, int P, int Q,
                    int accumulate) {
  __shared__ T As[TC_BK][TC_BM + 4];
  __shared__ T Bs[TC_BK][TC_BN + 4];
  const int64_t R = n_rows * B;
  const int64_t r0 = (int64_t)blockIdx.x * TC_BM;
  const int q0 = blockIdx.y * TC_BN;
  const int tid = threadIdx.x;
  const int tx = tid % 16, ty = tid / 16;  // thread computes rows ty*4..+3, cols tx*4..+3
  T acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = T(0);

  // A-tile loader: thread -> (row = tid / 4, 4 consecutive p starting at (tid % 4) * 4)
  const int a_row = tid / 4, a_p = (tid % 4) * 4;
  const int64_t ar = r0 + a_row;
  const bool a_row_ok = ar < R;
  const int64_t an = a_row_ok ? ar / B : 0;
  const int ab = a_row_ok ? (int)(ar - an * B) : 0;
  // B-tile loader: thread -> (k = tid / 16, 4 consecutive q starting at (tid % 16) * 4)
  const int b_k = tid / 16, b_q = (tid % 16) * 4;

  for (int t = 0; t < T_terms; ++t) {
    const T* __restrict__ Z = reinterpret_cast<const T*>(terms.ptr[t]) + an * terms.ld[t] + (int64_t)ab * P;
    const T* __restrict__ Wt = W + (int64_t)t * P * Q;
    for (int p0 = 0; p0 < P; p0 += TC_BK) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int p = p0 + a_p + i;
        As[a_p + i][a_row] = (a_row_ok && p < P) ? Z[p] : T(0);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int p = p0 + b_k, q = q0 + b_q + j;
        Bs[b_k][b_q + j] = (p < P && q < Q) ? Wt[(int64_t)p * Q + q] : T(0);
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < TC_BK; ++kk) {
        T a[4], b[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
        for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx * 4 + j];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fma(a[i], b[j], acc[i][j]);
      }
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t r = r0 + ty * 4 + i;
    if (r >= R) continue;
    const int64_t n = r / B;
    const int b = (int)(r - n * B);
    T* __restrict__ o = out + n * out_ld + (int64_t)b * Q;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int q = q0 + tx * 4 + j;
      if (q >= Q) continue;
      T val = acc[i][j];
      if (bias) val += bias_per_node ? bias[(int64_t)q * n_rows + n] : bias[q];
      if (accumulate & 1) val += o[q];
      if (accumulate & 2) val = val > T(0) ? val : T(0);   // fused ReLU epilogue (last launch of the chain only)
      o[q] = val;
    }
  }
}

int launch_tap_contract(int dtype, int64_t n_rows, int B, int P, int Q, int T, const void* const* zs,
                        const int64_t* z_ld, const void* W, const void* bias, int bias_per_node, void* out,
                        int64_t out_ld, int accumulate, cudaStream_t st, int act) {
  if (n_rows < 0 || B <= 0 || P <= 0 || Q <= 0 || T <= 0 || !zs || !z_ld || !W || !out) return B200GF_EINVAL;
  if (out_ld < (int64_t)B * Q) return B200GF_EINVAL;
  if (n_rows == 0) return B200GF_OK;
  if (dmma_contract_eligible(dtype, n_rows, B, P, Q, T, zs, z_ld, out, out_ld, accumulate)) {
    for (int t = 0; t < T; ++t)
      if (!zs[t] || z_ld[t] < (int64_t)B * P) return B200GF_EINVAL;
    int sms = 132, dev = 0;                      // FP64: the DMMA kernel (dmma_contract.cu)
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return launch_dmma_contract(sms, n_rows, B, P, Q, T, zs, z_ld, W, bias, bias_per_node, out, out_ld, st, act);
  }
  const int64_t R = n_rows * B;
  dim3 grid((unsigned)((R + TC_BM - 1) / TC_BM), (unsigned)((Q + TC_BN - 1) / TC_BN));
  const size_t es = dtype_size(dtype);
  for (int t0 = 0; t0 < T; t0 += TermList::MAX_TERMS) {
    const int tn = min(TermList::MAX_TERMS, T - t0);
    TermList tl;
    for (int i = 0; i < tn; ++i) {
      if (!zs[t0 + i] || z_ld[t0 + i] < (int64_t)B * P) return B200GF_EINVAL;
      tl.ptr[i] = zs[t0 + i];
      tl.ld[i] = z_ld[t0 + i];
    }
    const void* Wt = (const char*)W + (size_t)t0 * P * Q * es;
    const void* bb = t0 == 0 ? bias : nullptr;
    const int acc = ((t0 == 0) ? (accumulate ? 1 : 0) : 1) | ((act && t0 + TermList::MAX_TERMS >= T) ? 2 : 0);
    // the dtype is looked at only here, after this group's terms are checked
    const int rc = with_dtype(dtype, [&](auto tag) -> int {
      using Ty = decltype(tag);
      tap_contract_kernel<Ty><<<grid, 256, 0, st>>>(tl, tn, (const Ty*)Wt, (const Ty*)bb, bias_per_node, (Ty*)out, out_ld,
                                                    n_rows, B, P, Q, acc);
      LAUNCH_CHECK();
      return B200GF_OK;
    });
    if (rc) return rc;
  }
  return B200GF_OK;
}

// ---------------------------------------------------------------------------------------------------
// tap gradient (two-pass, deterministic): partial[chunk][t][p][q] = sum_{rows in chunk} A[r,p] V_t[r,q]
// ---------------------------------------------------------------------------------------------------
constexpr int TG_BP = 64, TG_BQ = 64, TG_BK = 16;

struct TapGradGeom {
  int64_t rows_per_chunk;
  int n_chunks;
  int p_tiles, q_tiles;
};

static TapGradGeom tap_grad_geom(int64_t n_rows, int B, int P, int Q, int T) {
  TapGradGeom g;
  g.p_tiles = (P + TG_BP - 1) / TG_BP;
  g.q_tiles = (Q + TG_BQ - 1) / TG_BQ;
  const int64_t R = n_rows * B;
  const int64_t per = (int64_t)((T + 4) / 5) * g.p_tiles * g.q_tiles;  // the FP32 fast path groups 5 terms per block
  int64_t want = (132 * 2 + per - 1) / per;  // aim at ~2 resident blocks per SM in total
  if (want < 1) want = 1;
  int64_t rpc = (R + want - 1) / want;
  if (rpc < 256) rpc = 256;
  rpc = (rpc + TG_BK - 1) / TG_BK * TG_BK;
  g.rows_per_chunk = rpc;
  g.n_chunks = (int)((R + rpc - 1) / rpc);
  if (g.n_chunks < 1) g.n_chunks = 1;
  return g;
}

size_t tap_grad_scratch_bytes(int dtype, int64_t n_rows, int B, int P, int Q, int T) {
  const TapGradGeom g = tap_grad_geom(n_rows, B, P, Q, T);
  return align_up((size_t)g.n_chunks * T * P * Q * dtype_size(dtype), 256);
}

template <typename T>
__global__ void __launch_bounds__(256)
tap_grad_partial_kernel(const T* __restrict__ A, int64_t a_ld, TermList vs, int64_t n_rows, int B, int P, int Q,
                        int64_t rows_per_chunk, int q_tiles, T* __restrict__ partial, int T_terms) {
  __shared__ T As[TG_BK][TG_BP + 4];
  __shared__ T Vs[TG_BK][TG_BQ + 4];
  const int chunk = blockIdx.x;
  const int t = blockIdx.y;
  const int p0 = (blockIdx.z / q_tiles) * TG_BP, q0 = (blockIdx.z % q_tiles) * TG_BQ;
  const int64_t R = n_rows * B;
  const int64_t rbeg = (int64_t)chunk * rows_per_chunk;
  const int64_t rend = min(R, rbeg + rows_per_chunk);
  const T* __restrict__ V = reinterpret_cast<const T*>(vs.ptr[t]);
  const int64_t v_ld = vs.ld[t];
  const int tid = threadIdx.x;
  const int tx = tid % 16, ty = tid / 16;  // thread owns p = p0 + ty*4.., q = q0 + tx*4..
  const int l_row = tid / 16, l_c = (tid % 16) * 4;  // loader: one of 16 rows, 4 consecutive columns
  T acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = T(0);

  for (int64_t r0 = rbeg; r0 < rend; r0 += TG_BK) {
    const int64_t r = r0 + l_row;
    const bool ok = r < rend;
    const int64_t n = ok ? r / B : 0;
    const int b = ok ? (int)(r - n * B) : 0;
    const T* __restrict__ ap = A + n * a_ld + (int64_t)b * P;
    const T* __restrict__ vp = V + n * v_ld + (int64_t)b * Q;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int p = p0 + l_c + i, q = q0 + l_c + i;
      As[l_row][l_c + i] = (ok && p < P) ? ap[p] : T(0);
      Vs[l_row][l_c + i] = (ok && q < Q) ? vp[q] : T(0);
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < TG_BK; ++kk) {
      T a[4], v[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = Vs[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fma(a[i], v[j], acc[i][j]);
    }
    __syncthreads();
  }
  T* __restrict__ o = partial + ((int64_t)chunk * T_terms + t) * P * Q;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int p = p0 + ty * 4 + i;
    if (p >= P) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int q = q0 + tx * 4 + j;
      if (q < Q) o[(int64_t)p * Q + q] = acc[i][j];
    }
  }
}

// FP32 fast path: one block = TPB terms x 64 threads, every thread an 8 x 8 micro-tile of its term's 64 x 64 output
// tile; the A tile is staged once per row step and shared by all TPB terms (4 LDS.128 per 64 FMAs).
// Needs 16-byte aligned rows (P, Q, a_ld, v_ld multiples of 4).  Same partial layout as the generic kernel.
template <int TPB>
__global__ void __launch_bounds__(64 * TPB, 1)
tap_grad_multi_kernel(const float* __restrict__ A, int64_t a_ld, TermList vs, int t_base, int64_t n_rows, int B, int P,
                      int Q, int64_t rows_per_chunk, int q_tiles, float* __restrict__ partial, int T_terms) {
  constexpr int BK = 16;
  constexpr int NT = 64 * TPB;
  constexpr int NV = (1 + TPB) * BK * 16;          // float4 per stage
  constexpr int PER = (NV + NT - 1) / NT;          // float4 per thread per stage
  __shared__ __align__(16) float As[2][BK][64];    // double-buffered: global loads of step s+1 overlap the FMAs of step s
  __shared__ __align__(16) float Vs[2][TPB][BK][64];
  const int chunk = blockIdx.x;
  const int p0 = (blockIdx.z / q_tiles) * 64, q0 = (blockIdx.z % q_tiles) * 64;
  const int64_t R = n_rows * B;
  const int64_t rbeg = (int64_t)chunk * rows_per_chunk;
  const int64_t rend = min(R, rbeg + rows_per_chunk);
  const int tid = threadIdx.x;
  const int tt = tid / 64, l64 = tid % 64;
  const int ty = l64 / 8, tx = l64 % 8;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  float4 stage[PER];
  auto fetch = [&](int64_t r0) {
#pragma unroll
    for (int u = 0; u < PER; ++u) {
      const int idx = tid + u * NT;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (idx < NV) {
        const int m = idx / (BK * 16);
        const int rem = idx - m * (BK * 16);
        const int kk = rem / 16, c4 = (rem % 16) * 4;
        const int64_t r = r0 + kk;
        if (r < rend) {
          const int64_t n = r / B;
          const int b = (int)(r - n * B);
          if (m == 0) {
            if (p0 + c4 < P) v = __ldg(reinterpret_cast<const float4*>(A + n * a_ld + (int64_t)b * P + p0 + c4));
          } else {
            const float* V = reinterpret_cast<const float*>(vs.ptr[t_base + m - 1]);
            if (q0 + c4 < Q) v = __ldg(reinterpret_cast<const float4*>(V + n * vs.ld[t_base + m - 1] + (int64_t)b * Q + q0 + c4));
          }
        }
      }
      stage[u] = v;
    }
  };
  auto commit = [&](int buf) {
#pragma unroll
    for (int u = 0; u < PER; ++u) {
      const int idx = tid + u * NT;
      if (idx < NV) {
        const int m = idx / (BK * 16);
        const int rem = idx - m * (BK * 16);
        const int kk = rem / 16, c4 = (rem % 16) * 4;
        if (m == 0) *reinterpret_cast<float4*>(&As[buf][kk][c4]) = stage[u];
        else *reinterpret_cast<float4*>(&Vs[buf][m - 1][kk][c4]) = stage[u];
      }
    }
  };

  if (rbeg < rend) {
    fetch(rbeg);
    commit(0);
  }
  __syncthreads();
  int buf = 0;
  for (int64_t r0 = rbeg; r0 < rend; r0 += BK) {
    const bool more = r0 + BK < rend;
    if (more) fetch(r0 + BK);                       // in flight while this step computes
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[8], v[8];
      *reinterpret_cast<float4*>(&a[0]) = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 8]);
      *reinterpret_cast<float4*>(&a[4]) = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 8 + 4]);
      *reinterpret_cast<float4*>(&v[0]) = *reinterpret_cast<const float4*>(&Vs[buf][tt][kk][tx * 8]);
      *reinterpret_cast<float4*>(&v[4]) = *reinterpret_cast<const float4*>(&Vs[buf][tt][kk][tx * 8 + 4]);
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], v[j], acc[i][j]);
    }
    if (more) commit(buf ^ 1);
    __syncthreads();
    buf ^= 1;
  }
  float* __restrict__ o = partial + ((int64_t)chunk * T_terms + t_base + tt) * P * Q;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int p = p0 + ty * 8 + i;
    if (p >= P) continue;
#pragma unroll
    for (int j = 0; j < 8; j += 4) {
      const int q = q0 + tx * 8 + j;
      if (q < Q) *reinterpret_cast<float4*>(o + (int64_t)p * Q + q) = make_float4(acc[i][j], acc[i][j + 1], acc[i][j + 2], acc[i][j + 3]);
    }
  }
}

template <int TPB>
static void launch_tap_grad_multi(dim3 grid, cudaStream_t st, const float* A, int64_t a_ld, const TermList& tl, int t_base,
                                  int64_t n_rows, int B, int P, int Q, int64_t rpc, int q_tiles, float* partial, int T) {
  tap_grad_multi_kernel<TPB><<<grid, 64 * TPB, 0, st>>>(A, a_ld, tl, t_base, n_rows, B, P, Q, rpc, q_tiles, partial, T);
}

// second pass: fixed-order sum over chunks; out_mode 1 scatters into the taps layout dh[F=Q,E,K,G=P]
template <typename T>
__global__ void tap_grad_reduce_kernel(const T* __restrict__ partial, int n_chunks, int T_terms, int P, int Q,
                                       T* __restrict__ dW, int out_mode, int E, int K) {
  const int64_t total = (int64_t)T_terms * P * Q;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    T s = T(0);
    for (int c = 0; c < n_chunks; ++c) s += partial[(int64_t)c * total + i];
    if (out_mode == 0) {
      dW[i] = s;
    } else {
      const int t = (int)(i / ((int64_t)P * Q));
      const int rem = (int)(i - (int64_t)t * P * Q);
      const int g = rem / Q, f = rem % Q;
      if (t == 0) {
        for (int e = 0; e < E; ++e) dW[(((int64_t)f * E + e) * K + 0) * P + g] = s;
      } else {
        const int e = (t - 1) / (K - 1), k = (t - 1) % (K - 1) + 1;
        dW[(((int64_t)f * E + e) * K + k) * P + g] = s;
      }
    }
  }
}

int launch_tap_grad(int dtype, int64_t n_rows, int B, int P, int Q, int T, const void* A, int64_t a_ld,
                    const void* const* vs, const int64_t* v_ld, void* dW, int out_mode, int E, int K,
                    void* scratch, size_t scratch_bytes, cudaStream_t st) {
  if (n_rows < 0 || B <= 0 || P <= 0 || Q <= 0 || T <= 0 || !A || !vs || !v_ld || !dW || !scratch) return B200GF_EINVAL;
  if (a_ld < (int64_t)B * P) return B200GF_EINVAL;
  if (scratch_bytes < tap_grad_scratch_bytes(dtype, n_rows, B, P, Q, T)) return B200GF_EWORKSPACE;
  if (dtype != B200GF_F32 && dtype != B200GF_F64) return B200GF_EUNSUPPORTED;
  const TapGradGeom g = tap_grad_geom(n_rows, B, P, Q, T);
  const size_t es = dtype_size(dtype);
  for (int t0 = 0; t0 < T; t0 += TermList::MAX_TERMS) {
    const int tn = min(TermList::MAX_TERMS, T - t0);
    TermList tl;
    for (int i = 0; i < tn; ++i) {
      if (!vs[t0 + i] || v_ld[t0 + i] < (int64_t)B * Q) return B200GF_EINVAL;
      tl.ptr[i] = vs[t0 + i];
      tl.ld[i] = v_ld[t0 + i];
    }
    dim3 grid((unsigned)g.n_chunks, (unsigned)tn, (unsigned)(g.p_tiles * g.q_tiles));
    // partial layout is [chunk][T][P][Q] over ALL T terms; offset the base so block t writes term t0 + t
    char* part = (char*)scratch + (size_t)t0 * P * Q * es;
    bool fast = dtype == B200GF_F32 && P % 4 == 0 && Q % 4 == 0 && a_ld % 4 == 0 && ((uintptr_t)A & 15) == 0;
    for (int i = 0; i < tn && fast; ++i) fast = tl.ld[i] % 4 == 0 && ((uintptr_t)tl.ptr[i] & 15) == 0;
    if (fast) {
      // terms in groups of up to 5 sharing the staged A tile
      for (int tb = 0; tb < tn; tb += 5) {
        const int tpb = min(5, tn - tb);
        dim3 g2((unsigned)g.n_chunks, 1, (unsigned)(g.p_tiles * g.q_tiles));
        const float* Af = (const float*)A;
        float* pf = (float*)part;
        switch (tpb) {
          case 1: launch_tap_grad_multi<1>(g2, st, Af, a_ld, tl, tb, n_rows, B, P, Q, g.rows_per_chunk, g.q_tiles, pf, T); break;
          case 2: launch_tap_grad_multi<2>(g2, st, Af, a_ld, tl, tb, n_rows, B, P, Q, g.rows_per_chunk, g.q_tiles, pf, T); break;
          case 3: launch_tap_grad_multi<3>(g2, st, Af, a_ld, tl, tb, n_rows, B, P, Q, g.rows_per_chunk, g.q_tiles, pf, T); break;
          case 4: launch_tap_grad_multi<4>(g2, st, Af, a_ld, tl, tb, n_rows, B, P, Q, g.rows_per_chunk, g.q_tiles, pf, T); break;
          default: launch_tap_grad_multi<5>(g2, st, Af, a_ld, tl, tb, n_rows, B, P, Q, g.rows_per_chunk, g.q_tiles, pf, T); break;
        }
        LAUNCH_CHECK();
      }
      continue;
    }
    const int rc = with_dtype(dtype, [&](auto tag) -> int {
      using Ty = decltype(tag);
      tap_grad_partial_kernel<Ty><<<grid, 256, 0, st>>>((const Ty*)A, a_ld, tl, n_rows, B, P, Q, g.rows_per_chunk,
                                                        g.q_tiles, (Ty*)part, T);
      LAUNCH_CHECK();
      return B200GF_OK;
    });
    if (rc) return rc;
  }
  const int blocks = grid_for((int64_t)T * P * Q, 256, 132 * 8);
  return with_dtype(dtype, [&](auto tag) -> int {
    using Ty = decltype(tag);
    tap_grad_reduce_kernel<Ty><<<blocks, 256, 0, st>>>((const Ty*)scratch, g.n_chunks, T, P, Q, (Ty*)dW, out_mode, E, K);
    LAUNCH_CHECK();
    return B200GF_OK;
  });
}

// ---------------------------------------------------------------------------------------------------
// bias gradient
// ---------------------------------------------------------------------------------------------------
constexpr int BG_ROWS = 2048;  // node rows per partial block

size_t bias_grad_scratch_bytes(int dtype, int64_t n_rows, int B, int F) {
  const int64_t chunks = (n_rows + BG_ROWS - 1) / BG_ROWS;
  return align_up((size_t)(chunks > 0 ? chunks : 1) * F * dtype_size(dtype), 256);
}

// per-feature bias [F] (the reference's F x 1): partial[chunk][f] = sum_{n in chunk, b} dy[n, b*F + f]
template <typename T>
__global__ void __launch_bounds__(256)
bias_grad_partial_kernel(const T* __restrict__ dy, int64_t dy_ld, int64_t n_rows, int B, int F, T* __restrict__ partial) {
  __shared__ T red[8][33];
  const int64_t n0 = (int64_t)blockIdx.x * BG_ROWS;
  const int64_t n1 = min(n_rows, n0 + BG_ROWS);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int f0 = 0; f0 < F; f0 += 32) {
    const int f = f0 + lane;
    T s = T(0);
    if (f < F)
      for (int64_t n = n0 + warp; n < n1; n += 8)
        for (int b = 0; b < B; ++b) s += dy[n * dy_ld + (int64_t)b * F + f];
    red[warp][lane] = s;
    __syncthreads();
    if (warp == 0 && f < F) {
      T tot = T(0);
#pragma unroll
      for (int w = 0; w < 8; ++w) tot += red[w][lane];
      partial[(int64_t)blockIdx.x * F + f] = tot;
    }
    __syncthreads();
  }
}

// FP32 fast path for compact rows (dy_ld == B*F) with (4*256) % F == 0: the chunk is one contiguous float4 stream and a
// thread always sees the same 4 columns, so it accumulates them in registers (4 loads in flight), then threads with the
// same column group are summed in a fixed order through shared memory.
__global__ void __launch_bounds__(256)
bias_grad_partial_vec_kernel(const float* __restrict__ dy, int64_t n_rows, int B, int F, float* __restrict__ partial) {
  __shared__ float4 red[256];
  const int64_t n0 = (int64_t)blockIdx.x * BG_ROWS;
  const int64_t n1 = min(n_rows, n0 + BG_ROWS);
  const int64_t nvec = (n1 - n0) * B * F / 4;
  const float4* __restrict__ base = reinterpret_cast<const float4*>(dy + n0 * B * F);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  int64_t i = threadIdx.x;
  for (; i + 3 * 256 < nvec; i += 4 * 256) {
    const float4 a = __ldg(base + i), b = __ldg(base + i + 256), c = __ldg(base + i + 512), d = __ldg(base + i + 768);
    acc.x += (a.x + b.x) + (c.x + d.x); acc.y += (a.y + b.y) + (c.y + d.y);
    acc.z += (a.z + b.z) + (c.z + d.z); acc.w += (a.w + b.w) + (c.w + d.w);
  }
  for (; i < nvec; i += 256) {
    const float4 a = __ldg(base + i);
    acc.x += a.x; acc.y += a.y; acc.z += a.z; acc.w += a.w;
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  const int groups = F / 4;  // threads tid, tid + groups, tid + 2*groups, ... hold the same columns
  if (threadIdx.x < groups) {
    float4 tot = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int t = threadIdx.x; t < 256; t += groups) {
      tot.x += red[t].x; tot.y += red[t].y; tot.z += red[t].z; tot.w += red[t].w;
    }
    float* o = partial + (int64_t)blockIdx.x * F + threadIdx.x * 4;
    o[0] = tot.x; o[1] = tot.y; o[2] = tot.z; o[3] = tot.w;
  }
}

template <typename T>
__global__ void bias_grad_reduce_kernel(const T* __restrict__ partial, int n_chunks, int F, T* __restrict__ db) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  T s = T(0);
  for (int c = 0; c < n_chunks; ++c) s += partial[(int64_t)c * F + f];
  db[f] = s;
}

// per-node bias [F, N]: db[f, n] = sum_b dy[n, b*F + f]
template <typename T>
__global__ void bias_grad_node_kernel(const T* __restrict__ dy, int64_t dy_ld, int64_t n_rows, int B, int F,
                                      T* __restrict__ db) {
  const int64_t total = n_rows * F;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t n = i / F;
    const int f = (int)(i - n * F);
    T s = T(0);
    for (int b = 0; b < B; ++b) s += dy[n * dy_ld + (int64_t)b * F + f];
    db[(int64_t)f * n_rows + n] = s;
  }
}

int launch_bias_grad(int dtype, int64_t n_rows, int B, int F, const void* dy, int64_t dy_ld, void* dbias,
                     int bias_per_node, void* scratch, size_t scratch_bytes, cudaStream_t st) {
  if (!dy || !dbias || n_rows < 0 || B <= 0 || F <= 0) return B200GF_EINVAL;
  if (dtype != B200GF_F32 && dtype != B200GF_F64) return B200GF_EUNSUPPORTED;
  if (bias_per_node) {
    const int64_t total = n_rows * F;
    if (total == 0) return B200GF_OK;
    return with_dtype(dtype, [&](auto tag) -> int {
      using T = decltype(tag);
      bias_grad_node_kernel<T><<<grid_for(total, 256, 132 * 8), 256, 0, st>>>((const T*)dy, dy_ld, n_rows, B, F, (T*)dbias);
      LAUNCH_CHECK();
      return B200GF_OK;
    });
  }
  if (!scratch || scratch_bytes < bias_grad_scratch_bytes(dtype, n_rows, B, F)) return B200GF_EWORKSPACE;
  const int n_chunks = (int)((n_rows + BG_ROWS - 1) / BG_ROWS);
  if (dtype == B200GF_F32) {
    const bool vec = F % 4 == 0 && 1024 % F == 0 && dy_ld == (int64_t)B * F && ((uintptr_t)dy & 15) == 0;
    if (n_chunks > 0 && vec)
      bias_grad_partial_vec_kernel<<<n_chunks, 256, 0, st>>>((const float*)dy, n_rows, B, F, (float*)scratch);
    else if (n_chunks > 0)
      bias_grad_partial_kernel<float><<<n_chunks, 256, 0, st>>>((const float*)dy, dy_ld, n_rows, B, F, (float*)scratch);
    bias_grad_reduce_kernel<float><<<(F + 127) / 128, 128, 0, st>>>((const float*)scratch, n_chunks, F, (float*)dbias);
  } else {
    if (n_chunks > 0)
      bias_grad_partial_kernel<double><<<n_chunks, 256, 0, st>>>((const double*)dy, dy_ld, n_rows, B, F, (double*)scratch);
    bias_grad_reduce_kernel<double><<<(F + 127) / 128, 128, 0, st>>>((const double*)scratch, n_chunks, F, (double*)dbias);
  }
  LAUNCH_CHECK_N(n_chunks > 0 ? 2 : 1);
  return B200GF_OK;
}

}  // namespace b200gf

extern "C" {

int b200gf_pack_taps(int dtype, const void* h, void* W, int F, int E, int K, int G, int transpose_taps, void* stream) {
  return b200gf::launch_pack_taps(dtype, h, W, F, E, K, G, transpose_taps, (cudaStream_t)stream);
}

int b200gf_tap_contract(int dtype, int64_t n_rows, int B, int P, int Q, int T, const void* const* zs,
                        const int64_t* z_ld, const void* W, const void* bias, int bias_per_node, void* out,
                        int64_t out_ld, int accumulate, void* scratch, size_t scratch_bytes, void* stream) {
  using namespace b200gf;
  if (n_rows < 0 || B <= 0 || P <= 0 || Q <= 0 || T <= 0 || !zs || !z_ld || !W || !out) return B200GF_EINVAL;
  if (scratch && scratch_bytes >= tc_contract_scratch_bytes(T, P, Q) && (reinterpret_cast<uintptr_t>(scratch) & 15) == 0 &&
      tc_contract_eligible(dtype, n_rows, B, P, Q, T, zs, z_ld, out, out_ld, accumulate)) {
    int dev = 0, sms = 132;
    CUDA_TRY(cudaGetDevice(&dev));
    CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    int rc = launch_split_w(W, scratch, T, P, Q, (cudaStream_t)stream);
    if (rc) return rc;
    return launch_tc_contract(sms, n_rows, B, P, Q, T, zs, scratch, bias, bias_per_node, out, out_ld, (cudaStream_t)stream);
  }
  return launch_tap_contract(dtype, n_rows, B, P, Q, T, zs, z_ld, W, bias, bias_per_node, out, out_ld, accumulate,
                             (cudaStream_t)stream);
}

size_t b200gf_tap_contract_scratch_bytes(int T, int P, int Q) { return b200gf::tc_contract_scratch_bytes(T, P, Q); }

int b200gf_tap_grad(int dtype, int64_t n_rows, int B, int P, int Q, int T, const void* A, int64_t a_ld,
                    const void* const* vs, const int64_t* v_ld, void* dW, void* scratch, size_t scratch_bytes,
                    void* stream) {
  return b200gf::launch_tap_grad(dtype, n_rows, B, P, Q, T, A, a_ld, vs, v_ld, dW, 0, 1, 1, scratch, scratch_bytes,
                                 (cudaStream_t)stream);
}

size_t b200gf_tap_grad_scratch_bytes(int dtype, int64_t n_rows, int B, int P, int Q, int T) {
  return b200gf::tap_grad_scratch_bytes(dtype, n_rows, B, P, Q, T);
}

}  // extern "C"
