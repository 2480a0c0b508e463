// ARMA graph filter by Jacobi iterations, general-diagonal path, behind the C ABI (reference jARMA,
// alegnn/utils/graphML.py:490-638; GraphFilterARMA :2714-2847).  Node-major only.  No allocation, no host
// synchronisation, one writer per output element and a fixed summation order everywhere, so a call is CUDA-graph
// capturable and bitwise reproducible.
//
// Per edge feature e, with S~ = S_e - diag(S_e), d = diag(S_e) and, for every column c = (f, p, g),
// r_c = 1 / (d - psi[f,e,p,g]) (a vector over the nodes; column convention S~ v):
//   z_0 = r . x_g,        z_t = r . (S~ z_{t-1})      t = 1..tMax
//   y_1 = r . (S~ x_g),   y_t = r . (S~ y_{t-1})      t = 2..tMax+1
//   u[b,f] += sum_{p,g} varphi[f,e,p,g] sum_t (-1)^t z_t  +  (-1)^(tMax+1) sum_{p,g} y_{tMax+1}
// The state of one edge feature is one wide matrix [N, ldw] holding both chains, columns (chain, b, f, p, g) with g
// innermost: C = 2 B Q, Q = F P G, ldw = padded_ld(C).  State t = [z_t | y_{t+1}], so one hop (the plan's FWD operator,
// which is S~ because the plan holds S~^T) advances both chains; arma_scale_acc_kernel then scales by r in place and adds
// the step's share of u into `out`.  x is hopped once on B G columns for y_1.
//
// Backward by adjoints with the BWD hop (S~^T), on the same wide layout: Lambda_t = [lambda_t | mu_{t+1}],
//   R_tMax = r . [(-1)^tMax varphi dU | (-1)^(tMax+1) dU],   R_t = r . (S~^T R_{t+1} + [(-1)^t varphi dU | 0])
//   dpsi   = sum_{i,b} sum_t R_t . State_t          dvarphi = sum_{i,b} dU sum_t (-1)^t z_t
//   dx_g  += sum_{f,p} R_0[z] + S~^T sum_{f,p} R_0[y]
// The per-element sums over t go to an accumulator [N, ldw] (columns (half, b, q): half 0 for psi, 1 for varphi), reduced
// over (i, b) by a deterministic two-pass column sum over fixed row pieces.
#include "../common.cuh"

using namespace b200gf;

namespace {

constexpr int ARMA_THREADS = 256;

// the column sums cut N rows into pieces of piece_rows(N) rows
int64_t arma_pieces(int64_t N) { return N == 0 ? 0 : (N + piece_rows(N) - 1) / piece_rows(N); }

// ---------------------------------------------------------------------------------------------------------------
// forward: one thread per output (i, b, f), over the P G contiguous columns of (b, f) in both chains.
//   SEED:  state[z] = r . x_g, state[y] = r . sx_g  (sx = S~ x), broadcast over (f, p)
//   !SEED: state = r . state in place (state holds the wide hop's result)
//   out[i, b F + f] += sgn sum_{p,g} varphi z  +  (last ? h2 sum_{p,g} y : 0)
// psi / varphi: [F][E][P][G], edge feature e.
// ---------------------------------------------------------------------------------------------------------------
template <typename T, bool SEED>
__global__ void __launch_bounds__(ARMA_THREADS)
arma_scale_acc_kernel(int64_t N, int B, int G, int F, int P, int E, int e, const T* __restrict__ d,
                      const T* __restrict__ psi, const T* __restrict__ varphi, const T* __restrict__ x, int64_t x_ld,
                      const T* __restrict__ sx, int64_t sx_ld, T* state, int64_t ldw, T sgn, int last, T h2,
                      T* __restrict__ out, int64_t out_ld) {
  const int PG = P * G;
  const int64_t BQ = (int64_t)B * F * PG;
  const int64_t total = N * B * F;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = idx / ((int64_t)B * F);
    const int bf = (int)(idx - i * B * F);
    const int b = bf / F, f = bf - (bf / F) * F;
    const T di = d[i];
    const T* __restrict__ ps = psi + ((int64_t)f * E + e) * PG;
    const T* __restrict__ vp = varphi + ((int64_t)f * E + e) * PG;
    T* zr = state + i * ldw + (int64_t)bf * PG;
    T* yr = zr + BQ;
    T acc = T(0), accy = T(0);
    for (int k = 0; k < PG; ++k) {
      const T r = T(1) / (di - ps[k]);
      const int g = k % G;
      const T z = r * (SEED ? x[i * x_ld + (int64_t)b * G + g] : zr[k]);
      const T y = r * (SEED ? sx[i * sx_ld + (int64_t)b * G + g] : yr[k]);
      zr[k] = z;
      yr[k] = y;
      acc = fma(vp[k], z, acc);
      if (last) accy += y;
    }
    T v = sgn * acc;
    if (last) v = fma(h2, accy, v);
    out[i * out_ld + bf] += v;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// backward step t: one thread per (i, b, f).
//   INIT (t = tMax): Lambda = [sgn varphi dU | h2 dU];   else Lambda = R + [sgn varphi dU | 0] (R = the BWD hop's result)
//   R = r . Lambda (written in place);  acc[psi] (+)= R[z] z_t + R[y] y_{t+1};  acc[varphi] (+)= sgn dU z_t
// st: the saved forward state t.  sgn = (-1)^t.
// ---------------------------------------------------------------------------------------------------------------
template <typename T, bool INIT>
__global__ void __launch_bounds__(ARMA_THREADS)
arma_bwd_step_kernel(int64_t N, int B, int G, int F, int P, int E, int e, const T* __restrict__ d,
                     const T* __restrict__ psi, const T* __restrict__ varphi, const T* __restrict__ dy, int64_t dy_ld,
                     const T* __restrict__ st, T* R, T* __restrict__ acc, int64_t ldw, T sgn, T h2) {
  const int PG = P * G;
  const int64_t BQ = (int64_t)B * F * PG;
  const int64_t total = N * B * F;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = idx / ((int64_t)B * F);
    const int bf = (int)(idx - i * B * F);
    const int f = bf % F;
    const T di = d[i];
    const T du = dy[i * dy_ld + bf];
    const T* __restrict__ ps = psi + ((int64_t)f * E + e) * PG;
    const T* __restrict__ vp = varphi + ((int64_t)f * E + e) * PG;
    const int64_t o = i * ldw + (int64_t)bf * PG;
    for (int k = 0; k < PG; ++k) {
      const T r = T(1) / (di - ps[k]);
      const T a = sgn * vp[k] * du;
      const T lz = INIT ? a : R[o + k] + a;
      const T ly = INIT ? h2 * du : R[o + BQ + k];
      const T rz = r * lz, ry = r * ly;
      R[o + k] = rz;
      R[o + BQ + k] = ry;
      const T z = st[o + k], y = st[o + BQ + k];
      const T gp = fma(ry, y, rz * z);
      const T gv = sgn * (du * z);
      if (INIT) {
        acc[o + k] = gp;
        acc[o + BQ + k] = gv;
      } else {
        acc[o + k] += gp;
        acc[o + BQ + k] += gv;
      }
    }
  }
}

// dst[i, b G + g] = (accumulate ? dst : 0) + (sum_{f,p} R[i, chain B Q + b Q + (f P + p) G + g] + add[i, b G + g]),
// f and p ascending; add may be null.  One thread per (i, b, g).
template <typename T>
__global__ void __launch_bounds__(ARMA_THREADS)
arma_fold_kernel(int64_t N, int B, int G, int F, int P, const T* __restrict__ R, int64_t ldw, int chain,
                 const T* __restrict__ add, int64_t add_ld, T* dst, int64_t dst_ld, int accumulate) {
  const int64_t Q = (int64_t)F * P * G;
  const int64_t total = N * B * G;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = idx / ((int64_t)B * G);
    const int bg = (int)(idx - i * B * G);
    const int b = bg / G, g = bg - (bg / G) * G;
    const T* __restrict__ row = R + i * ldw + (int64_t)chain * B * Q + (int64_t)b * Q + g;
    T s = T(0);
    for (int fp = 0; fp < F * P; ++fp) s += row[(int64_t)fp * G];
    if (add) s += add[i * add_ld + bg];
    T* o = dst + i * dst_ld + bg;
    *o = accumulate ? *o + s : s;
  }
}

// pass 1: partial[piece][j] = sum over the piece's rows (ascending), then b ascending, of acc[i, half B Q + b Q + q],
// j = half Q + q.  One block per piece.
template <typename T>
__global__ void __launch_bounds__(ARMA_THREADS)
arma_colsum_partial_kernel(int64_t N, int B, int64_t Q, const T* __restrict__ acc, int64_t ldw, int64_t chunk,
                           T* __restrict__ partial) {
  const int64_t piece = blockIdx.x;
  const int64_t i0 = piece * chunk, i1 = min(N, i0 + chunk);
  for (int64_t j = threadIdx.x; j < 2 * Q; j += blockDim.x) {
    const int64_t half = j / Q, q = j - half * Q;
    const T* __restrict__ col = acc + half * B * Q + q;
    T s = T(0);
    for (int64_t i = i0; i < i1; ++i)
      for (int b = 0; b < B; ++b) s += col[i * ldw + (int64_t)b * Q];
    partial[piece * 2 * Q + j] = s;
  }
}

// pass 2: the pieces summed in order into dpsi (half 0) / dvarphi (half 1) at [f][e][p][g].
template <typename T>
__global__ void __launch_bounds__(ARMA_THREADS)
arma_colsum_reduce_kernel(int64_t pieces, int F, int P, int G, int E, int e, const T* __restrict__ partial,
                          T* __restrict__ dpsi, T* __restrict__ dvarphi) {
  const int64_t Q = (int64_t)F * P * G;
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < 2 * Q; j += (int64_t)gridDim.x * blockDim.x) {
    const int64_t half = j / Q, q = j - half * Q;
    T s = T(0);
    for (int64_t p = 0; p < pieces; ++p) s += partial[p * 2 * Q + j];
    const int64_t f = q / (P * G), pg = q - f * P * G;
    (half == 0 ? dpsi : dvarphi)[((int64_t)f * E + e) * P * G + pg] = s;
  }
}

struct ArmaDims {
  int64_t N, C, Q, ldw, ldn;
  size_t es, wide, narrow;
};

ArmaDims arma_dims(const b200gf_plan* p, int B, int G, int F, int P) {
  ArmaDims a;
  a.N = p->n_rows;
  a.Q = (int64_t)F * P * G;
  a.C = 2 * (int64_t)B * a.Q;
  a.ldw = padded_ld(a.C, p->dtype);
  a.ldn = padded_ld((int64_t)B * G, p->dtype);
  a.es = dtype_size(p->dtype);
  a.wide = (size_t)a.N * a.ldw * a.es;
  a.narrow = (size_t)a.N * a.ldn * a.es;
  return a;
}

// mode 0: forward without saved states (sx + two ping-pong states); 1: forward into caller states (sx);
// 2: backward (two adjoint states, the accumulator, two narrow buffers, the column-sum partials)
struct ArmaWs {
  void* sx = nullptr;
  void* w[2] = {nullptr, nullptr};
  void* acc = nullptr;
  void* n1 = nullptr;
  void* n2 = nullptr;
  void* partial = nullptr;
  size_t bytes = 0;
};

ArmaWs carve_arma(const b200gf_plan* p, void* ws, int B, int G, int F, int P, int mode) {
  const ArmaDims a = arma_dims(p, B, G, F, P);
  Carver c(ws);
  ArmaWs w;
  if (mode == 0 || mode == 1) w.sx = c.take(a.narrow);
  if (mode == 0 || mode == 2) {
    w.w[0] = c.take(a.wide);
    w.w[1] = c.take(a.wide);
  }
  if (mode == 2) {
    w.acc = c.take(a.wide);
    w.n1 = c.take(a.narrow);
    w.n2 = c.take(a.narrow);
    w.partial = c.take((size_t)arma_pieces(a.N) * 2 * a.Q * a.es);
  }
  w.bytes = c.off;
  return w;
}

bool arma_bad_dims(const b200gf_plan* plan, int tMax, int B, int G, int F, int P) {
  if (!plan || tMax < 0 || B <= 0 || G <= 0 || F <= 0 || P <= 0) return true;
  return plan->n_rows != plan->n_cols;                 // partitioned plans are not supported here
}

bool arma_too_wide(int B, int G, int F, int P) {
  return 2 * (int64_t)B * F * P * G > INT32_MAX || (int64_t)F * P * G > INT32_MAX / 2;
}

template <typename T>
int launch_scale_acc(bool seed, const b200gf_plan* p, int B, int G, int F, int P, int e, const void* d, const void* psi,
                     const void* varphi, const void* x, int64_t x_ld, const void* sx, int64_t sx_ld, void* state,
                     int64_t ldw, int t, int tMax, void* out, int64_t out_ld, cudaStream_t st) {
  const int64_t N = p->n_rows;
  const int grid = grid_for(N * B * F, ARMA_THREADS, p->sm_count * 8);
  const T sgn = (t & 1) ? T(-1) : T(1), h2 = ((tMax + 1) & 1) ? T(-1) : T(1);
  const T* dd = (const T*)d + (int64_t)e * N;
  if (seed)
    arma_scale_acc_kernel<T, true><<<grid, ARMA_THREADS, 0, st>>>(N, B, G, F, P, p->E, e, dd, (const T*)psi,
                                                                  (const T*)varphi, (const T*)x, x_ld, (const T*)sx,
                                                                  sx_ld, (T*)state, ldw, sgn, t == tMax, h2, (T*)out,
                                                                  out_ld);
  else
    arma_scale_acc_kernel<T, false><<<grid, ARMA_THREADS, 0, st>>>(N, B, G, F, P, p->E, e, dd, (const T*)psi,
                                                                   (const T*)varphi, nullptr, 0, nullptr, 0, (T*)state,
                                                                   ldw, sgn, t == tMax, h2, (T*)out, out_ld);
  LAUNCH_CHECK();
  return B200GF_OK;
}

template <typename T>
int arma_forward_t(const b200gf_plan* p, const void* d, const void* psi, const void* varphi, int tMax, int B, int G,
                   int F, int P, const void* x, int64_t x_ld, void* out, int64_t out_ld, void* states, const ArmaWs& w,
                   cudaStream_t st) {
  const ArmaDims a = arma_dims(p, B, G, F, P);
  int rc;
  for (int e = 0; e < p->E; ++e) {
    auto state = [&](int t) -> void* {
      return states ? (char*)states + ((size_t)e * (tMax + 1) + t) * a.wide : w.w[t & 1];
    };
    if ((rc = plan_hop(p, p->fwd[e], x, x_ld, w.sx, a.ldn, B * G, st))) return rc;
    if ((rc = launch_scale_acc<T>(true, p, B, G, F, P, e, d, psi, varphi, x, x_ld, w.sx, a.ldn, state(0), a.ldw, 0,
                                  tMax, out, out_ld, st)))
      return rc;
    for (int t = 1; t <= tMax; ++t) {
      if ((rc = plan_hop(p, p->fwd[e], state(t - 1), a.ldw, state(t), a.ldw, (int)a.C, st))) return rc;
      if ((rc = launch_scale_acc<T>(false, p, B, G, F, P, e, d, psi, varphi, nullptr, 0, nullptr, 0, state(t), a.ldw,
                                    t, tMax, out, out_ld, st)))
        return rc;
    }
  }
  return B200GF_OK;
}

template <typename T>
int arma_backward_t(const b200gf_plan* p, const void* d, const void* psi, const void* varphi, int tMax, int B, int G,
                    int F, int P, const void* dy, int64_t dy_ld, const void* states, void* dx, int64_t dx_ld, void* dpsi,
                    void* dvarphi, const ArmaWs& w, cudaStream_t st) {
  const ArmaDims a = arma_dims(p, B, G, F, P);
  const int64_t N = a.N;
  const int E = p->E;
  const int sms = p->sm_count;
  const int gstep = grid_for(N * B * F, ARMA_THREADS, sms * 8);
  const int gfold = grid_for(N * B * G, ARMA_THREADS, sms * 8);
  const T h2 = ((tMax + 1) & 1) ? T(-1) : T(1);
  const int64_t chunk = piece_rows(N), pieces = arma_pieces(N);
  int rc;
  for (int e = 0; e < E; ++e) {
    const T* dd = (const T*)d + (int64_t)e * N;
    auto saved = [&](int t) { return (const T*)((const char*)states + ((size_t)e * (tMax + 1) + t) * a.wide); };
    int cur = 0;
    arma_bwd_step_kernel<T, true><<<gstep, ARMA_THREADS, 0, st>>>(
        N, B, G, F, P, E, e, dd, (const T*)psi, (const T*)varphi, (const T*)dy, dy_ld, saved(tMax), (T*)w.w[cur],
        (T*)w.acc, a.ldw, (tMax & 1) ? T(-1) : T(1), h2);
    LAUNCH_CHECK();
    for (int t = tMax - 1; t >= 0; --t) {
      if ((rc = plan_hop(p, p->bwd[e], w.w[cur], a.ldw, w.w[1 - cur], a.ldw, (int)a.C, st))) return rc;
      cur = 1 - cur;
      arma_bwd_step_kernel<T, false><<<gstep, ARMA_THREADS, 0, st>>>(
          N, B, G, F, P, E, e, dd, (const T*)psi, (const T*)varphi, (const T*)dy, dy_ld, saved(t), (T*)w.w[cur],
          (T*)w.acc, a.ldw, (t & 1) ? T(-1) : T(1), h2);
      LAUNCH_CHECK();
    }
    if (dx) {
      arma_fold_kernel<T><<<gfold, ARMA_THREADS, 0, st>>>(N, B, G, F, P, (const T*)w.w[cur], a.ldw, 1, nullptr, 0,
                                                          (T*)w.n1, a.ldn, 0);
      LAUNCH_CHECK();
      if ((rc = plan_hop(p, p->bwd[e], w.n1, a.ldn, w.n2, a.ldn, B * G, st))) return rc;
      arma_fold_kernel<T><<<gfold, ARMA_THREADS, 0, st>>>(N, B, G, F, P, (const T*)w.w[cur], a.ldw, 0,
                                                          (const T*)w.n2, a.ldn, (T*)dx, dx_ld, 1);
      LAUNCH_CHECK();
    }
    arma_colsum_partial_kernel<T><<<(unsigned)pieces, ARMA_THREADS, 0, st>>>(N, B, a.Q, (const T*)w.acc, a.ldw, chunk,
                                                                            (T*)w.partial);
    arma_colsum_reduce_kernel<T><<<grid_for(2 * a.Q, ARMA_THREADS, sms * 8), ARMA_THREADS, 0, st>>>(
        pieces, F, P, G, E, e, (const T*)w.partial, (T*)dpsi, (T*)dvarphi);
    LAUNCH_CHECK_N(2);
  }
  return B200GF_OK;
}

}  // namespace

extern "C" {

size_t b200gf_arma_workspace_bytes(const b200gf_plan* plan, int B, int G, int F, int P, int tMax, int what) {
  if (arma_bad_dims(plan, tMax, B, G, F, P) || what < 0 || what > 3 || arma_too_wide(B, G, F, P)) return 0;
  if (what == 3) return (size_t)plan->E * (tMax + 1) * arma_dims(plan, B, G, F, P).wide;
  return carve_arma(plan, nullptr, B, G, F, P, what).bytes + 256;
}

int b200gf_arma_forward(const b200gf_plan* plan, const void* d, const void* psi, const void* varphi, int tMax, int B,
                        int G, int F, int P, const void* x, int64_t x_ld, void* out, int64_t out_ld, void* states,
                        void* workspace, size_t workspace_bytes, void* stream) {
  if (arma_bad_dims(plan, tMax, B, G, F, P) || !d || !psi || !varphi || !x || !out) return B200GF_EINVAL;
  if (x_ld < (int64_t)B * G || out_ld < (int64_t)B * F) return B200GF_EINVAL;
  if (arma_too_wide(B, G, F, P)) return B200GF_EUNSUPPORTED;
  // a misaligned states buffer is reported after a missing workspace and before a short one
  if (workspace && states && ((uintptr_t)states & 255) != 0) return B200GF_EINVAL;
  const ArmaWs w = carve_arma(plan, workspace, B, G, F, P, states ? 1 : 0);
  if (int rc = check_workspace(workspace, w.bytes, workspace_bytes, true)) return rc;
  if (plan->n_rows == 0) return B200GF_OK;
  return with_dtype(plan->dtype, [&](auto tag) {
    return arma_forward_t<decltype(tag)>(plan, d, psi, varphi, tMax, B, G, F, P, x, x_ld, out, out_ld, states, w,
                                         (cudaStream_t)stream);
  });
}

int b200gf_arma_backward(const b200gf_plan* plan, const void* d, const void* psi, const void* varphi, int tMax, int B,
                         int G, int F, int P, const void* dy, int64_t dy_ld, const void* states, void* dx, int64_t dx_ld,
                         void* dpsi, void* dvarphi, void* workspace, size_t workspace_bytes, void* stream) {
  if (arma_bad_dims(plan, tMax, B, G, F, P) || !plan->has_bwd) return B200GF_EINVAL;
  if (!d || !psi || !varphi || !dy || !states || !dpsi || !dvarphi) return B200GF_EINVAL;
  if (dy_ld < (int64_t)B * F || (dx && dx_ld < (int64_t)B * G)) return B200GF_EINVAL;
  if (arma_too_wide(B, G, F, P)) return B200GF_EUNSUPPORTED;
  const ArmaWs w = carve_arma(plan, workspace, B, G, F, P, 2);
  if (int rc = check_workspace(workspace, w.bytes, workspace_bytes, true)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (plan->n_rows == 0) {
    const size_t n = (size_t)F * plan->E * P * G * dtype_size(plan->dtype);
    CUDA_TRY(cudaMemsetAsync(dpsi, 0, n, st));
    CUDA_TRY(cudaMemsetAsync(dvarphi, 0, n, st));
    return B200GF_OK;
  }
  return with_dtype(plan->dtype, [&](auto tag) {
    return arma_backward_t<decltype(tag)>(plan, d, psi, varphi, tMax, B, G, F, P, dy, dy_ld, states, dx, dx_ld, dpsi,
                                          dvarphi, w, st);
  });
}

}  // extern "C"
