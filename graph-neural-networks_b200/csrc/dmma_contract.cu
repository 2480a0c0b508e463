// FP64 tap contraction on the FP64 tensor-core path (mma.sync.m8n8k4.f64 — DMMA), the contraction of the reference's
// default dtype (every example runs torch.float64: examples/sourceLocGNN.py:40):
//
//     out[(n,b), q] = act( bias + sum_t sum_p Z_t[(n,b), p] * W[t][p][q] )       (graphML.py:170-175)
//
// replaces tap_contract_kernel<double> (4x4 register-tile FMA) when eligible.
//
// Mapping: persistent CTAs (256 threads, one per SM and 64-column block of Q).  The taps of the CTA's column block,
// W[T][P][64], stay in shared memory for the whole kernel (row pitch 68 doubles: the four k-rows of a B fragment land 8
// banks apart, so a half-warp's 64-bit loads are conflict-free); Z tiles (128 rows x 16 k) stream through two
// register-staged shared-memory buffers (row pitch 20 doubles).  Each warp owns 16 rows x (8 NJ) columns = 2 x NJ
// accumulator fragments; per k4-step a lane issues 2 + NJ LDS.64 for 2 NJ DMMA.
#include "common.cuh"

namespace b200gf {
namespace dmma {

constexpr int BM = 128, BKC = 16;
constexpr int WP_PAD = 4;     // W row pitch = QB + 4 doubles
constexpr int ZP = 20;        // pitch of a Z-tile row (doubles)
constexpr int THREADS = 256;
constexpr int MAX_T = 16;

struct Params {
  const double* Z[MAX_T];
  int64_t z_ld[MAX_T];
  const double* W;            // [T][P][Q]
  const double* bias;         // [Q], [Q, n_rows] or null
  double* out;
  int64_t out_ld;
  int64_t R, n_rows;
  int T, P, Q, B, num_tiles, bias_per_node, relu;
};

__device__ __forceinline__ void dmma(double& d0, double& d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
               : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}

template <int NJ>   // NJ 8-column fragments per warp row block: column block QB = 8 * NJ (64 or 32)
__global__ void __launch_bounds__(THREADS, 1) contract_f64_kernel(const __grid_constant__ Params prm) {
  constexpr int QB = 8 * NJ, WP = QB + WP_PAD;
  extern __shared__ __align__(16) unsigned char smem_dmma[];
  double* Ws = reinterpret_cast<double*>(smem_dmma);                   // [T*P][WP]
  const int T = prm.T, P = prm.P, Q = prm.Q, B = prm.B;
  double* Zs = Ws + (size_t)T * P * WP;                                // [2][BM][ZP]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int q0 = blockIdx.y * QB;
  for (int i = tid; i < T * P * QB; i += THREADS) {
    const int row = i / QB, qq = i - row * QB;
    Ws[(size_t)row * WP + qq] = prm.W[(size_t)row * Q + q0 + qq];
  }
  __syncthreads();

  const int cpt = P / BKC;                                             // k-chunks per term
  const int chunks = T * cpt;
  // loader mapping: thread -> (row = tid / 2, 8 consecutive k = (tid % 2) * 8 .. +7) as four double2
  const int l_row = tid >> 1, l_k = (tid & 1) * 8;
  const int fr = lane >> 2, fk = lane & 3;                             // fragment coordinates

  for (int tile = blockIdx.x; tile < prm.num_tiles; tile += gridDim.x) {
    const int64_t r0 = (int64_t)tile * BM;
    double acc[2][NJ][2];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < NJ; ++j) { acc[i][j][0] = 0.0; acc[i][j][1] = 0.0; }
    // this thread's loader row (n, b) -> base offsets
    const int64_t lr = r0 + l_row;
    const bool l_ok = lr < prm.R;
    const int64_t ln = l_ok ? lr / B : 0;
    const int lb = l_ok ? (int)(lr - ln * B) : 0;
    double2 stage[4];
    auto fetch = [&](int c) {
      const int t = c / cpt, p0 = (c - t * cpt) * BKC;
      if (l_ok) {
        const double2* src = reinterpret_cast<const double2*>(prm.Z[t] + ln * prm.z_ld[t] + (int64_t)lb * P + p0 + l_k);
#pragma unroll
        for (int i = 0; i < 4; ++i) stage[i] = __ldg(src + i);
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) stage[i] = make_double2(0.0, 0.0);
      }
    };
    auto stash = [&](int buf) {
      double2* dst = reinterpret_cast<double2*>(Zs + ((size_t)buf * BM + l_row) * ZP + l_k);
#pragma unroll
      for (int i = 0; i < 4; ++i) dst[i] = stage[i];
    };
    fetch(0);
    __syncthreads();            // the previous tile's last reads of Zs are done
    stash(0);
    __syncthreads();
    for (int c = 0; c < chunks; ++c) {
      const int buf = c & 1;
      if (c + 1 < chunks) fetch(c + 1);
      const int t = c / cpt, p0 = (c - t * cpt) * BKC;
      const double* zt = Zs + ((size_t)buf * BM + warp * 16) * ZP;
      const double* wt = Ws + ((size_t)t * P + p0) * WP;
#pragma unroll
      for (int k4 = 0; k4 < BKC; k4 += 4) {
        const double a0 = zt[(fr) * ZP + k4 + fk];
        const double a1 = zt[(8 + fr) * ZP + k4 + fk];
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          const double b = wt[(k4 + fk) * WP + j * 8 + fr];
          dmma(acc[0][j][0], acc[0][j][1], a0, b);
          dmma(acc[1][j][0], acc[1][j][1], a1, b);
        }
      }
      if (c + 1 < chunks) stash(buf ^ 1);     // the other buffer was last read in iteration c-1 (barrier below)
      __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int64_t r = r0 + warp * 16 + i * 8 + fr;
      if (r < prm.R) {
        const int64_t n = r / B;
        const int b = (int)(r - n * B);
        double* o = prm.out + n * prm.out_ld + (int64_t)b * Q + q0 + fk * 2;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          double v0 = acc[i][j][0], v1 = acc[i][j][1];
          if (prm.bias) {
            const int q = q0 + j * 8 + fk * 2;
            if (prm.bias_per_node) { v0 += prm.bias[(int64_t)q * prm.n_rows + n]; v1 += prm.bias[(int64_t)(q + 1) * prm.n_rows + n]; }
            else { v0 += __ldg(prm.bias + q); v1 += __ldg(prm.bias + q + 1); }
          }
          if (prm.relu) { v0 = v0 > 0.0 ? v0 : 0.0; v1 = v1 > 0.0 ? v1 : 0.0; }
          *reinterpret_cast<double2*>(o + j * 8) = make_double2(v0, v1);
        }
      }
    }
  }
}

static size_t smem_bytes(int T, int P, int QB) { return ((size_t)T * P * (QB + WP_PAD) + (size_t)2 * BM * ZP) * 8; }

}  // namespace dmma

bool dmma_contract_eligible(int dtype, int64_t n_rows, int B, int P, int Q, int T, const void* const* zs,
                            const int64_t* z_ld, const void* out, int64_t out_ld, int accumulate) {
  if (dtype != B200GF_F64 || accumulate) return false;
  if (T < 1 || T > dmma::MAX_T || P % dmma::BKC != 0) return false;
  if (!(Q % 64 == 0 || Q == 32)) return false;
  const int QB = Q % 64 == 0 ? 64 : 32;
  if (dmma::smem_bytes(T, P, QB) > 227 * 1024) return false;
  if (n_rows * B < dmma::BM) return false;                                  // tiny problems: launch-bound either way
  if ((reinterpret_cast<uintptr_t>(out) & 15) != 0 || out_ld % 2 != 0) return false;
  for (int t = 0; t < T; ++t)
    if (z_ld[t] % 2 != 0 || (reinterpret_cast<uintptr_t>(zs[t]) & 15) != 0) return false;
  return true;
}

int launch_dmma_contract(int sm_count, int64_t n_rows, int B, int P, int Q, int T, const void* const* zs,
                         const int64_t* z_ld, const void* W, const void* bias, int bias_per_node, void* out,
                         int64_t out_ld, cudaStream_t st, int act) {
  using namespace dmma;
  Params prm;
  for (int t = 0; t < MAX_T; ++t) {
    prm.Z[t] = reinterpret_cast<const double*>(zs[t < T ? t : 0]);
    prm.z_ld[t] = z_ld[t < T ? t : 0];
  }
  prm.W = (const double*)W; prm.bias = (const double*)bias; prm.out = (double*)out; prm.out_ld = out_ld;
  prm.R = n_rows * B; prm.n_rows = n_rows;
  prm.T = T; prm.P = P; prm.Q = Q; prm.B = B; prm.bias_per_node = bias_per_node; prm.relu = act;
  prm.num_tiles = (int)((prm.R + BM - 1) / BM);
  const int QB = Q % 64 == 0 ? 64 : 32;
  const int qblocks = Q / QB;
  const size_t smem = smem_bytes(T, P, QB);
  int gx = sm_count / qblocks;
  if (gx < 1) gx = 1;
  if (gx > prm.num_tiles) gx = prm.num_tiles;
  dim3 grid((unsigned)gx, (unsigned)qblocks);
  if (QB == 64) {
    CUDA_TRY(cudaFuncSetAttribute(contract_f64_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    contract_f64_kernel<8><<<grid, THREADS, smem, st>>>(prm);
  } else {
    CUDA_TRY(cudaFuncSetAttribute(contract_f64_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    contract_f64_kernel<4><<<grid, THREADS, smem, st>>>(prm);
  }
  LAUNCH_CHECK();
  return B200GF_OK;
}

}  // namespace b200gf
