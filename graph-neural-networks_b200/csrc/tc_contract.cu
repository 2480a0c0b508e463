// Tensor-core tap contraction for FP32 (sm_90a: TMA + wgmma tf32 + mbarrier), error-compensated ("3xTF32").
//
//   out[r, q] = bias[q] + sum_t sum_p Z_t[r, p] * W_t[p, q]          r = node * B + b
//
// replaces the reference's [B,N,EKG] x [EKG,F] torch.matmul + bias (alegnn/utils/graphML.py:170-175).
// A single TF32 pass misses the 1e-4 tolerance over E*K*G = 320 terms (SURVEY.md §7 hard part 3), so every operand
// is split x = hi + lo with hi = the 19 leading bits (exact in TF32) and the product is accumulated in FP32 registers as
//   hi*hi + lo*hi + hi*lo            (the dropped lo*lo term is ~2^-22 relative).
//
// One persistent CTA per SM, 384 threads = 3 warpgroups:
//   warpgroup 0   TMA producer (one lane): per 32-float k-chunk, one 128 x 32 tile of Z_t (128-byte swizzle) + the
//                 matching Q x 32 tiles of W_hi and W_lo (pre-split, K-major) into a shared-memory ring of stages
//   warpgroups 1-2  consumers, 64 rows of the 128-row tile each: split their half of the Z tile in place (hi over the
//                 tile, lo next to it; the transform is element-wise, so the swizzled layout does not matter),
//                 fence.proxy.async, then 3 x 4 wgmma.m64nNk8 (N = Q rounded up to a power of two, the rows of W past Q
//                 are never stored) per stage into FP32 register accumulators; the stage goes back to the producer once
//                 the next stage's MMAs are issued (wgmma.wait_group 1), and the epilogue adds the bias, applies the
//                 fused ReLU and stores the accumulators straight from registers.
#include <cuda.h>

#include "common.cuh"

namespace b200gf {
namespace tc {

constexpr int BM = 128;       // rows per tile (two warpgroups x wgmma M = 64)
constexpr int BK = 32;        // floats per k-chunk = one 128-byte swizzle row
constexpr int MMA_K = 8;      // tf32: 32 bytes per instruction along K
constexpr int MAX_T = 16;     // terms (tensor maps travel as kernel parameters)
constexpr int THREADS = 384;
constexpr int A_BYTES = BM * BK * 4;  // 16 KB
constexpr int HALF_BYTES = A_BYTES / 2;
constexpr int SMEM_BUDGET = 200 * 1024;
constexpr unsigned SPIN_LIMIT = 1u << 24;  // bounded waits: a protocol bug traps instead of hanging the GPU

struct Params {
  CUtensorMap a_map[MAX_T];
  CUtensorMap bhi_map, blo_map;
  const float* bias;
  float* out;
  int64_t out_ld;
  int64_t R;        // total rows = n_rows * B
  int64_t n_rows;
  int T, P, Q, B;
  int num_tiles;
  int stages;
  int bias_per_node;
  int relu;          // epilogue activation: out = max(out, 0)  (fused GraphFilter -> ReLU layer, architectures.py:287)
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  unsigned spins = 0;
  while (true) {
    asm volatile(
        "{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
        : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    if (done) break;
    if (++spins > SPIN_LIMIT) __trap();
  }
}

__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint32_t bar, uint32_t dst, int x, int y) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(dst), "l"(map), "r"(bar), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ void tma_load_3d(const CUtensorMap* map, uint32_t bar, uint32_t dst, int x, int y, int z) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
               ::"r"(dst), "l"(map), "r"(bar), "r"(x), "r"(y), "r"(z) : "memory");
}

// wgmma shared-memory descriptor of a K-major, 128-byte-swizzled operand tile: 8-row groups 1024 bytes apart (SBO),
// LBO unused (=1), swizzle mode 1 (128 B) at bits 62-63.  Stepping along K inside the swizzle atom adds bytes to the start.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}

// D[64 x N] (+)= A[64 x 8] * B[N x 8]^T, both from shared memory; N / 2 FP32 accumulators per thread
template <int N>
__device__ __forceinline__ void wgmma_tf32(float* d, uint64_t a, uint64_t b);
template <>
__device__ __forceinline__ void wgmma_tf32<16>(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n .reg .pred p;\n setp.ne.b32 p, %10, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {"
      "%0,%1,%2,%3,%4,%5,%6,%7"
      "}, %8, %9, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(a), "l"(b), "r"(1));
}
template <>
__device__ __forceinline__ void wgmma_tf32<32>(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n .reg .pred p;\n setp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15"
      "}, %16, %17, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "r"(1));
}
template <>
__device__ __forceinline__ void wgmma_tf32<64>(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n .reg .pred p;\n setp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31"
      "}, %32, %33, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(1));
}
template <>
__device__ __forceinline__ void wgmma_tf32<128>(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n .reg .pred p;\n setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
      "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"
      "}, %64, %65, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(1));
}
template <>
__device__ __forceinline__ void wgmma_tf32<256>(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n .reg .pred p;\n setp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
      "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
      "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,"
      "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,"
      "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,"
      "%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127"
      "}, %128, %129, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(a), "l"(b), "r"(1));
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ float tf32_hi(float v) { return __uint_as_float(__float_as_uint(v) & 0xFFFFE000u); }

__host__ __device__ constexpr int b_bytes(int NP) { return NP * BK * 4; }
__host__ __device__ constexpr int stage_bytes(int NP) { return 2 * A_BYTES + 2 * b_bytes(NP); }

// NP: the wgmma N, Q rounded up to a power of two (16 .. 256)
template <int NP>
__global__ void __launch_bounds__(THREADS, 1) tc_contract_kernel(const __grid_constant__ Params prm) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  // 1024-byte alignment for the 128-byte swizzle atoms
  unsigned char* smem = (unsigned char*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  constexpr int SB = stage_bytes(NP);
  const int S = prm.stages;
  const int Q = prm.Q;
  uint64_t* full = (uint64_t*)(smem + (size_t)S * SB);   // [S] TMA landed
  uint64_t* empty = full + S;                            // [S] both consumers' MMAs done with the stage

  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;
  const int cpt = prm.P / BK;                      // k-chunks per term
  const int chunks = prm.T * cpt;

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(smem_u32(full + s), 1);
      mbar_init(smem_u32(empty + s), 8);           // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer
    if (threadIdx.x == 0) {
      const uint32_t tx = A_BYTES + 2 * Q * BK * 4;
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < prm.num_tiles; tile += gridDim.x) {
        for (int t = 0; t < prm.T; ++t) {
          for (int pc = 0; pc < cpt; ++pc, ++it) {
            const int s = it % S;
            const uint32_t ph = (it / S) & 1;
            mbar_wait(smem_u32(empty + s), ph ^ 1);
            unsigned char* st = smem + (size_t)s * SB;
            const uint32_t bar = smem_u32(full + s);
            mbar_expect_tx(bar, tx);
            tma_load_2d(&prm.a_map[t], bar, smem_u32(st), pc * BK, tile * BM);
            tma_load_3d(&prm.bhi_map, bar, smem_u32(st + 2 * A_BYTES), pc * BK, 0, t);
            tma_load_3d(&prm.blo_map, bar, smem_u32(st + 2 * A_BYTES + b_bytes(NP)), pc * BK, 0, t);
          }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers (warpgroups 1 and 2)
  const int h = wg - 1;                            // which 64-row half of the tile
  const int tid = threadIdx.x & 127;
  const int wq = tid >> 5;                         // warp within the warpgroup: rows 16 wq .. 16 wq + 15
  uint32_t it = 0;
  for (int tile = blockIdx.x; tile < prm.num_tiles; tile += gridDim.x) {
    float d[NP / 2];
#pragma unroll
    for (int i = 0; i < NP / 2; ++i) d[i] = 0.f;
    for (int c = 0; c < chunks; ++c, ++it) {
      const int s = it % S;
      const uint32_t ph = (it / S) & 1;
      mbar_wait(smem_u32(full + s), ph);
      unsigned char* st = smem + (size_t)s * SB;
      float4* A = (float4*)(st + h * HALF_BYTES);
      float4* Alo = (float4*)(st + A_BYTES + h * HALF_BYTES);
#pragma unroll
      for (int i = 0; i < HALF_BYTES / 16 / 128; ++i) {
        const int idx = i * 128 + tid;
        const float4 v = A[idx];
        float4 hi, lo;
        hi.x = tf32_hi(v.x); hi.y = tf32_hi(v.y); hi.z = tf32_hi(v.z); hi.w = tf32_hi(v.w);
        lo.x = v.x - hi.x; lo.y = v.y - hi.y; lo.z = v.z - hi.z; lo.w = v.w - hi.w;
        A[idx] = hi;
        Alo[idx] = lo;
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic writes -> visible to the tensor core
      asm volatile("bar.sync %0, 128;" ::"r"(wg) : "memory");         // the whole half is split before any MMA reads it
      const uint32_t sa = smem_u32(st);
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < BK / MMA_K; ++j) {
        const uint64_t a_hi = gmma_desc(sa + h * HALF_BYTES + j * MMA_K * 4);
        const uint64_t a_lo = gmma_desc(sa + A_BYTES + h * HALF_BYTES + j * MMA_K * 4);
        const uint64_t b_hi = gmma_desc(sa + 2 * A_BYTES + j * MMA_K * 4);
        const uint64_t b_lo = gmma_desc(sa + 2 * A_BYTES + b_bytes(NP) + j * MMA_K * 4);
        wgmma_tf32<NP>(d, a_hi, b_hi);
        wgmma_tf32<NP>(d, a_lo, b_hi);
        wgmma_tf32<NP>(d, a_hi, b_lo);
      }
      wgmma_commit();
      wgmma_wait<1>();                             // the previous stage's MMAs have retired: hand it back
      if (c > 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(empty + (it - 1) % S));
      }
    }
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(empty + (it - 1) % S));

    // epilogue: accumulator d[4 n + 2 i + j] holds row 16 wq + lane / 4 + 8 i, column 8 n + 2 (lane % 4) + j
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int64_t r = (int64_t)tile * BM + h * 64 + wq * 16 + (lane >> 2) + 8 * i;
      if (r >= prm.R) continue;
      const int64_t n = r / prm.B;
      const int b = (int)(r - n * prm.B);
      float* orow = prm.out + n * prm.out_ld + (int64_t)b * Q;
#pragma unroll
      for (int nb = 0; nb < NP / 8; ++nb) {
        const int q = nb * 8 + 2 * (lane & 3);
        if (q >= Q) break;
        float2 o = make_float2(d[4 * nb + 2 * i], d[4 * nb + 2 * i + 1]);
        if (prm.bias) {
          if (prm.bias_per_node) {
            o.x += prm.bias[(int64_t)q * prm.n_rows + n]; o.y += prm.bias[(int64_t)(q + 1) * prm.n_rows + n];
          } else {
            o.x += __ldg(prm.bias + q); o.y += __ldg(prm.bias + q + 1);
          }
        }
        if (prm.relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); }
        *reinterpret_cast<float2*>(orow + q) = o;
      }
    }
  }
}

// taps h[F,E,K,G] -> K-major hi / lo operand tiles Whi/Wlo [t][Q][P]
//   forward  (to_input = 0): Q = F, P = G,  W[t][f][g] = tap(t, f, g)
//   backward (to_input = 1): Q = G, P = F,  W[t][g][f] = tap(t, f, g)
__global__ void pack_taps_split_kernel(const float* __restrict__ h, float* __restrict__ Whi, float* __restrict__ Wlo,
                                       int F, int E, int K, int G, int to_input) {
  const int Tn = 1 + E * (K - 1);
  const int64_t total = (int64_t)Tn * G * F;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i / ((int64_t)G * F));
    const int rem = (int)(i - (int64_t)t * G * F);
    int f, g;
    if (to_input) { g = rem / F; f = rem % F; }
    else { f = rem / G; g = rem % G; }
    float val;
    if (t == 0) {
      val = 0.f;
      for (int e = 0; e < E; ++e) val += h[(((int64_t)f * E + e) * K + 0) * G + g];
    } else {
      const int e = (t - 1) / (K - 1), k = (t - 1) % (K - 1) + 1;
      val = h[(((int64_t)f * E + e) * K + k) * G + g];
    }
    const float hi = tf32_hi(val);
    Whi[i] = hi;
    Wlo[i] = val - hi;
  }
}

// generic W[T][P][Q] (p-major, the b200gf_tap_contract layout) -> Whi/Wlo [t][Q][P]
__global__ void split_w_kernel(const float* __restrict__ W, float* __restrict__ Whi, float* __restrict__ Wlo, int T, int P,
                               int Q) {
  const int64_t total = (int64_t)T * P * Q;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i / ((int64_t)P * Q));
    const int rem = (int)(i - (int64_t)t * P * Q);
    const int q = rem / P, p = rem % P;
    const float val = W[((int64_t)t * P + p) * Q + q];
    const float hi = tf32_hi(val);
    Whi[i] = hi;
    Wlo[i] = val - hi;
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
    else
      (void)cudaGetLastError();
  }
  return fn;
}

// wgmma N for Q outputs: the next power of two (the B tile rows past Q are never stored)
static int n_pad(int Q) {
  int n = 16;
  while (n < Q) n <<= 1;
  return n;
}

static int stages_for(int Q) {
  int s = SMEM_BUDGET / stage_bytes(n_pad(Q));
  if (s > 4) s = 4;
  return s;
}

template <int NP>
static cudaError_t launch_np(const Params& prm, int grid, cudaStream_t st) {
  const size_t smem = (size_t)prm.stages * stage_bytes(NP) + 1024 /*alignment slack*/ + 256 /*barriers*/;
  cudaError_t e = cudaFuncSetAttribute(tc_contract_kernel<NP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  tc_contract_kernel<NP><<<grid, THREADS, smem, st>>>(prm);
  return cudaSuccess;
}

}  // namespace tc

size_t tc_contract_scratch_bytes(int T, int P, int Q) { return align_up((size_t)2 * T * P * Q * sizeof(float), 256); }

bool tc_contract_eligible(int dtype, int64_t n_rows, int B, int P, int Q, int T, const void* const* zs,
                          const int64_t* z_ld, const void* out, int64_t out_ld, int accumulate) {
  if (dtype != B200GF_F32 || accumulate) return false;
  if (T < 1 || T > tc::MAX_T) return false;
  if (P % tc::BK != 0 || Q % 16 != 0 || Q < 16 || Q > 256) return false;
  if (tc::stages_for(Q) < 2) return false;
  if (n_rows * B < tc::BM) return false;                        // tiny problems: the FMA kernel is launch-bound anyway
  if (n_rows * B > (int64_t)INT32_MAX) return false;             // TMA coordinates are 32-bit
  if ((reinterpret_cast<uintptr_t>(out) & 15) != 0 || out_ld % 4 != 0) return false;
  for (int t = 0; t < T; ++t) {
    if (z_ld[t] != (int64_t)B * P) return false;                 // rows (n, b) must be uniformly P apart
    if ((reinterpret_cast<uintptr_t>(zs[t]) & 15) != 0) return false;
  }
  return tc::get_encode() != nullptr;
}

int launch_pack_taps_split(const void* h, void* whi_wlo, int F, int E, int K, int G, int to_input, cudaStream_t st) {
  const int64_t total = (int64_t)(1 + E * (K - 1)) * G * F;
  float* hi = (float*)whi_wlo;
  float* lo = hi + total;
  const int blocks = (int)imin64((total + 255) / 256, 132 * 8);
  tc::pack_taps_split_kernel<<<blocks, 256, 0, st>>>((const float*)h, hi, lo, F, E, K, G, to_input);
  LAUNCH_CHECK();
  return B200GF_OK;
}

int launch_split_w(const void* W, void* whi_wlo, int T, int P, int Q, cudaStream_t st) {
  const int64_t total = (int64_t)T * P * Q;
  float* hi = (float*)whi_wlo;
  float* lo = hi + total;
  const int blocks = (int)imin64((total + 255) / 256, 132 * 8);
  tc::split_w_kernel<<<blocks, 256, 0, st>>>((const float*)W, hi, lo, T, P, Q);
  LAUNCH_CHECK();
  return B200GF_OK;
}

// whi_wlo: device [2][T][Q][P] (hi then lo), K-major; everything else as launch_tap_contract
int launch_tc_contract(int sm_count, int64_t n_rows, int B, int P, int Q, int T, const void* const* zs,
                       const void* whi_wlo, const void* bias, int bias_per_node, void* out, int64_t out_ld,
                       cudaStream_t st, int act) {
  using namespace tc;
  EncodeTiledFn encode = get_encode();
  if (!encode) return B200GF_EUNSUPPORTED;
  Params prm;
  const int64_t R = n_rows * B;
  for (int t = 0; t < T; ++t) {
    const cuuint64_t dims[2] = {(cuuint64_t)P, (cuuint64_t)R};
    const cuuint64_t strides[1] = {(cuuint64_t)P * 4};
    const cuuint32_t box[2] = {BK, BM};
    const cuuint32_t estr[2] = {1, 1};
    if (encode(&prm.a_map[t], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(zs[t]), dims, strides, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return B200GF_EINVAL;
  }
  for (int t = T; t < MAX_T; ++t) prm.a_map[t] = prm.a_map[0];
  {
    const cuuint64_t dims[3] = {(cuuint64_t)P, (cuuint64_t)Q, (cuuint64_t)T};
    const cuuint64_t strides[2] = {(cuuint64_t)P * 4, (cuuint64_t)P * Q * 4};
    const cuuint32_t box[3] = {BK, (cuuint32_t)Q, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    float* hi = (float*)const_cast<void*>(whi_wlo);
    float* lo = hi + (int64_t)T * P * Q;
    if (encode(&prm.bhi_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, hi, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return B200GF_EINVAL;
    if (encode(&prm.blo_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, lo, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return B200GF_EINVAL;
  }
  prm.bias = (const float*)bias;
  prm.out = (float*)out;
  prm.out_ld = out_ld;
  prm.R = R;
  prm.n_rows = n_rows;
  prm.T = T; prm.P = P; prm.Q = Q; prm.B = B;
  prm.num_tiles = (int)((R + BM - 1) / BM);
  prm.stages = stages_for(Q);
  prm.bias_per_node = bias_per_node;
  prm.relu = act;
  const int grid = prm.num_tiles < sm_count ? prm.num_tiles : sm_count;
  switch (n_pad(Q)) {
    case 16: CUDA_TRY(launch_np<16>(prm, grid, st)); break;
    case 32: CUDA_TRY(launch_np<32>(prm, grid, st)); break;
    case 64: CUDA_TRY(launch_np<64>(prm, grid, st)); break;
    case 128: CUDA_TRY(launch_np<128>(prm, grid, st)); break;
    case 256: CUDA_TRY(launch_np<256>(prm, grid, st)); break;
    default: return B200GF_EUNSUPPORTED;
  }
  LAUNCH_CHECK();
  return B200GF_OK;
}

}  // namespace b200gf
