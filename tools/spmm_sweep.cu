// Tuning sweep for the hop kernel (spmm_kernels.cuh) on a synthetic random graph.  Not part of the library.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 tools/spmm_sweep.cu -o tools/spmm_sweep
//   tools/spmm_sweep [N=1000000] [deg=32] [C=64] [reps=10] [peakGBs=3350 (H100 SXM data sheet)]
// Prints one line per variant: registers, resident blocks/SM, ms per hop, algorithmic GB/s (gather model,
// SURVEY.md §8d) and the fraction of the given HBM bandwidth.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include <random>
#include <vector>

#include "../graph-neural-networks_b200/csrc/spmm_kernels.cuh"
#include "spmm_async_variant.cuh"

using namespace b200gf;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1);} } while (0)

struct Problem {
  int64_t N; int C; int64_t nnz;
  int64_t* rowptr; int32_t* rowptr32; int32_t* col; float* val; float* src; float* dst; float* ref;
  int sm_count;
  double bytes;
};

template <int L, int U, int THREADS, int MINB, int HINT, bool PF, int SH = 0>
double run(const Problem& P, const char* name, int reps, double peak, int blocks_per_sm_override = 0, bool is_ref = false,
         float frac = 1.0f) {
  auto kern = spmm_hop_kernel<float, 4, L, U, THREADS, MINB, HINT, PF, SH>;
  cudaFuncAttributes fa;
  CK(cudaFuncGetAttributes(&fa, kern));
  int occ = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, THREADS, 0));
  int use = blocks_per_sm_override > 0 ? std::min(blocks_per_sm_override, occ) : occ;
  const int n_chunks = (P.C + L * 4 - 1) / (L * 4);
  const int64_t items = P.N * n_chunks;
  int64_t blocks = std::min<int64_t>((items + THREADS / 32 - 1) / (THREADS / 32), (int64_t)P.sm_count * use);
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  CK(cudaMemset(P.dst, 0xff, (size_t)P.N * P.C * 4));
  for (int i = 0; i < 2; ++i)
    kern<<<(unsigned)blocks, THREADS>>>(P.rowptr, P.col, P.val, P.src, P.C, P.dst, P.C, P.N, P.C, n_chunks, frac, ScatterArgs<float>{});
  CK(cudaGetLastError());
  CK(cudaDeviceSynchronize());
  float best = 1e30f, sum = 0;
  for (int i = 0; i < reps; ++i) {
    CK(cudaEventRecord(e0));
    kern<<<(unsigned)blocks, THREADS>>>(P.rowptr, P.col, P.val, P.src, P.C, P.dst, P.C, P.N, P.C, n_chunks, frac, ScatterArgs<float>{});
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
    best = std::min(best, ms); sum += ms;
  }
  // correctness vs the first variant
  double maxdiff = 0;
  if (is_ref) {
    CK(cudaMemcpy(P.ref, P.dst, (size_t)P.N * P.C * 4, cudaMemcpyDeviceToDevice));
  } else {
    std::vector<float> a(1 << 16), b(1 << 16);
    CK(cudaMemcpy(a.data(), P.dst, a.size() * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(b.data(), P.ref, b.size() * 4, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < a.size(); ++i) maxdiff = std::max(maxdiff, (double)fabsf(a[i] - b[i]));
  }
  const double avg = sum / reps;
  printf("%-34s regs=%3d occ=%2d use=%2d blocks=%6lld  avg %.3f ms  best %.3f ms  %.0f GB/s  frac %.3f  maxdiff %.2e\n",
         name, fa.numRegs, occ, use, (long long)blocks, avg, best, P.bytes / (avg * 1e-3) / 1e9,
         P.bytes / (avg * 1e-3) / 1e9 / peak, maxdiff);
  fflush(stdout);
  return avg;
}


template <typename KernT, typename LaunchT>
double time_variant(const Problem& P, const char* name, int reps, double peak, KernT kern, int threads, size_t smem,
                    int blocks_per_sm_cap, int64_t max_blocks, LaunchT launch) {
  cudaFuncAttributes fa;
  if (smem > 48 * 1024) CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CK(cudaFuncGetAttributes(&fa, kern));
  int occ = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, smem));
  int use = blocks_per_sm_cap > 0 ? std::min(blocks_per_sm_cap, occ) : occ;
  int64_t blocks = std::min<int64_t>(max_blocks, (int64_t)P.sm_count * use);
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  CK(cudaMemset(P.dst, 0xff, (size_t)P.N * P.C * 4));
  for (int i = 0; i < 2; ++i) launch((unsigned)blocks);
  CK(cudaGetLastError());
  CK(cudaDeviceSynchronize());
  float best = 1e30f, sum = 0;
  for (int i = 0; i < reps; ++i) {
    CK(cudaEventRecord(e0));
    launch((unsigned)blocks);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
    best = std::min(best, ms); sum += ms;
  }
  // full comparison against the reference variant's output
  std::vector<float> a((size_t)P.N * P.C), b((size_t)P.N * P.C);
  CK(cudaMemcpy(a.data(), P.dst, a.size() * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(b.data(), P.ref, b.size() * 4, cudaMemcpyDeviceToHost));
  double maxdiff = 0;
  for (size_t i = 0; i < a.size(); ++i) {
    double d = fabs((double)a[i] - (double)b[i]);
    if (!(d <= maxdiff)) maxdiff = d;   // NaN-propagating
  }
  const double avg = sum / reps;
  printf("%-34s regs=%3d smem=%6zu occ=%2d use=%2d blocks=%6lld  avg %.3f ms  best %.3f ms  %.0f GB/s  frac %.3f  maxdiff(all) %.2e\n",
         name, fa.numRegs, smem, occ, use, (long long)blocks, avg, best, P.bytes / (avg * 1e-3) / 1e9,
         P.bytes / (avg * 1e-3) / 1e9 / peak, maxdiff);
  fflush(stdout);
  return avg;
}

template <int L, int U, int THREADS, int MINB, int HINT, int SH = 0>
double run_v2w(const Problem& P, const char* name, int reps, double peak, float frac = 1.0f) {   // 256-bit loads (VEC = 8)
  const int n_chunks = (P.C + L * 8 - 1) / (L * 8);
  const int64_t maxb = ((int64_t)P.N + THREADS / 32 - 1) / (THREADS / 32);
  auto kern = spmm_hop_v2_kernel<float, int32_t, 8, L, U, THREADS, MINB, HINT, 0, SH>;
  return time_variant(P, name, reps, peak, kern, THREADS, 0, 0, maxb, [&](unsigned blocks) {
    kern<<<dim3(blocks, n_chunks), THREADS>>>(P.rowptr32, P.col, P.val, P.src, P.C, P.dst, P.C, (int)P.N, P.C, frac, ScatterParam<float, 0>{});
  });
}

template <int L, int U, int THREADS, int MINB, int HINT, bool I32>
double run_v2(const Problem& P, const char* name, int reps, double peak) {
  const int n_chunks = (P.C + L * 4 - 1) / (L * 4);
  const int64_t maxb = ((int64_t)P.N + THREADS / 32 - 1) / (THREADS / 32);
  if constexpr (I32) {
    auto kern = spmm_hop_v2_kernel<float, int32_t, 4, L, U, THREADS, MINB, HINT, 0>;
    return time_variant(P, name, reps, peak, kern, THREADS, 0, 0, maxb, [&](unsigned blocks) {
      kern<<<dim3(blocks, n_chunks), THREADS>>>(P.rowptr32, P.col, P.val, P.src, P.C, P.dst, P.C, (int)P.N, P.C, 1.0f, ScatterParam<float, 0>{});
    });
  } else {
    auto kern = spmm_hop_v2_kernel<float, int64_t, 4, L, U, THREADS, MINB, HINT, 0>;
    return time_variant(P, name, reps, peak, kern, THREADS, 0, 0, maxb, [&](unsigned blocks) {
      kern<<<dim3(blocks, n_chunks), THREADS>>>(P.rowptr, P.col, P.val, P.src, P.C, P.dst, P.C, (int)P.N, P.C, 1.0f, ScatterParam<float, 0>{});
    });
  }
}

template <int L, int SLOTS, int THREADS, int MINB, int HINT>
double run_async(const Problem& P, const char* name, int reps, double peak) {
  const int n_chunks = (P.C + L * 4 - 1) / (L * 4);
  const size_t smem = (size_t)(THREADS / 32) * 2 * SLOTS * L * 16;
  const int64_t nblk = (P.N + 31) / 32;
  const int64_t maxb = (nblk + THREADS / 32 - 1) / (THREADS / 32);
  auto kern = spmm_hop_async_kernel<float, int32_t, 4, L, SLOTS, THREADS, MINB, HINT, 0>;
  return time_variant(P, name, reps, peak, kern, THREADS, smem, 0, maxb, [&](unsigned blocks) {
    kern<<<dim3(blocks, n_chunks), THREADS, smem>>>(P.rowptr32, P.col, P.val, P.src, P.C, P.dst, P.C, (int)P.N, P.C, ScatterParam<float, 0>{});
  });
}

// multi-row-per-warp kernel for narrow rows
template <int L, int GS, int U, int MINB, int HINT>
double run_mr(const Problem& P, const char* name, int reps, double peak) {
  constexpr int THREADS = 256;
  auto kern = spmm_hop_multirow_kernel<float, 4, L, GS, U, THREADS, MINB, HINT>;
  cudaFuncAttributes fa;
  CK(cudaFuncGetAttributes(&fa, kern));
  int occ = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, THREADS, 0));
  const int rpw = 32 / GS;
  const int64_t warps_needed = (P.N + rpw - 1) / rpw;
  int64_t blocks = std::min<int64_t>((warps_needed + 7) / 8, (int64_t)P.sm_count * occ);
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  CK(cudaMemset(P.dst, 0xff, (size_t)P.N * P.C * 4));
  for (int i = 0; i < 2; ++i) kern<<<(unsigned)blocks, THREADS>>>(P.rowptr, P.col, P.val, P.src, P.C, P.dst, P.C, P.N, P.C, ScatterArgs<float>{});
  CK(cudaGetLastError());
  CK(cudaDeviceSynchronize());
  float sum = 0;
  for (int i = 0; i < reps; ++i) {
    CK(cudaEventRecord(e0));
    kern<<<(unsigned)blocks, THREADS>>>(P.rowptr, P.col, P.val, P.src, P.C, P.dst, P.C, P.N, P.C, ScatterArgs<float>{});
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
    sum += ms;
  }
  std::vector<float> a(1 << 16), b(1 << 16);
  CK(cudaMemcpy(a.data(), P.dst, a.size() * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(b.data(), P.ref, b.size() * 4, cudaMemcpyDeviceToHost));
  double maxdiff = 0;
  for (size_t i = 0; i < a.size(); ++i) maxdiff = std::max(maxdiff, (double)fabsf(a[i] - b[i]));
  const double avg = sum / reps;
  printf("%-34s regs=%3d occ=%2d blocks=%6lld  avg %.3f ms  %.0f GB/s  frac %.3f  maxdiff %.2e\n", name, fa.numRegs, occ,
         (long long)blocks, avg, P.bytes / (avg * 1e-3) / 1e9, P.bytes / (avg * 1e-3) / 1e9 / peak, maxdiff);
  fflush(stdout);
  return avg;
}

// multi-row kernel with 32-byte lanes (VEC = 8)
template <int L, int GS, int U, int MINB, int HINT, int VEC = 8>
double run_mr_w(const Problem& P, const char* name, int reps, double peak) {
  constexpr int THREADS = 256;
  auto kern = spmm_hop_multirow_v2_kernel<float, int32_t, VEC, L, GS, U, THREADS, MINB, HINT, 0>;
  const int rpw = 32 / GS;
  const int64_t warps_needed = (P.N + rpw - 1) / rpw;
  return time_variant(P, name, reps, peak, kern, THREADS, 0, 0, (warps_needed + 7) / 8, [&](unsigned blocks) {
    kern<<<blocks, THREADS>>>(P.rowptr32, P.col, P.val, P.src, P.C, P.dst, P.C, (int)P.N, P.C, ScatterParam<float, 0>{});
  });
}

int main(int argc, char** argv) {
  const int64_t N = argc > 1 ? atoll(argv[1]) : 1000000;
  const int deg = argc > 2 ? atoi(argv[2]) : 32;
  const int C = argc > 3 ? atoi(argv[3]) : 64;
  const int reps = argc > 4 ? atoi(argv[4]) : 10;
  const double peak = argc > 5 ? atof(argv[5]) : 3350.0;
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
  printf("device %s  SMs %d  N=%lld deg=%d C=%d\n", prop.name, prop.multiProcessorCount, (long long)N, deg, C);
  printf("L2 %d MB, persistingL2CacheMaxSize %d MB, accessPolicyMaxWindowSize %d MB\n", prop.l2CacheSize >> 20,
         prop.persistingL2CacheMaxSize >> 20, prop.accessPolicyMaxWindowSize >> 20);
  if (getenv("SWEEP_PERSIST_MB")) {   // L2 set-aside for evict_last ("persisting") lines; the default is 0
    size_t want = (size_t)atoi(getenv("SWEEP_PERSIST_MB")) << 20, got = 0;
    cudaError_t e = cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, want);
    cudaDeviceGetLimit(&got, cudaLimitPersistingL2CacheSize);
    printf("cudaLimitPersistingL2CacheSize: asked %zu MB -> %s, now %zu MB\n", want >> 20, cudaGetErrorString(e), got >> 20);
  }

  std::mt19937_64 rng(12345);
  std::poisson_distribution<int> pd(deg);
  std::vector<int64_t> rowptr(N + 1, 0);
  for (int64_t i = 0; i < N; ++i) rowptr[i + 1] = rowptr[i] + pd(rng);
  const int64_t nnz = rowptr[N];
  std::vector<int32_t> col(nnz);
  std::vector<float> val(nnz);
  std::uniform_int_distribution<int32_t> ud(0, (int32_t)N - 1);
  for (int64_t i = 0; i < N; ++i) {
    for (int64_t j = rowptr[i]; j < rowptr[i + 1]; ++j) col[j] = ud(rng);
    std::sort(col.begin() + rowptr[i], col.begin() + rowptr[i + 1]);
  }
  for (int64_t j = 0; j < nnz; ++j) val[j] = 1.0f / deg;
  std::vector<float> x((size_t)N * C);
  for (auto& v : x) v = (float)((rng() >> 40) * (1.0 / (1 << 24))) - 0.5f;

  Problem P;
  P.N = N; P.C = C; P.nnz = nnz; P.sm_count = prop.multiProcessorCount;
  CK(cudaMalloc(&P.rowptr, (N + 1) * 8)); CK(cudaMalloc(&P.rowptr32, (N + 1) * 4)); CK(cudaMalloc(&P.col, nnz * 4)); CK(cudaMalloc(&P.val, nnz * 4));
  CK(cudaMalloc(&P.src, (size_t)N * C * 4)); CK(cudaMalloc(&P.dst, (size_t)N * C * 4)); CK(cudaMalloc(&P.ref, (size_t)N * C * 4));
  CK(cudaMemcpy(P.rowptr, rowptr.data(), (N + 1) * 8, cudaMemcpyHostToDevice));
  { std::vector<int32_t> r32(rowptr.begin(), rowptr.end()); CK(cudaMemcpy(P.rowptr32, r32.data(), (N + 1) * 4, cudaMemcpyHostToDevice)); }
  CK(cudaMemcpy(P.col, col.data(), nnz * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(P.val, val.data(), nnz * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(P.src, x.data(), (size_t)N * C * 4, cudaMemcpyHostToDevice));
  P.bytes = (double)nnz * 8 + (double)(N + 1) * 8 + (double)nnz * C * 4 + (double)N * C * 4;
  printf("nnz=%lld  algorithmic bytes/hop %.3f GB  (at %.0f GB/s: %.3f ms)\n", (long long)nnz, P.bytes / 1e9, peak,
         P.bytes / peak / 1e6);

  // copy-bandwidth sanity line (same definition as MEASURED_PEAKS.json: read + write bytes)
  {
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    const size_t nb = (size_t)N * C * 4;
    CK(cudaMemcpy(P.dst, P.src, nb, cudaMemcpyDeviceToDevice));
    CK(cudaEventRecord(e0));
    for (int i = 0; i < 10; ++i) CK(cudaMemcpyAsync(P.dst, P.src, nb, cudaMemcpyDeviceToDevice));
    CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
    printf("cudaMemcpy D2D %zu MB: %.0f GB/s (read+write)\n", nb >> 20, 2.0 * nb * 10 / (ms * 1e-3) / 1e9);
  }

  // Each variant is run in 3 separate rounds (interleaved with the others) to expose run-to-run noise.
  struct V { const char* name; std::function<double(bool)> fn; double ms[3]; };
  std::vector<V> vs;
#define ADD(NAME, ...) vs.push_back(V{NAME, [&](bool ref) { return run<__VA_ARGS__>(P, NAME, reps, peak, 0, ref, 1.0f); }, {0, 0, 0}})
  //                                   L   U  THR MINB HINT PF SH
#define ADDW(NAME, FRAC, ...) vs.push_back(V{NAME, [&](bool) { return run_v2w<__VA_ARGS__>(P, NAME, reps, peak, FRAC); }, {0, 0, 0}})
#define ADDMR(NAME, ...) vs.push_back(V{NAME, [&](bool) { return run_mr<__VA_ARGS__>(P, NAME, reps, peak); }, {0, 0, 0}})
  //                                  L  GS  U MINB HINT
#define ADDMRW(NAME, ...) vs.push_back(V{NAME, [&](bool) { return run_mr_w<__VA_ARGS__>(P, NAME, reps, peak); }, {0, 0, 0}})
  if (C <= 16 && getenv("SWEEP_R2")) {   // narrow rows with 32-byte lanes (feature-sharded slices at 4 / 8 GPUs)
    if (C <= 8) {
      ADD("1row  L2 U2 EL mb6 (ref)",     2, 2, 256, 6, 3, false);
      ADDMR("r1 mrow L2 GS8  U2 EL mb6",  2, 8, 2, 6, 3);
      ADDMRW("w mrow L1 GS8  U1 mb6",     1, 8, 1, 6, 3);
      ADDMRW("w mrow L1 GS8  U1 mb8",     1, 8, 1, 8, 3);
      ADDMRW("w mrow L1 GS4  U1 mb8",     1, 4, 1, 8, 3);
      ADDMRW("w mrow L1 GS16 U1 mb6",     1, 16, 1, 6, 3);
      ADDMRW("w mrow L1 GS32 U1 mb8",     1, 32, 1, 8, 3);
      ADDMRW("w mrow L1 GS8  U1 mb8 noEL", 1, 8, 1, 8, 1);
      ADDMRW("v2-16B mrow L2 GS8 U2 mb6",  2, 8, 2, 6, 3, 4);
      ADDMRW("w mrow L1 GS8  U1 mb5",     1, 8, 1, 5, 3);
      ADDMRW("w mrow L1 GS8  U1 mb4",     1, 8, 1, 4, 3);
      ADDMRW("w mrow L1 GS16 U1 mb4",     1, 16, 1, 4, 3);
    } else {
      ADD("1row  L4 U2 EL mb6 (ref)",     4, 2, 256, 6, 3, false);
      ADDMR("r1 mrow L4 GS16 U2 EL mb8",  4, 16, 2, 8, 3);
      ADDMRW("w mrow L2 GS16 U2 mb6",     2, 16, 2, 6, 3);
      ADDMRW("w mrow L2 GS16 U1 mb8",     2, 16, 1, 8, 3);
      ADDMRW("w mrow L2 GS8  U1 mb8",     2, 8, 1, 8, 3);
      ADDMRW("w mrow L2 GS32 U2 mb6",     2, 32, 2, 6, 3);
      ADDMRW("w mrow L2 GS16 U2 mb6 noEL", 2, 16, 2, 6, 1);
      ADDMRW("v2-16B mrow L4 GS16 U2 mb8", 4, 16, 2, 8, 3, 4);
      ADDMRW("w mrow L2 GS16 U2 mb4",     2, 16, 2, 4, 3);
      ADDMRW("w mrow L2 GS16 U1 mb5",     2, 16, 1, 5, 3);
      ADDMRW("w mrow L2 GS8  U2 mb4",     2, 8, 2, 4, 3);
      ADDMRW("w mrow L2 GS8  U2 mb3",     2, 8, 2, 3, 3);
      ADDMRW("w mrow L2 GS8  U2 mb5",     2, 8, 2, 5, 3);
    }
  } else if (C <= 8) {           // feature-sharded multi-GPU slices: 32-byte rows
    ADD("1row  L2 U2 EL mb6",          2, 2, 256, 6, 3, false);
    ADDMR("mrow L2 GS4  U2 EL mb6",    2, 4, 2, 6, 3);
    ADDMR("mrow L2 GS8  U2 EL mb6",    2, 8, 2, 6, 3);
    ADDMR("mrow L2 GS8  U1 EL mb6",    2, 8, 1, 6, 3);
    ADDMR("mrow L2 GS16 U2 EL mb6",    2, 16, 2, 6, 3);
    ADDMR("mrow L2 GS8  U2 ldg mb6",   2, 8, 2, 6, 0);
    ADDMR("mrow L2 GS8  U2 EL mb8",    2, 8, 2, 8, 3);
    ADDMR("mrow L2 GS8  U2 EL mb4",    2, 8, 2, 4, 3);
  } else if (C <= 16) {
    ADD("1row  L4 U2 EL mb6",          4, 2, 256, 6, 3, false);
    ADDMR("mrow L4 GS8  U2 EL mb6",    4, 8, 2, 6, 3);
    ADDMR("mrow L4 GS16 U2 EL mb6",    4, 16, 2, 6, 3);
    ADDMR("mrow L4 GS16 U4 EL mb6",    4, 16, 4, 6, 3);
    ADDMR("mrow L4 GS16 U2 ldg mb6",   4, 16, 2, 6, 0);
    ADDMR("mrow L4 GS16 U2 EL mb8",    4, 16, 2, 8, 3);
  } else if (C <= 32) {
    ADD("1row  L8 U2 EL mb8",          8, 2, 256, 8, 3, false);
    ADD("1row  L8 U4 EL mb6",          8, 4, 256, 6, 3, false);
    ADDMR("mrow L8 GS16 U2 EL mb6",    8, 16, 2, 6, 3);
    ADDMR("mrow L8 GS16 U2 EL mb8",    8, 16, 2, 8, 3);
    ADDMR("mrow L8 GS32 U4 EL mb6",    8, 32, 4, 6, 3);
    ADDMR("mrow L8 GS16 U2 ldg mb6",   8, 16, 2, 6, 0);
  } else if (C <= 64 && getenv("SWEEP_R2") && atoi(getenv("SWEEP_R2")) == 4) {
    // column-split passes with the wide-lane kernel: the gathered slab per pass shrinks towards the L2 (2 x 32 columns:
    // 128 MB, 4 x 16 columns: 64 MB at N = 1M) at the price of re-reading col/val once per pass
    ADD("r1 shipped (EL noPF mb6)",    16, 4, 256, 6, 3, false);
    ADDW("w 1pass L8 U4 mb4 EL",   1.0f,  8, 4, 256, 4, 3);
    ADDW("w 2pass L4 U4 mb4 EL",   1.0f,  4, 4, 256, 4, 3);
    ADDW("w 2pass L4 U2 mb6 EL",   1.0f,  4, 2, 256, 6, 3);
    ADDW("w 2pass L4 U2 mb8 EL",   1.0f,  4, 2, 256, 8, 3);
    ADDW("w 2pass L4 U4 mb4 noEL", 1.0f,  4, 4, 256, 4, 1);
    ADDW("w 2pass L4 U1 mb8 EL",   1.0f,  4, 1, 256, 8, 3);
    ADDW("w 4pass L2 U2 mb6 EL",   1.0f,  2, 2, 256, 6, 3);
    ADDW("w 4pass L2 U1 mb8 EL",   1.0f,  2, 1, 256, 8, 3);
    ADDW("w 4pass L2 U2 mb8 noEL", 1.0f,  2, 2, 256, 8, 1);
  } else if (C <= 64 && getenv("SWEEP_R2") && atoi(getenv("SWEEP_R2")) == 3) {
    ADD("r1 shipped (EL noPF mb6)",    16, 4, 256, 6, 3, false);
    ADDW("w U4 mb4 EL all",        1.0f,  8, 4, 256, 4, 3);
    ADDW("w U4 mb4 noEL",          1.0f,  8, 4, 256, 4, 1);
    ADDW("w U4 mb4 ELf .15",       0.15f, 8, 4, 256, 4, 2);
    ADDW("w U4 mb4 ELf .25",       0.25f, 8, 4, 256, 4, 2);
    ADDW("w U4 mb4 ELf .35",       0.35f, 8, 4, 256, 4, 2);
    ADDW("w U4 mb4 ELf .45",       0.45f, 8, 4, 256, 4, 2);
    ADDW("w U4 mb4 ELf/EF .15",    0.15f, 8, 4, 256, 4, 6);
    ADDW("w U4 mb4 ELf/EF .25",    0.25f, 8, 4, 256, 4, 6);
    ADDW("w U4 mb4 ELf/EF .35",    0.35f, 8, 4, 256, 4, 6);
    ADDW("w U4 mb4 ELf/EF .45",    0.45f, 8, 4, 256, 4, 6);
    ADDW("w U4 mb4 ELf .25 st.cs", 0.25f, 8, 4, 256, 4, 2, 1);
    ADDW("w U4 mb4 ELf .35 st.cs", 0.35f, 8, 4, 256, 4, 2, 1);
  } else if (C <= 64 && getenv("SWEEP_R2") && atoi(getenv("SWEEP_R2")) == 2) {
    ADD("r1 shipped (EL noPF mb6)",    16, 4, 256, 6, 3, false);
    //                                 L  U  THR MINB HINT SH
    ADDW("w U4 mb4 EL all",        1.0f,  8, 4, 256, 4, 3);
    ADDW("w U1 mb8 EL all",        1.0f,  8, 1, 256, 8, 3);
    ADDW("w U2 mb8 EL all",        1.0f,  8, 2, 256, 8, 3);
    ADDW("w U4 mb4 EL all st.cs",  1.0f,  8, 4, 256, 4, 3, 1);
    ADDW("w U4 mb4 noEL",          1.0f,  8, 4, 256, 4, 1);
    ADDW("w U4 mb4 ELf .25",       0.25f, 8, 4, 256, 4, 2);
    ADDW("w U4 mb4 ELf .35",       0.35f, 8, 4, 256, 4, 2);
    ADDW("w U4 mb4 ELf .45",       0.45f, 8, 4, 256, 4, 2);
    ADDW("w U4 mb4 ELf .60",       0.60f, 8, 4, 256, 4, 2);
    ADDW("w U4 mb4 ELf/EF .25",    0.25f, 8, 4, 256, 4, 6);
    ADDW("w U4 mb4 ELf/EF .35",    0.35f, 8, 4, 256, 4, 6);
    ADDW("w U4 mb4 ELf/EF .45",    0.45f, 8, 4, 256, 4, 6);
    ADDW("w U4 mb4 ELf/EF .60",    0.60f, 8, 4, 256, 4, 6);
    ADDW("w U4 mb4 ELf/EF .35 cs", 0.35f, 8, 4, 256, 4, 6, 1);
    ADDW("w U1 mb8 ELf/EF .35",    0.35f, 8, 1, 256, 8, 6);
    ADDW("w U4 t128 mb8 EL all",   1.0f,  8, 4, 128, 8, 3);
    ADDW("w U2 t128 mb12 EL all",  1.0f,  8, 2, 128, 12, 3);
    ADDW("w U8 mb2 EL all",        1.0f,  8, 8, 256, 2, 3);
    ADDW("w U6 mb3 EL all",        1.0f,  8, 6, 256, 3, 3);
  } else if (C <= 64 && getenv("SWEEP_R2")) {
#define ADDV2(NAME, ...) vs.push_back(V{NAME, [&](bool) { return run_v2<__VA_ARGS__>(P, NAME, reps, peak); }, {0, 0, 0}})
#define ADDAS(NAME, ...) vs.push_back(V{NAME, [&](bool) { return run_async<__VA_ARGS__>(P, NAME, reps, peak); }, {0, 0, 0}})
    ADD("r1 shipped (EL noPF mb6)",    16, 4, 256, 6, 3, false);
    //                                  L  U  THR MINB HINT I32
    ADDV2("v2 i64 U4 mb6",             16, 4, 256, 6, 3, false);
    ADDV2("v2 i32 U4 mb6",             16, 4, 256, 6, 3, true);
    ADDV2("v2 i32 U4 mb5",             16, 4, 256, 5, 3, true);
    ADDV2("v2 i32 U4 mb7",             16, 4, 256, 7, 3, true);
    ADDV2("v2 i32 U2 mb8",             16, 2, 256, 8, 3, true);
    ADDV2("v2 i32 U6 mb5",             16, 6, 256, 5, 3, true);
    ADDV2("v2 i32 U8 mb4",             16, 8, 256, 4, 3, true);
    ADDV2("v2 i32 U4 mb6 noEL",        16, 4, 256, 6, 1, true);
#define ADDV2W(NAME, ...) vs.push_back(V{NAME, [&](bool) { return run_v2w<__VA_ARGS__>(P, NAME, reps, peak); }, {0, 0, 0}})
    ADDV2W("v2 ldg256 L8 U2 mb6",       8, 2, 256, 6, 3);
    ADDV2W("v2 ldg256 L8 U2 mb8",       8, 2, 256, 8, 3);
    ADDV2W("v2 ldg256 L8 U3 mb5",       8, 3, 256, 5, 3);
    ADDV2W("v2 ldg256 L8 U4 mb4",       8, 4, 256, 4, 3);
    ADDV2W("v2 ldg256 L8 U1 mb8",       8, 1, 256, 8, 3);
    //                                  L SLOTS THR MINB HINT
    ADDAS("async S32 t128 mb3 EL",     16, 32, 128, 3, 3);
    ADDAS("async S32 t256 mb1 EL",     16, 32, 256, 1, 3);
    ADDAS("async S32 t128 mb3 noEL",   16, 32, 128, 3, 1);
    ADDAS("async S64 t128 mb1 EL",     16, 64, 128, 1, 3);
    ADDAS("async S64 t96  mb2 EL",     16, 64, 96, 2, 3);
    ADDAS("async S32 t64  mb6 EL",     16, 32, 64, 6, 3);
    ADDAS("async S32 t128 mb2 EL",     16, 32, 128, 2, 3);
  } else if (C <= 64) {
    ADD("noalloc PF   mb6",            16, 4, 256, 6, 1, true);
    ADDMR("mrow L16 GS32 U2 EL mb6",   16, 32, 2, 6, 3);
    ADD("noalloc noPF mb6",            16, 4, 256, 6, 1, false);
    ADD("ldg     noPF mb6",            16, 4, 256, 6, 0, false);
    ADD("ELimm1  PF   mb1(64r)",       16, 4, 256, 1, 3, true);
    ADD("ELimm1  PF   mb6",            16, 4, 256, 6, 3, true);
    ADD("ELimm1  noPF mb6",            16, 4, 256, 6, 3, false);
    ADD("ELimm1  noPF mb5",            16, 4, 256, 5, 3, false);
    ADD("ELimm1  noPF mb4",            16, 4, 256, 4, 3, false);
    ADD("ELreg1  noPF mb6",            16, 4, 256, 6, 2, false);
    ADD("ELimm.5 noPF mb6",            16, 4, 256, 6, 4, false);
    ADD("EL.5/EF noPF mb6",            16, 4, 256, 6, 5, false);
    ADD("ELimm1  noPF mb6 st.cs",      16, 4, 256, 6, 3, false, 1);
    ADD("ELimm1  noPF mb8 U2",         16, 2, 256, 8, 3, false);
    ADD("ELimm1  noPF t128 mb12",      16, 4, 128, 12, 3, false);
    ADD("ELimm1  noPF t512 mb3",       16, 4, 512, 3, 3, false);
  } else {
    ADD("noalloc PF   mb6",            32, 4, 256, 6, 1, true);
    ADD("noalloc noPF mb6",            32, 4, 256, 6, 1, false);
    ADD("ELimm1  PF   mb4",            32, 4, 256, 4, 3, true);
    ADD("ELimm1  noPF mb4",            32, 4, 256, 4, 3, false);
    ADD("ELimm1  noPF mb6",            32, 4, 256, 6, 3, false);
    ADD("ELreg1  noPF mb6",            32, 4, 256, 6, 2, false);
    ADD("ELimm1  noPF mb6 st.cs",      32, 4, 256, 6, 3, false, 1);
  }
  for (int round = 0; round < 3; ++round)
    for (size_t i = 0; i < vs.size(); ++i) vs[i].ms[round] = vs[i].fn(round == 0 && i == 0);
  printf("\nsummary (avg ms per round, algorithmic GB/s of the median round, frac of %.0f GB/s)\n", peak);
  for (auto& v : vs) {
    double m[3] = {v.ms[0], v.ms[1], v.ms[2]};
    std::sort(m, m + 3);
    printf("%-28s %.3f %.3f %.3f   median %.3f ms  %.0f GB/s  frac %.3f\n", v.name, v.ms[0], v.ms[1], v.ms[2], m[1],
           P.bytes / (m[1] * 1e-3) / 1e9, P.bytes / (m[1] * 1e-3) / 1e9 / peak);
  }
  return 0;
}
