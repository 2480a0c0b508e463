// Plan = device-resident CSR gather operators for the GSO.  Replaces GraphFilter.addGSO's dense E x N x N
// tensor (reference alegnn/utils/graphML.py:2116-2123).
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>

#include "common.cuh"

using namespace b200gf;

namespace b200gf {
std::atomic<long long> g_launch_count{0};
}

namespace {

struct HostCsr {
  std::vector<int64_t> rowptr;
  std::vector<int32_t> col;
  std::vector<unsigned char> val;  // nnz * elem bytes
};

// copy (host or device) -> host vector; cudaMemcpyDefault resolves the direction through UVA
template <typename V>
int fetch(std::vector<V>& dst, const void* src, size_t count) {
  try {
    dst.resize(count);
  } catch (const std::bad_alloc&) {
    return B200GF_ENOMEM;
  }
  if (count == 0) return B200GF_OK;
  CUDA_TRY(cudaMemcpy(dst.data(), src, count * sizeof(V), cudaMemcpyDefault));
  return B200GF_OK;
}

int validate_csr(const HostCsr& A, int64_t n_rows, int64_t n_cols) {
  if (A.rowptr[0] != 0) return B200GF_EINVAL;
  for (int64_t i = 0; i < n_rows; ++i)
    if (A.rowptr[i + 1] < A.rowptr[i]) return B200GF_EINVAL;
  const int64_t nnz = A.rowptr[n_rows];
  for (int64_t j = 0; j < nnz; ++j)
    if (A.col[j] < 0 || (int64_t)A.col[j] >= n_cols) return B200GF_EINVAL;
  return B200GF_OK;
}

// counting-sort transpose of a square CSR (deterministic: entries of each output row keep ascending source-row order)
int transpose_host(const HostCsr& A, int64_t N, size_t es, HostCsr& At) {
  const int64_t nnz = A.rowptr[N];
  try {
    At.rowptr.assign(N + 1, 0);
    At.col.resize(nnz);
    At.val.resize((size_t)nnz * es);
  } catch (const std::bad_alloc&) {
    return B200GF_ENOMEM;
  }
  for (int64_t j = 0; j < nnz; ++j) At.rowptr[A.col[j] + 1]++;
  for (int64_t i = 0; i < N; ++i) At.rowptr[i + 1] += At.rowptr[i];
  std::vector<int64_t> cursor(At.rowptr.begin(), At.rowptr.end() - 1);
  for (int64_t i = 0; i < N; ++i) {
    for (int64_t j = A.rowptr[i]; j < A.rowptr[i + 1]; ++j) {
      const int64_t dst = cursor[A.col[j]]++;
      At.col[dst] = (int32_t)i;
      std::memcpy(&At.val[(size_t)dst * es], &A.val[(size_t)j * es], es);
    }
  }
  return B200GF_OK;
}

int upload(const HostCsr& A, int64_t n_rows, size_t es, CsrDev& D) {
  const int64_t nnz = A.rowptr[n_rows];
  D.nnz = nnz;
  D.owned = true;
  if (cudaMalloc(&D.rowptr, (size_t)(n_rows + 1) * sizeof(int64_t)) != cudaSuccess) return B200GF_ENOMEM;
  // +1 element so empty operators still get valid pointers
  if (cudaMalloc(&D.col, (size_t)(nnz + 1) * sizeof(int32_t)) != cudaSuccess) return B200GF_ENOMEM;
  if (cudaMalloc(&D.val, (size_t)(nnz + 1) * es) != cudaSuccess) return B200GF_ENOMEM;
  CUDA_TRY(cudaMemcpy(D.rowptr, A.rowptr.data(), (size_t)(n_rows + 1) * sizeof(int64_t), cudaMemcpyHostToDevice));
  if (nnz < (int64_t)INT32_MAX) {   // 32-bit copy of the offsets for the hop kernel's 32-bit index arithmetic
    std::vector<int32_t> r32;
    try {
      r32.assign(A.rowptr.begin(), A.rowptr.end());
    } catch (const std::bad_alloc&) {
      return B200GF_ENOMEM;
    }
    if (cudaMalloc(&D.rowptr32, (size_t)(n_rows + 1) * sizeof(int32_t)) != cudaSuccess) return B200GF_ENOMEM;
    CUDA_TRY(cudaMemcpy(D.rowptr32, r32.data(), (size_t)(n_rows + 1) * sizeof(int32_t), cudaMemcpyHostToDevice));
  }
  if (nnz > 0) {
    CUDA_TRY(cudaMemcpy(D.col, A.col.data(), (size_t)nnz * sizeof(int32_t), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(D.val, A.val.data(), (size_t)nnz * es, cudaMemcpyHostToDevice));
  }
  return B200GF_OK;
}

int fetch_csr(HostCsr& A, int64_t n_rows, size_t es, const int64_t* rowptr, const int32_t* col, const void* val) {
  int rc = fetch(A.rowptr, rowptr, (size_t)n_rows + 1);
  if (rc) return rc;
  const int64_t nnz = A.rowptr[n_rows];
  if (nnz < 0 || (nnz > 0 && (!col || !val))) return B200GF_EINVAL;
  if ((rc = fetch(A.col, col, (size_t)nnz))) return rc;
  if ((rc = fetch(A.val, val, (size_t)nnz * es))) return rc;
  return B200GF_OK;
}

int init_device(b200gf_plan* p, int device) {
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0 || device < 0 || device >= count) {
    (void)cudaGetLastError();
    return B200GF_ENODEVICE;
  }
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) return B200GF_ENODEVICE;  // built for sm_90a only
  CUDA_TRY(cudaSetDevice(device));
  p->device = device;
  p->sm_count = prop.multiProcessorCount;
  int l2 = 0;
  CUDA_TRY(cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, device));
  p->l2_bytes = l2;
  return B200GF_OK;
}

// restores the caller's current device when a plan_create call returns (plan_destroy does the same by hand)
struct DeviceGuard {
  int prev = -1;
  DeviceGuard() { if (cudaGetDevice(&prev) != cudaSuccess) { prev = -1; (void)cudaGetLastError(); } }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

void free_windows(CsrDev& D) {
  if (D.owned) {
    if (D.win_rowptr32) cudaFree(D.win_rowptr32);
    if (D.win_col) cudaFree(D.win_col);
    if (D.win_val) cudaFree(D.win_val);
  }
  D.win_rowptr32 = nullptr; D.win_col = nullptr; D.win_val = nullptr;
  D.win_rows = 0; D.n_win = 0;
}

void free_csr(CsrDev& D) {
  free_windows(D);
  if (!D.owned) return;
  if (D.rowptr) cudaFree(D.rowptr);
  if (D.rowptr32) cudaFree(D.rowptr32);
  if (D.col) cudaFree(D.col);
  if (D.val) cudaFree(D.val);
  D.rowptr = nullptr; D.rowptr32 = nullptr; D.col = nullptr; D.val = nullptr;
}

// Window-major copy of a square operator (CsrDev::win_*): a counting sort of the entries by (column window, row) that
// keeps each row's entry order.  O(nnz + W * N) on the host.  The new copy is built aside and replaces D's only once it
// is complete: on any error D keeps what it had, and nothing half-built or allocated is left behind.
int build_windows(const HostCsr& A, int64_t N, size_t es, int64_t R, CsrDev& D) {
  const int64_t nnz = A.rowptr[N];
  if (N == 0 || R <= 0) return B200GF_EUNSUPPORTED;
  const int64_t W = (N - 1) / R + 1;
  if (nnz >= (int64_t)INT32_MAX || W * (N + 1) >= (int64_t)INT32_MAX) return B200GF_EUNSUPPORTED;
  std::vector<int32_t> rp, col, cursor;
  std::vector<unsigned char> val;
  try {
    rp.assign((size_t)(W * (N + 1)), 0);
    col.resize((size_t)nnz);
    val.resize((size_t)nnz * es);
    cursor.resize((size_t)(W * N));
  } catch (const std::bad_alloc&) {
    return B200GF_ENOMEM;
  }
  // count into rp[w * (N + 1) + i + 1], then an exclusive scan in window-major order gives every row's start
  for (int64_t i = 0; i < N; ++i)
    for (int64_t j = A.rowptr[i]; j < A.rowptr[i + 1]; ++j) rp[(size_t)((A.col[j] / R) * (N + 1) + i + 1)]++;
  int32_t run = 0;
  for (int64_t w = 0; w < W; ++w) {
    int32_t* r = rp.data() + w * (N + 1);
    r[0] = run;
    for (int64_t i = 1; i <= N; ++i) r[i] += r[i - 1];
    run = r[N];
  }
  for (int64_t w = 0; w < W; ++w)
    for (int64_t i = 0; i < N; ++i) cursor[(size_t)(w * N + i)] = rp[(size_t)(w * (N + 1) + i)];
  for (int64_t i = 0; i < N; ++i) {
    for (int64_t j = A.rowptr[i]; j < A.rowptr[i + 1]; ++j) {
      const int32_t dst = cursor[(size_t)((A.col[j] / R) * N + i)]++;
      col[dst] = A.col[j];
      std::memcpy(&val[(size_t)dst * es], &A.val[(size_t)j * es], es);
    }
  }
  CsrDev nw;   // owned
  const auto upload_copy = [&]() -> int {
    if (cudaMalloc(&nw.win_rowptr32, rp.size() * sizeof(int32_t)) != cudaSuccess) return B200GF_ENOMEM;
    if (cudaMalloc(&nw.win_col, (size_t)(nnz + 1) * sizeof(int32_t)) != cudaSuccess) return B200GF_ENOMEM;
    if (cudaMalloc(&nw.win_val, (size_t)(nnz + 1) * es) != cudaSuccess) return B200GF_ENOMEM;
    CUDA_TRY(cudaMemcpy(nw.win_rowptr32, rp.data(), rp.size() * sizeof(int32_t), cudaMemcpyHostToDevice));
    if (nnz > 0) {
      CUDA_TRY(cudaMemcpy(nw.win_col, col.data(), (size_t)nnz * sizeof(int32_t), cudaMemcpyHostToDevice));
      CUDA_TRY(cudaMemcpy(nw.win_val, val.data(), (size_t)nnz * es, cudaMemcpyHostToDevice));
    }
    return B200GF_OK;
  };
  if (const int rc = upload_copy()) {
    free_windows(nw);
    (void)cudaGetLastError();   // a failed cudaMalloc must not surface at a later launch check
    return rc;
  }
  free_windows(D);
  D.win_rowptr32 = nw.win_rowptr32; D.win_col = nw.win_col; D.win_val = nw.win_val;
  D.win_rows = R;
  D.n_win = (int)W;
  return B200GF_OK;
}

// the window copies of a symmetric plan's backward operators alias the forward ones, as the CSR does
void share_windows(const CsrDev& from, CsrDev& to) {
  to.win_rows = from.win_rows; to.n_win = from.n_win;
  to.win_rowptr32 = from.win_rowptr32; to.win_col = from.win_col; to.win_val = from.win_val;
}

}  // namespace

extern "C" {

int b200gf_version(void) { return B200GF_VERSION; }

int64_t b200gf_launch_count(int reset) {
  return reset ? g_launch_count.exchange(0, std::memory_order_relaxed) : g_launch_count.load(std::memory_order_relaxed);
}

const char* b200gf_strerror(int rc) {
  switch (rc) {
    case B200GF_OK: return "ok";
    case B200GF_EINVAL: return "b200gf: invalid argument";
    case B200GF_EUNSUPPORTED: return "b200gf: unsupported dtype or size";
    case B200GF_ENOMEM: return "b200gf: out of memory";
    case B200GF_EWORKSPACE: return "b200gf: workspace too small";
    case B200GF_ENODEVICE: return "b200gf: no sm_90 CUDA device";
    default: break;
  }
  if (rc <= B200GF_ECUDA) {
    static thread_local std::string msg;
    msg = std::string("b200gf: CUDA error: ") + cudaGetErrorString((cudaError_t)(B200GF_ECUDA - rc));
    return msg.c_str();
  }
  return "b200gf: unknown error";
}

void b200gf_plan_destroy(b200gf_plan* plan) {
  if (!plan) return;
  int prev = -1;
  cudaGetDevice(&prev);
  cudaSetDevice(plan->device);
  for (auto& d : plan->fwd) free_csr(d);
  for (auto& d : plan->bwd) free_csr(d);
  for (auto e : plan->prof_start) cudaEventDestroy(e);
  for (auto e : plan->prof_stop) cudaEventDestroy(e);
  if (prev >= 0) cudaSetDevice(prev);
  delete plan;
}

int b200gf_plan_create(b200gf_plan** out, int device, int64_t N, int E, const int64_t* const* rowptr,
                       const int32_t* const* colidx, const void* const* vals, int dtype) {
  if (!out || N < 0 || E <= 0 || !rowptr || !colidx || !vals) return B200GF_EINVAL;
  if (dtype != B200GF_F32 && dtype != B200GF_F64) return B200GF_EUNSUPPORTED;
  if (N > (int64_t)INT32_MAX) return B200GF_EUNSUPPORTED;
  *out = nullptr;
  DeviceGuard guard;   // init_device() switches to the plan's device; the caller's current device is restored on return
  b200gf_plan* p = new (std::nothrow) b200gf_plan();
  if (!p) return B200GF_ENOMEM;
  int rc = init_device(p, device);
  if (rc) { delete p; return rc; }
  p->dtype = dtype; p->n_rows = N; p->n_cols = N; p->E = E; p->has_bwd = true;
  p->fwd.resize(E); p->bwd.resize(E);
  const size_t es = dtype_size(dtype);
  bool all_sym = true;
  for (int e = 0; e < E && rc == B200GF_OK; ++e) {
    if (!rowptr[e]) { rc = B200GF_EINVAL; break; }  // colidx / vals may be null for an edgeless S_e
    HostCsr A, At;
    if ((rc = fetch_csr(A, N, es, rowptr[e], colidx[e], vals[e]))) break;
    if ((rc = validate_csr(A, N, N))) break;
    if ((rc = transpose_host(A, N, es, At))) break;
    const bool sym = A.rowptr == At.rowptr && A.col == At.col && A.val == At.val;
    // |i - j| > N/8 holds for 77 % of the non-zeros of a graph without locality (Erdos-Renyi), and for few of a graph
    // numbered community by community
    int64_t far = 0;
    for (int64_t i = 0; i < N; ++i)
      for (int64_t j = A.rowptr[i]; j < A.rowptr[i + 1]; ++j) far += 8 * std::abs(i - (int64_t)A.col[j]) > N;
    const bool spread = 2 * far > A.rowptr[N];
    all_sym = all_sym && sym;
    if ((rc = upload(At, N, es, p->fwd[e]))) break;   // forward gathers along columns of S_e
    p->fwd[e].spread = spread;
    // the default window copy is optional: an operator too large for 32-bit window offsets, or a copy that does not
    // fit the host or the device, keeps the plain hop
    const int64_t R = hop_window_rows(N, p->l2_bytes, spread);
    const auto windows = [&](const HostCsr& M, CsrDev& D) {
      const int r = R > 0 ? build_windows(M, N, es, R, D) : B200GF_OK;
      return r == B200GF_EUNSUPPORTED || r == B200GF_ENOMEM ? B200GF_OK : r;
    };
    if ((rc = windows(At, p->fwd[e]))) break;
    if (sym) {
      p->bwd[e] = p->fwd[e];
      p->bwd[e].owned = false;
    } else {
      if ((rc = upload(A, N, es, p->bwd[e]))) break;
      if ((rc = windows(A, p->bwd[e]))) break;
    }
    p->bwd[e].spread = spread;
  }
  if (rc) { b200gf_plan_destroy(p); return rc; }
  p->symmetric = all_sym;
  p->from_gso = true;
  *out = p;
  return B200GF_OK;
}

int b200gf_plan_create_ops(b200gf_plan** out, int device, int64_t n_rows, int64_t n_cols, int E,
                           const int64_t* const* fwd_rowptr, const int32_t* const* fwd_colidx,
                           const void* const* fwd_vals, const int64_t* const* bwd_rowptr,
                           const int32_t* const* bwd_colidx, const void* const* bwd_vals, int dtype) {
  if (!out || n_rows < 0 || n_cols < 0 || E <= 0 || !fwd_rowptr || !fwd_colidx || !fwd_vals) return B200GF_EINVAL;
  if (dtype != B200GF_F32 && dtype != B200GF_F64) return B200GF_EUNSUPPORTED;
  if (n_cols > (int64_t)INT32_MAX) return B200GF_EUNSUPPORTED;
  *out = nullptr;
  DeviceGuard guard;   // init_device() switches to the plan's device; the caller's current device is restored on return
  b200gf_plan* p = new (std::nothrow) b200gf_plan();
  if (!p) return B200GF_ENOMEM;
  int rc = init_device(p, device);
  if (rc) { delete p; return rc; }
  p->dtype = dtype; p->n_rows = n_rows; p->n_cols = n_cols; p->E = E;
  p->has_bwd = bwd_rowptr && bwd_colidx && bwd_vals;
  p->fwd.resize(E);
  if (p->has_bwd) p->bwd.resize(E);
  const size_t es = dtype_size(dtype);
  for (int e = 0; e < E && rc == B200GF_OK; ++e) {
    HostCsr A;
    if (!fwd_rowptr[e]) { rc = B200GF_EINVAL; break; }
    if ((rc = fetch_csr(A, n_rows, es, fwd_rowptr[e], fwd_colidx[e], fwd_vals[e]))) break;
    if ((rc = validate_csr(A, n_rows, n_cols))) break;
    if ((rc = upload(A, n_rows, es, p->fwd[e]))) break;
    if (p->has_bwd) {
      HostCsr Bm;
      if (!bwd_rowptr[e]) { rc = B200GF_EINVAL; break; }
      if ((rc = fetch_csr(Bm, n_rows, es, bwd_rowptr[e], bwd_colidx[e], bwd_vals[e]))) break;
      if ((rc = validate_csr(Bm, n_rows, n_cols))) break;
      if ((rc = upload(Bm, n_rows, es, p->bwd[e]))) break;
    }
  }
  if (rc) { b200gf_plan_destroy(p); return rc; }
  *out = p;
  return B200GF_OK;
}

// Device-side plan build: the caller already holds both gather operators as DEVICE CSR arrays (e.g. built with a few
// sort / scan kernels for a GSO that changes every batch — LSIGF_DB's space-time operator); they are copied device to
// device into plan-owned memory, nothing travels through the host except the two 8-byte nnz counts.
namespace {
__global__ void narrow_rowptr_kernel(const int64_t* __restrict__ in, int32_t* __restrict__ out, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = (int32_t)in[i];
}

int adopt(const int64_t* rowptr, const int32_t* col, const void* val, int64_t n_rows, size_t es, CsrDev& D) {
  if (!rowptr) return B200GF_EINVAL;
  int64_t nnz = 0;
  CUDA_TRY(cudaMemcpy(&nnz, rowptr + n_rows, sizeof(int64_t), cudaMemcpyDeviceToHost));
  if (nnz < 0 || (nnz > 0 && (!col || !val))) return B200GF_EINVAL;
  D.nnz = nnz;
  D.owned = true;
  if (cudaMalloc(&D.rowptr, (size_t)(n_rows + 1) * sizeof(int64_t)) != cudaSuccess) return B200GF_ENOMEM;
  if (cudaMalloc(&D.col, (size_t)(nnz + 1) * sizeof(int32_t)) != cudaSuccess) return B200GF_ENOMEM;
  if (cudaMalloc(&D.val, (size_t)(nnz + 1) * es) != cudaSuccess) return B200GF_ENOMEM;
  CUDA_TRY(cudaMemcpy(D.rowptr, rowptr, (size_t)(n_rows + 1) * sizeof(int64_t), cudaMemcpyDeviceToDevice));
  if (nnz > 0) {
    CUDA_TRY(cudaMemcpy(D.col, col, (size_t)nnz * sizeof(int32_t), cudaMemcpyDeviceToDevice));
    CUDA_TRY(cudaMemcpy(D.val, val, (size_t)nnz * es, cudaMemcpyDeviceToDevice));
  }
  if (nnz < (int64_t)INT32_MAX) {
    if (cudaMalloc(&D.rowptr32, (size_t)(n_rows + 1) * sizeof(int32_t)) != cudaSuccess) return B200GF_ENOMEM;
    narrow_rowptr_kernel<<<(int)imin64((n_rows + 256) / 256, 132 * 8), 256>>>(D.rowptr, D.rowptr32, n_rows + 1);
    LAUNCH_CHECK();
  }
  return B200GF_OK;
}
}  // namespace

int b200gf_plan_create_device(b200gf_plan** out, int device, int64_t N, int E, const int64_t* const* fwd_rowptr,
                              const int32_t* const* fwd_colidx, const void* const* fwd_vals,
                              const int64_t* const* bwd_rowptr, const int32_t* const* bwd_colidx,
                              const void* const* bwd_vals, int dtype) {
  if (!out || N < 0 || E <= 0 || !fwd_rowptr || !fwd_colidx || !fwd_vals) return B200GF_EINVAL;
  if (dtype != B200GF_F32 && dtype != B200GF_F64) return B200GF_EUNSUPPORTED;
  if (N > (int64_t)INT32_MAX) return B200GF_EUNSUPPORTED;
  *out = nullptr;
  DeviceGuard guard;
  b200gf_plan* p = new (std::nothrow) b200gf_plan();
  if (!p) return B200GF_ENOMEM;
  int rc = init_device(p, device);
  if (rc) { delete p; return rc; }
  p->dtype = dtype; p->n_rows = N; p->n_cols = N; p->E = E;
  p->has_bwd = bwd_rowptr && bwd_colidx && bwd_vals;
  p->fwd.resize(E);
  if (p->has_bwd) p->bwd.resize(E);
  const size_t es = dtype_size(dtype);
  for (int e = 0; e < E && rc == B200GF_OK; ++e) {
    if ((rc = adopt(fwd_rowptr[e], fwd_colidx[e], fwd_vals[e], N, es, p->fwd[e]))) break;
    if (p->has_bwd && (rc = adopt(bwd_rowptr[e], bwd_colidx[e], bwd_vals[e], N, es, p->bwd[e]))) break;
  }
  if (rc == B200GF_OK && cudaDeviceSynchronize() != cudaSuccess) rc = B200GF_ECUDA - (int)cudaGetLastError();
  if (rc) { b200gf_plan_destroy(p); return rc; }
  *out = p;
  return B200GF_OK;
}

int64_t b200gf_plan_info(const b200gf_plan* plan, int what) {
  if (!plan) return B200GF_EINVAL;
  switch (what) {
    case 0: return plan->n_rows;
    case 1: return plan->n_cols;
    case 2: return plan->E;
    case 3: return plan->dtype;
    case 4: return plan->device;
    case 5: { int64_t s = 0; for (auto& d : plan->fwd) s += d.nnz; return s; }
    case 6: return plan->symmetric ? 1 : 0;
    case 7: return plan->l2_bytes;
    case 8: return plan->fwd.empty() ? 0 : plan->fwd[0].win_rows;
    default: return B200GF_EINVAL;
  }
}

int b200gf_plan_set_hop_windows(b200gf_plan* plan, int64_t rows) {
  if (!plan || rows < 0) return B200GF_EINVAL;
  if (!plan->from_gso) return B200GF_EUNSUPPORTED;
  DeviceGuard guard;
  CUDA_TRY(cudaSetDevice(plan->device));
  CUDA_TRY(cudaDeviceSynchronize());   // no hop in flight reads the copies about to be replaced
  const int64_t N = plan->n_rows;
  const size_t es = dtype_size(plan->dtype);
  if (rows > 0) {   // sizes no copy can take: the plan stays as it is
    if (N == 0 || ((N - 1) / rows + 1) * (N + 1) >= (int64_t)INT32_MAX) return B200GF_EUNSUPPORTED;
    for (int e = 0; e < plan->E; ++e)
      if (plan->fwd[e].nnz >= (int64_t)INT32_MAX || plan->bwd[e].nnz >= (int64_t)INT32_MAX) return B200GF_EUNSUPPORTED;
  }
  // the backward operators of a symmetric plan alias the forward ones and their copies: they are re-pointed after the
  // forward ones change, so that no operator keeps pointers into a freed copy
  const auto share_all = [&]() {
    for (int e = 0; e < plan->E; ++e)
      if (!plan->bwd[e].owned) share_windows(plan->fwd[e], plan->bwd[e]);
  };
  for (int e = 0; e < plan->E; ++e) {
    for (int dir = 0; dir < 2; ++dir) {
      CsrDev& D = dir == 0 ? plan->fwd[e] : plan->bwd[e];
      if (!D.owned) continue;
      if (rows == 0) { free_windows(D); continue; }
      HostCsr M;
      int rc = fetch_csr(M, N, es, D.rowptr, D.col, D.val);
      if (rc == B200GF_OK) rc = build_windows(M, N, es, rows, D);
      if (rc) {   // a failed rebuild leaves no copy anywhere: every hop of the plan takes the plain path
        for (int f = 0; f < plan->E; ++f) {
          free_windows(plan->fwd[f]);
          free_windows(plan->bwd[f]);
        }
        share_all();
        return rc;
      }
      share_all();
    }
  }
  share_all();
  return B200GF_OK;
}

int b200gf_plan_set_l2_bytes(b200gf_plan* plan, int64_t bytes) {
  if (!plan || bytes < 0) return B200GF_EINVAL;
  plan->l2_bytes = bytes;
  return B200GF_OK;
}

}  // extern "C"
