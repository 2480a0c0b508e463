// LSIGF forward / backward orchestration behind the C ABI (reference alegnn/utils/graphML.py:83-176 and its
// autograd).  No allocation, no host synchronisation: everything is enqueued on the caller's stream and
// all scratch lives in the caller-provided workspace, so a call is CUDA-graph capturable.
//
// Forward   z_{e,0} = x ; z_{e,k} = z_{e,k-1} · S_e   (K-1 hops per edge feature, spmm.cu)
//           y = sum_{e,k} z_{e,k} · h[:,e,k,:]^T + b   (tap contraction; wgmma 3xTF32 when eligible, FMA otherwise)
// Backward  V_{e,0} = dy ; V_{e,k} = V_{e,k-1} · S_e^T (K-1 hops with the other operator)
//           dx = sum_{e,k} V_{e,k} · h[:,e,k,:]        dh[f,e,k,g] = sum_{b,n} V_{e,k}[b,f,n] x[b,g,n]
//           db = sum dy.   Only x is needed from the forward: no z_{e,k} is saved.
#include "common.cuh"

using namespace b200gf;

namespace {

struct FwdWs {
  void* xn = nullptr;   // node-major copy of x (only when x arrives feature-major)
  void* z = nullptr;    // E*(K-1) hop outputs, each [n_cols, ldc]
  void* W = nullptr;    // packed taps [T, G, F]
  void* yn = nullptr;   // node-major y (only when y must be returned feature-major)
  size_t bytes = 0;
};

FwdWs carve_fwd(const b200gf_plan* p, void* ws, int B, int G, int F, int K, int x_layout, int y_layout) {
  const size_t es = dtype_size(p->dtype);
  const int64_t ldc = padded_ld((int64_t)B * G, p->dtype), ldf = padded_ld((int64_t)B * F, p->dtype);
  const int T = 1 + p->E * (K - 1);
  Carver c(ws);
  FwdWs w;
  if (x_layout == B200GF_FEATURE_MAJOR) w.xn = c.take((size_t)p->n_cols * ldc * es);
  w.z = c.take((size_t)p->E * (K - 1) * p->n_cols * ldc * es);
  w.W = c.take((size_t)2 * T * G * F * es);  // x2: hi / lo operand copies of the tensor-core path
  if (y_layout == B200GF_FEATURE_MAJOR) w.yn = c.take((size_t)p->n_rows * ldf * es);
  w.bytes = c.off;
  return w;
}

struct BwdWs {
  void* dyn = nullptr;  // node-major dy
  void* xn = nullptr;   // node-major x
  void* v = nullptr;    // E*(K-1) hop outputs [n_cols, ldf]
  void* W = nullptr;    // packed taps [T, F, G]
  void* dxn = nullptr;  // node-major dx
  void* tg = nullptr;   // tap-grad partials
  void* bg = nullptr;   // bias-grad partials
  size_t tg_bytes = 0, bg_bytes = 0;
  size_t bytes = 0;
};

BwdWs carve_bwd(const b200gf_plan* p, void* ws, int B, int G, int F, int K, int in_layout) {
  const size_t es = dtype_size(p->dtype);
  const int64_t ldc = padded_ld((int64_t)B * G, p->dtype), ldf = padded_ld((int64_t)B * F, p->dtype);
  const int T = 1 + p->E * (K - 1);
  Carver c(ws);
  BwdWs w;
  // sized for the worst case of the layout flags (both dy and x feature-major, dx feature-major)
  if (in_layout == B200GF_FEATURE_MAJOR) {
    w.dyn = c.take((size_t)p->n_cols * ldf * es);
    w.xn = c.take((size_t)p->n_cols * ldc * es);
    w.dxn = c.take((size_t)p->n_rows * ldc * es);
  }
  w.v = c.take((size_t)p->E * (K - 1) * p->n_cols * ldf * es);
  w.W = c.take((size_t)2 * T * G * F * es);
  w.tg_bytes = tap_grad_scratch_bytes(p->dtype, p->n_rows, B, G, F, T);
  w.tg = c.take(w.tg_bytes);
  w.bg_bytes = bias_grad_scratch_bytes(p->dtype, p->n_rows, B, F);
  w.bg = c.take(w.bg_bytes);
  w.bytes = c.off;
  return w;
}

bool bad_layout(int l) { return l != B200GF_FEATURE_MAJOR && l != B200GF_NODE_MAJOR; }

}  // namespace

namespace b200gf {
int plan_hop(const b200gf_plan* p, const CsrDev& A, const void* src, int64_t src_ld, void* dst, int64_t dst_ld, int C,
             cudaStream_t st, const ScatterHost* sh, const BcastHost* bh) {
  const bool prof = p->prof_used < (int)p->prof_start.size();
  if (prof) CUDA_TRY(cudaEventRecord(p->prof_start[p->prof_used], st));
  // partitioned plans (one node shard per GPU) keep the chunk width of their row width
  const int64_t l2 = p->n_rows == p->n_cols ? p->l2_bytes : 0;
  const int rc = launch_hop(p->dtype, p->sm_count, l2, A, p->n_rows, src, src_ld, dst, dst_ld, C, st, sh, bh);
  if (prof) {
    CUDA_TRY(cudaEventRecord(p->prof_stop[p->prof_used], st));
    p->prof_used++;
  }
  return rc;
}

int hop_chain(const b200gf_plan* p, const std::vector<CsrDev>& ops, const void* src, int64_t src_ld, void* buf, int64_t ld,
              int C, int K, std::vector<const void*>& zs, std::vector<int64_t>& zld, cudaStream_t st) {
  const size_t slot = (size_t)p->n_rows * ld * dtype_size(p->dtype);
  zs.assign(1 + p->E * (K - 1), nullptr);
  zld.assign(1 + p->E * (K - 1), ld);
  zs[0] = src;
  zld[0] = src_ld;
  for (int e = 0; e < p->E; ++e) {
    const void* prev = src;
    int64_t prev_ld = src_ld;
    for (int k = 1; k < K; ++k) {
      const int t = 1 + e * (K - 1) + (k - 1);
      void* dst = (char*)buf + (t - 1) * slot;
      if (int rc = plan_hop(p, ops[e], prev, prev_ld, dst, ld, C, st)) return rc;
      zs[t] = dst;
      prev = dst;
      prev_ld = ld;
    }
  }
  return B200GF_OK;
}
}  // namespace b200gf

extern "C" {

int b200gf_profile_hops(b200gf_plan* plan, int capacity) {
  if (!plan || capacity < 0) return B200GF_EINVAL;
  for (auto e : plan->prof_start) cudaEventDestroy(e);
  for (auto e : plan->prof_stop) cudaEventDestroy(e);
  plan->prof_start.clear();
  plan->prof_stop.clear();
  plan->prof_used = 0;
  for (int i = 0; i < capacity; ++i) {
    cudaEvent_t a, b;
    CUDA_TRY(cudaEventCreate(&a));
    CUDA_TRY(cudaEventCreate(&b));
    plan->prof_start.push_back(a);
    plan->prof_stop.push_back(b);
  }
  return B200GF_OK;
}

int b200gf_profile_read(b200gf_plan* plan, float* ms, int n) {
  if (!plan || (!ms && n > 0) || n < 0) return B200GF_EINVAL;
  const int used = plan->prof_used < n ? plan->prof_used : n;
  for (int i = 0; i < used; ++i) {
    CUDA_TRY(cudaEventSynchronize(plan->prof_stop[i]));
    CUDA_TRY(cudaEventElapsedTime(&ms[i], plan->prof_start[i], plan->prof_stop[i]));
  }
  plan->prof_used = 0;
  return used;
}

size_t b200gf_workspace_bytes(const b200gf_plan* plan, int B, int G, int F, int K, int in_layout, int backward) {
  if (!plan || B <= 0 || G <= 0 || F <= 0 || K <= 0) return 0;
  if (backward) return carve_bwd(plan, nullptr, B, G, F, K, in_layout).bytes + 256;
  return carve_fwd(plan, nullptr, B, G, F, K, in_layout, in_layout).bytes + 256;
}

static int forward_impl(const b200gf_plan* plan, const void* x, int x_layout, int64_t x_ld, const void* h,
                        const void* bias, int bias_per_node, void* y, int y_layout, int64_t y_ld, void* workspace,
                        size_t workspace_bytes, int B, int G, int F, int K, int act, void* stream) {
  if (act != B200GF_ACT_NONE && act != B200GF_ACT_RELU) return B200GF_EINVAL;
  if (!plan || !x || !h || !y || B <= 0 || G <= 0 || F <= 0 || K <= 0) return B200GF_EINVAL;
  if (bad_layout(x_layout) || bad_layout(y_layout)) return B200GF_EINVAL;
  if (plan->n_rows != plan->n_cols) return B200GF_EINVAL;  // partitioned plans use the building blocks
  const int64_t N = plan->n_rows;
  const int64_t C = (int64_t)B * G, CF = (int64_t)B * F;
  if (x_layout == B200GF_NODE_MAJOR && x_ld < C) return B200GF_EINVAL;
  if (y_layout == B200GF_NODE_MAJOR && y_ld < CF) return B200GF_EINVAL;
  if (C > INT32_MAX || CF > INT32_MAX) return B200GF_EUNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  const int dt = plan->dtype;
  const int E = plan->E;
  const int T = 1 + E * (K - 1);
  if (N == 0) return B200GF_OK;

  // carve with the caller's actual layouts (never larger than what workspace_bytes() reported)
  FwdWs w = carve_fwd(plan, workspace, B, G, F, K, x_layout, y_layout);
  int rc;
  if ((rc = check_workspace(workspace, w.bytes, workspace_bytes, false))) return rc;
  const int64_t ldc = padded_ld(C, dt), ldf = padded_ld(CF, dt);

  const void* x0 = x;
  int64_t x0_ld = x_ld;
  if (x_layout == B200GF_FEATURE_MAJOR) {
    if ((rc = launch_to_node_major(dt, x, w.xn, ldc, N, (int)C, st))) return rc;
    x0 = w.xn;
    x0_ld = ldc;
  }
  std::vector<const void*> zs;
  std::vector<int64_t> zld;
  if ((rc = hop_chain(plan, plan->fwd, x0, x0_ld, w.z, ldc, (int)C, K, zs, zld, st))) return rc;
  void* yo = y_layout == B200GF_NODE_MAJOR ? y : w.yn;
  const int64_t yo_ld = y_layout == B200GF_NODE_MAJOR ? y_ld : ldf;
  if (tc_contract_eligible(dt, N, B, G, F, T, zs.data(), zld.data(), yo, yo_ld, 0)) {
    // tensor cores: wgmma 3xTF32, operands K-major: W[t][f][g]
    if ((rc = launch_pack_taps_split(h, w.W, F, E, K, G, 0, st))) return rc;
    if ((rc = launch_tc_contract(plan->sm_count, N, B, G, F, T, zs.data(), w.W, bias, bias_per_node, yo, yo_ld, st, act)))
      return rc;
  } else {
    if ((rc = launch_pack_taps(dt, h, w.W, F, E, K, G, 0, st))) return rc;
    if ((rc = launch_tap_contract(dt, N, B, G, F, T, zs.data(), zld.data(), w.W, bias, bias_per_node, yo, yo_ld, 0, st, act)))
      return rc;
  }
  if (y_layout == B200GF_FEATURE_MAJOR)
    if ((rc = launch_to_feature_major(dt, w.yn, ldf, y, N, (int)CF, st))) return rc;
  return B200GF_OK;
}

int b200gf_forward(const b200gf_plan* plan, const void* x, int x_layout, int64_t x_ld, const void* h,
                   const void* bias, int bias_per_node, void* y, int y_layout, int64_t y_ld, void* workspace,
                   size_t workspace_bytes, int B, int G, int F, int K, void* stream) {
  return forward_impl(plan, x, x_layout, x_ld, h, bias, bias_per_node, y, y_layout, y_ld, workspace, workspace_bytes, B, G,
                      F, K, B200GF_ACT_NONE, stream);
}

int b200gf_forward_act(const b200gf_plan* plan, const void* x, int x_layout, int64_t x_ld, const void* h,
                       const void* bias, int bias_per_node, void* y, int y_layout, int64_t y_ld, void* workspace,
                       size_t workspace_bytes, int B, int G, int F, int K, int activation, void* stream) {
  return forward_impl(plan, x, x_layout, x_ld, h, bias, bias_per_node, y, y_layout, y_ld, workspace, workspace_bytes, B, G,
                      F, K, activation, stream);
}

int b200gf_backward(const b200gf_plan* plan, const void* dy, int dy_layout, int64_t dy_ld, const void* x,
                    int x_layout, int64_t x_ld, const void* h, void* dx, int dx_layout, int64_t dx_ld, void* dh,
                    void* dbias, int bias_per_node, void* workspace, size_t workspace_bytes, int B, int G, int F,
                    int K, void* stream) {
  if (!plan || !dy || !x || !h || !dh || B <= 0 || G <= 0 || F <= 0 || K <= 0) return B200GF_EINVAL;
  if (bad_layout(dy_layout) || bad_layout(x_layout) || (dx && bad_layout(dx_layout))) return B200GF_EINVAL;
  if (plan->n_rows != plan->n_cols || !plan->has_bwd) return B200GF_EINVAL;
  const int64_t N = plan->n_rows;
  const int64_t C = (int64_t)B * G, CF = (int64_t)B * F;
  if (dy_layout == B200GF_NODE_MAJOR && dy_ld < CF) return B200GF_EINVAL;
  if (x_layout == B200GF_NODE_MAJOR && x_ld < C) return B200GF_EINVAL;
  if (dx && dx_layout == B200GF_NODE_MAJOR && dx_ld < C) return B200GF_EINVAL;
  if (C > INT32_MAX || CF > INT32_MAX) return B200GF_EUNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  const int dt = plan->dtype;
  const size_t es = dtype_size(dt);
  const int E = plan->E;
  const int T = 1 + E * (K - 1);
  const bool any_fm = dy_layout == B200GF_FEATURE_MAJOR || x_layout == B200GF_FEATURE_MAJOR ||
                      (dx && dx_layout == B200GF_FEATURE_MAJOR);
  BwdWs w = carve_bwd(plan, workspace, B, G, F, K, any_fm ? B200GF_FEATURE_MAJOR : B200GF_NODE_MAJOR);
  int rc;
  if ((rc = check_workspace(workspace, w.bytes, workspace_bytes, true))) return rc;
  const int64_t ldc = padded_ld(C, dt), ldf = padded_ld(CF, dt);
  if (N == 0) {
    CUDA_TRY(cudaMemsetAsync(dh, 0, (size_t)F * E * K * G * es, st));
    if (dbias && !bias_per_node) CUDA_TRY(cudaMemsetAsync(dbias, 0, (size_t)F * es, st));
    return B200GF_OK;
  }

  const void* dy0 = dy;
  int64_t dy0_ld = dy_ld;
  if (dy_layout == B200GF_FEATURE_MAJOR) {
    if ((rc = launch_to_node_major(dt, dy, w.dyn, ldf, N, (int)CF, st))) return rc;
    dy0 = w.dyn;
    dy0_ld = ldf;
  }
  const void* x0 = x;
  int64_t x0_ld = x_ld;
  if (x_layout == B200GF_FEATURE_MAJOR) {
    if ((rc = launch_to_node_major(dt, x, w.xn, ldc, N, (int)C, st))) return rc;
    x0 = w.xn;
    x0_ld = ldc;
  }

  std::vector<const void*> vs;
  std::vector<int64_t> vld;
  if ((rc = hop_chain(plan, plan->bwd, dy0, dy0_ld, w.v, ldf, (int)CF, K, vs, vld, st))) return rc;
  if (dx) {
    void* dxo = dx_layout == B200GF_NODE_MAJOR ? dx : w.dxn;
    const int64_t dxo_ld = dx_layout == B200GF_NODE_MAJOR ? dx_ld : ldc;
    if (tc_contract_eligible(dt, N, B, F, G, T, vs.data(), vld.data(), dxo, dxo_ld, 0)) {
      if ((rc = launch_pack_taps_split(h, w.W, F, E, K, G, 1, st))) return rc;  // K-major W[t][g][f]
      if ((rc = launch_tc_contract(plan->sm_count, N, B, F, G, T, vs.data(), w.W, nullptr, 0, dxo, dxo_ld, st))) return rc;
    } else {
      if ((rc = launch_pack_taps(dt, h, w.W, F, E, K, G, 1, st))) return rc;  // W[t][f][g]
      if ((rc = launch_tap_contract(dt, N, B, F, G, T, vs.data(), vld.data(), w.W, nullptr, 0, dxo, dxo_ld, 0, st)))
        return rc;
    }
    if (dx_layout == B200GF_FEATURE_MAJOR)
      if ((rc = launch_to_feature_major(dt, w.dxn, ldc, dx, N, (int)C, st))) return rc;
  }
  if ((rc = launch_tap_grad(dt, N, B, G, F, T, x0, x0_ld, vs.data(), vld.data(), dh, 1, E, K, w.tg, w.tg_bytes, st)))
    return rc;
  if (dbias)
    if ((rc = launch_bias_grad(dt, N, B, F, dy0, dy0_ld, dbias, bias_per_node, w.bg, w.bg_bytes, st))) return rc;
  return B200GF_OK;
}

}  // extern "C"
