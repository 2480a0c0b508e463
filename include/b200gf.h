/*
 * b200gf — C ABI of the H100-native LSIGF graph-filter path.
 *
 * This is the drop-in boundary for ONE path of alelab-upenn/graph-neural-networks (alegnn 0.4.0):
 *
 *     LSIGF(h, S, x, b=None)            alegnn/utils/graphML.py:83-176
 *     GraphFilter.addGSO / .forward     alegnn/utils/graphML.py:2116-2144
 *     (their autograd backward)         SURVEY.md §8 a-8
 *
 * The reference is pure Python on top of torch.matmul; it has no FFI.  The entry points below are what
 * a binding for that path would bind (the ctypes stub a maintainer would add is shown in INTEGRATION.md,
 * and shipped in graph-neural-networks_b200/_cabi.py).
 *
 * Conventions
 *   - plain C types only; every call returns int: 0 = OK, <0 = error (see b200gf_strerror). No exceptions,
 *     no printing, no abort.
 *   - all data pointers are DEVICE pointers on the plan's device unless stated otherwise; the library never
 *     allocates inside forward/backward (caller passes a workspace) and never synchronises the host, so
 *     the calls are CUDA-graph capturable.  Work is enqueued on the cudaStream_t passed in (as void*).
 *   - dtype: B200GF_F32 or B200GF_F64 (the reference's examples run in float64, examples/sourceLocGNN.py:40).
 *   - "feature-major" layout  = the reference's  [B, G, N] contiguous tensor  (graphML.py:108-109);
 *     "node-major" layout     = [N, ld] with the B*G feature columns of one node contiguous, ld >= B*G.
 *     Column index of (b, g) is b*G + g in both.
 *   - row-vector shift (graphML.py:159):  (x S)[., j] = sum_i x[., i] S[i, j].
 */
#ifndef B200GF_H_
#define B200GF_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200gf_plan b200gf_plan;

enum { B200GF_F32 = 0, B200GF_F64 = 1 };

/* layouts for x / y / dy / dx */
enum { B200GF_FEATURE_MAJOR = 0, B200GF_NODE_MAJOR = 1 };

/* hop direction */
enum { B200GF_HOP_FWD = 0 /* dst = S^T src : forward shift x·S */, B200GF_HOP_BWD = 1 /* dst = S src */ };

/* error codes */
enum {
  B200GF_OK = 0,
  B200GF_EINVAL = -1,      /* bad argument (null pointer, negative size, shape mismatch)           */
  B200GF_EUNSUPPORTED = -2,/* dtype / size not supported                                           */
  B200GF_ENOMEM = -3,      /* host or device allocation failed in plan_create                      */
  B200GF_EWORKSPACE = -4,  /* workspace smaller than b200gf_workspace_bytes()                      */
  B200GF_ENODEVICE = -5,   /* no CUDA device / wrong architecture (needs sm_90)                    */
  B200GF_ECUDA = -1000     /* -(1000 + cudaError_t)                                                */
};

const char* b200gf_strerror(int rc);
int b200gf_version(void);

/* Number of CUDA kernels this library has launched in this process (every launch site counts itself); reset != 0
 * returns the count and zeroes it.  bench.py reports it as `gpu_launches` for the timed region. */
int64_t b200gf_launch_count(int reset);

/* ------------------------------------------------------------------------------------------------
 * Plan = the device-resident sparse form of the GSO.  Replaces GraphFilter.addGSO (graphML.py:2116-2123),
 * which stores a dense E x N x N tensor.
 *
 * b200gf_plan_create: S_e given as CSR (row i lists the non-zeros S_e[i, j]); rowptr[e] has N+1 int64,
 * colidx[e] has nnz_e int32, vals[e] has nnz_e elements of `dtype`.  Arrays may live on host or device
 * (the library copies them).  The plan builds and owns both gather operators: CSR(S_e^T) for the forward
 * shift and CSR(S_e) for the backward shift.
 * ---------------------------------------------------------------------------------------------- */
int b200gf_plan_create(b200gf_plan** out, int device, int64_t N, int E,
                       const int64_t* const* rowptr, const int32_t* const* colidx,
                       const void* const* vals, int dtype);

/* Pre-partitioned variant used by the node-partitioned (multi-GPU) path: the caller supplies the gather
 * operators directly.  fwd = rows [r0, r1) of S_e^T, bwd = rows [r0, r1) of S_e (bwd_* may be NULL when
 * no backward is needed); n_rows = r1 - r0 local rows, n_cols = global N (column indices are global). */
int b200gf_plan_create_ops(b200gf_plan** out, int device, int64_t n_rows, int64_t n_cols, int E,
                           const int64_t* const* fwd_rowptr, const int32_t* const* fwd_colidx,
                           const void* const* fwd_vals,
                           const int64_t* const* bwd_rowptr, const int32_t* const* bwd_colidx,
                           const void* const* bwd_vals, int dtype);

/* Device-side variant for GSOs that change every batch (LSIGF_DB's space-time operator, graphML.py:977-1094): both
 * operators given as DEVICE CSR arrays with valid indices (fwd = rows of S_e^T, bwd = rows of S_e, square N x N, columns
 * ascending inside a row; bwd_* may be NULL); they are copied device to device, nothing but the nnz counts is read back
 * by the host and nothing is validated. */
int b200gf_plan_create_device(b200gf_plan** out, int device, int64_t N, int E,
                              const int64_t* const* fwd_rowptr, const int32_t* const* fwd_colidx,
                              const void* const* fwd_vals,
                              const int64_t* const* bwd_rowptr, const int32_t* const* bwd_colidx,
                              const void* const* bwd_vals, int dtype);

void b200gf_plan_destroy(b200gf_plan* plan);

/* introspection: what = 0 n_rows, 1 n_cols, 2 E, 3 dtype, 4 device, 5 nnz (sum over e, forward operator),
 * 6 symmetric (1 if every S_e == S_e^T bit-for-bit, so both operators share storage), 7 L2 bytes the hops size their
 * column chunks against (b200gf_plan_set_l2_bytes), 8 rows R per source window of the window-major operator copies
 * (b200gf_plan_set_hop_windows), 0 when the plan has none */
int64_t b200gf_plan_info(const b200gf_plan* plan, int what);

/* L2 size (bytes) the plan's hops size their gathered column chunks against; plan creation reads it from the device
 * (cudaDevAttrL2CacheSize).  0 turns the sizing off: every hop then uses the chunk width its row width alone selects.
 * Results differ only by the summation order of the chunk fold.  For A/B timing and tests; bytes < 0 is EINVAL. */
int b200gf_plan_set_l2_bytes(b200gf_plan* plan, int64_t bytes);

/* Window-major copies of the plan's gather operators: window w holds the entries whose source row lies in
 * [w * rows, (w + 1) * rows).  A hop with a plain epilogue over rows of at least 128 bytes then runs one launch per
 * (128-byte column chunk, window), each adding its window's partial sums into the destination, so that what the
 * gathers read at a time is an L2-sized source range.  b200gf_plan_create builds them when a 128-byte chunk of the
 * source does not fit the L2 and the gathers spread over the whole source; the plan's L2 size at 0 turns their use off.
 * The default takes at most 8 windows.  rows = 0 drops the copies, rows > 0 rebuilds them.  This is a setup call: it
 * synchronizes the device, frees and allocates, so a CUDA graph captured on the plan before it reads freed copies and
 * must be captured again.  Results differ from the plain hop only by the summation order of the window sums.
 * rows < 0 or a null plan is EINVAL; plans from b200gf_plan_create_ops / _create_device are EUNSUPPORTED, and so is a
 * window count whose offsets W * (N + 1) or operator whose nnz do not fit 32 bits (the plan is left as it was).  Any
 * other failure of a rebuild (ENOMEM, a CUDA error) leaves the plan without window copies: every hop then takes the
 * plain path. */
int b200gf_plan_set_hop_windows(b200gf_plan* plan, int64_t rows);

/* ------------------------------------------------------------------------------------------------
 * LSIGF forward  (graphML.py:83-176)
 *   y[b,f,n] = sum_e sum_k sum_g h[f,e,k,g] (x_g S_e^k)[n] + bias
 * x: layout x_layout; x_ld = row stride in elements when node-major (ignored otherwise).
 * h: [F,E,K,G] contiguous.  bias: NULL, [F] (bias_per_node = 0; the reference's F x 1) or [F,N]
 * (bias_per_node = 1).  y: layout y_layout; y_ld as for x.
 * workspace: b200gf_workspace_bytes(plan, B, G, F, K, x_layout, 0) bytes, 256-byte aligned.
 * ---------------------------------------------------------------------------------------------- */
int b200gf_forward(const b200gf_plan* plan,
                   const void* x, int x_layout, int64_t x_ld,
                   const void* h, const void* bias, int bias_per_node,
                   void* y, int y_layout, int64_t y_ld,
                   void* workspace, size_t workspace_bytes,
                   int B, int G, int F, int K, void* stream);

/* The same with the layer's activation fused into the contraction epilogue (SURVEY.md §8 f-1): the reference's
 * selection architectures apply nn.ReLU right after every GraphFilter (alegnn/modules/architectures.py:274-296).
 * activation: B200GF_ACT_NONE or B200GF_ACT_RELU (y = max(LSIGF(...), 0)); no extra pass over y. */
enum { B200GF_ACT_NONE = 0, B200GF_ACT_RELU = 1 };
int b200gf_forward_act(const b200gf_plan* plan,
                       const void* x, int x_layout, int64_t x_ld,
                       const void* h, const void* bias, int bias_per_node,
                       void* y, int y_layout, int64_t y_ld,
                       void* workspace, size_t workspace_bytes,
                       int B, int G, int F, int K, int activation, void* stream);

/* Backward of the fused ReLU from the layer OUTPUT alone: out = dy where y > 0, else 0 (node-major [n_rows, ld]). */
int b200gf_relu_backward(int dtype, const void* y, int64_t y_ld, const void* dy, int64_t dy_ld,
                         void* out, int64_t out_ld, int64_t n_rows, int C, void* stream);

/* MaxPoolLocal (alegnn/utils/graphML.py:1968-2019) on node-major data: out[i, c] = max_j x[nb[i, j], c], i < n_out,
 * nb = the layer's neighbourhood matrix [n_out, max_nb] (int32, rows padded with a member of the list, as
 * graphTools.computeNeighborhood 'matrix' pads them).  argmax (optional, int32 [n_out, C]) receives the winning node of
 * every output element; the backward zeroes dx [n_in, dx_ld] and adds dy[i, c] to dx[argmax[i, c], c]. */
int b200gf_maxpool_forward(int dtype, const void* x, int64_t x_ld, int64_t n_in, int C,
                           const int32_t* nb, int64_t n_out, int max_nb,
                           void* out, int64_t out_ld, int32_t* argmax, void* stream);
int b200gf_maxpool_backward(int dtype, const void* dy, int64_t dy_ld, const int32_t* argmax, int64_t n_out, int C,
                            void* dx, int64_t dx_ld, int64_t n_in, void* stream);

/* LSIGF backward (autograd of the above; SURVEY.md §8 a-8)
 *   V_{e,0} = dy,  V_{e,k} = V_{e,k-1} S_e^T              (K-1 hops with the backward operator)
 *   dx      = sum_{e,k,f} h[f,e,k,g] V_{e,k}[.,f,.]        (NULL to skip)
 *   dh[f,e,k,g] = sum_{b,n} V_{e,k}[b,f,n] x[b,g,n]         (never NULL)
 *   dbias   = sum_b (and sum_n unless bias_per_node) dy     (NULL to skip)
 * x must be the forward input (same layout rules).  workspace: b200gf_workspace_bytes(..., 1). */
int b200gf_backward(const b200gf_plan* plan,
                    const void* dy, int dy_layout, int64_t dy_ld,
                    const void* x, int x_layout, int64_t x_ld,
                    const void* h,
                    void* dx, int dx_layout, int64_t dx_ld,
                    void* dh, void* dbias, int bias_per_node,
                    void* workspace, size_t workspace_bytes,
                    int B, int G, int F, int K, void* stream);

/* in_layout = B200GF_FEATURE_MAJOR if ANY of x / y / dy / dx is feature-major, else B200GF_NODE_MAJOR */
size_t b200gf_workspace_bytes(const b200gf_plan* plan, int B, int G, int F, int K,
                              int in_layout, int backward);

/* Measurement hook (bench.py): b200gf_profile_hops(plan, capacity) makes b200gf_forward / b200gf_backward bracket
 * each of their next `capacity` hop launches with CUDA events on the launching stream (capacity 0 turns it off and
 * frees the events).  b200gf_profile_read synchronises those events, writes up to n per-launch durations in ms
 * (launch order) and resets the counter; returns how many were written, or <0 on error. */
int b200gf_profile_hops(b200gf_plan* plan, int capacity);
int b200gf_profile_read(b200gf_plan* plan, float* ms, int n);

/* ------------------------------------------------------------------------------------------------
 * Building blocks (used by the node-partitioned path, which interleaves hops with NCCL all-gathers,
 * and by the parity tests).  All node-major.
 * ---------------------------------------------------------------------------------------------- */

/* one shift: dst[r, 0:C] = sum_j A_e[r, j] src[j, 0:C] for the plan's n_rows rows; A = S_e^T (FWD) or S_e (BWD).
 * src has n_cols rows of stride src_ld, dst has n_rows rows of stride dst_ld.  The vector kernels load and store whole
 * 16- or 32-byte vectors, so they read src[j, C : min(src_ld, padded)) and may write dst[r, C : min(dst_ld, padded)),
 * padded = C rounded up to 32 bytes (8 floats / 4 doubles); those dst columns hold no meaningful value afterwards.
 * Nothing at or past that column, and no row at or past n_rows, is written. */
int b200gf_hop(const b200gf_plan* plan, int e, int direction,
               const void* src, int64_t src_ld, void* dst, int64_t dst_ld, int C, void* stream);

/* Fused hop + collective for the feature-sharded multi-GPU path (one compute step followed by an exchange becomes
 * one kernel): as b200gf_hop, and additionally every computed row slice is stored over NVLink straight into the
 * row-local contraction operand of the rank that owns the node row.  peers: HOST array of n_peers (<= 16) device
 * pointers obtained with b200gf_symm_import (peer p's operand, [rows_per_peer, out_ld]); node row r goes to peer
 * r / rows_per_peer, local row r % rows_per_peer; local column b*gl + g lands at b*stride_b + out_col + g.
 * Needs the 16-byte vector path (gl, out_ld, out_col, stride_b multiples of 4 floats / 2 doubles).
 * b200gf_scatter_rows does the same for an existing node-major matrix (the k = 0 term). */
int b200gf_hop_scatter(const b200gf_plan* plan, int e, int direction,
                       const void* src, int64_t src_ld, void* dst, int64_t dst_ld, int C,
                       const void* const* peers, int n_peers, int64_t rows_per_peer,
                       int64_t out_ld, int64_t out_col, int gl, int64_t stride_b, void* stream);
int b200gf_scatter_rows(int dtype, const void* src, int64_t src_ld, int64_t n_rows, int C,
                        const void* const* peers, int n_peers, int64_t rows_per_peer,
                        int64_t out_ld, int64_t out_col, int gl, int64_t stride_b, void* stream);

/* Fused hop + all-gather for the node-sharded multi-GPU path (SURVEY.md §8e): the plan holds this rank's n_rows rows of
 * the operator (b200gf_plan_create_ops, global column indices); every computed row r is written to row row0 + r of the
 * full-height matrix [n_total, out_ld] of EVERY rank — `peers`: HOST array of n_peers (<= 16) device pointers to those
 * matrices (own one included; b200gf_symm_import or any peer-mapped allocation), so the next hop can start as soon as a
 * fence (b200gf_peer_signal / b200gf_peer_wait) has passed.  If `mc` is not NULL it is the NVSwitch multicast alias of
 * the same buffers and each row is written once with multimem.st instead of n_peers stores.  Rows must be 32-byte
 * aligned on both sides (src_ld, out_ld multiples of 8 floats / 4 doubles).  b200gf_bcast_rows does the same for an
 * existing row block (the k = 0 term x). */
int b200gf_hop_bcast(const b200gf_plan* plan, int e, int direction,
                     const void* src, int64_t src_ld, int C,
                     const void* const* peers, int n_peers, const void* mc,
                     int64_t row0, int64_t out_ld, void* stream);
int b200gf_bcast_rows(int dtype, const void* src, int64_t src_ld, int64_t n_rows, int C,
                      const void* const* peers, int n_peers, const void* mc,
                      int64_t row0, int64_t out_ld, void* stream);

/* 2-D process grid (P = P_r row groups x P_c column groups): one hop with BOTH epilogues.  The plan holds the rows of the
 * rank's row group; src / the all-gather destinations hold only the rank's column group (C = B * G / P_c columns).  Every
 * computed row is (a) written to row row0 + r of the full-height matrix [., bc_ld] of the n_bc ranks of the same COLUMN
 * group (bc_peers; n_bc = 0 for the last hop of a chain: no successor needs it) and (b) delivered to the contraction
 * operand of the rank of the same ROW group that owns node row r (sc_peers[r / rows_per_peer], local row
 * r % rows_per_peer, column b*stride_b + out_col + g — as in b200gf_hop_scatter).  Rows of at least 64 bytes, 32-byte
 * aligned everywhere. */
int b200gf_hop_grid(const b200gf_plan* plan, int e, int direction,
                    const void* src, int64_t src_ld, int C,
                    const void* const* bc_peers, int n_bc, int64_t row0, int64_t bc_ld,
                    const void* const* sc_peers, int n_sc, int64_t rows_per_peer,
                    int64_t out_ld, int64_t out_col, int gl, int64_t stride_b, void* stream);

/* Symmetric buffers for the above: device memory that other processes of the same node can map (CUDA IPC).
 * alloc zero-fills; export writes a 64-byte handle to send to the peers (torch.distributed); import maps a peer's
 * handle and enables peer access; close unmaps. */
int b200gf_symm_alloc(void** ptr, size_t bytes);
int b200gf_symm_free(void* ptr);
int b200gf_symm_export(void* ptr, void* handle64);
int b200gf_symm_import(const void* handle64, void** ptr);
int b200gf_symm_close(void* ptr);

/* Peer fence over symmetric memory (no NCCL): every rank owns an array of n_peers uint64 flags and one uint64 step
 * counter in its symmetric allocation (both zero-initialised).  b200gf_peer_signal increments the local step counter,
 * issues a system-scope fence (so the peer stores of this rank's earlier kernels are visible first) and writes the new
 * step into slot my_rank of every peer's flag array (peer_flags: HOST array of n_peers device pointers, own array
 * included).  b200gf_peer_wait blocks the stream until all n_peers slots of MY flag array have reached the local step.
 * signal-then-wait after the scatters == "every rank's scatters have landed here".  Fixed addresses only, so both
 * calls can be captured in a CUDA graph.  A peer that never signals traps the waiting kernel (bounded spin). */
int b200gf_peer_signal(const void* const* peer_flags, int n_peers, int my_rank, void* local_step, void* stream);
int b200gf_peer_wait(const void* my_flags, int n_peers, const void* local_step, void* stream);

/* tap contraction: out[n, b*Q + q] = bias + sum_t sum_p Z_t[n, b*P + p] * W[t][p][q]   for n < n_rows.
 * zs: HOST array of T device pointers (node-major, stride z_ld[t]); W: device [T,P,Q] contiguous;
 * bias NULL / [Q] / [Q, n_rows] (bias_per_node).  accumulate != 0 adds to the existing `out`.
 * scratch (optional, b200gf_tap_contract_scratch_bytes(T,P,Q) bytes, 16-byte aligned): when given, FP32 problems
 * with P % 32 == 0, Q % 16 == 0, Q <= 256, T <= 16, z_ld == B*P and accumulate == 0 run on the tensor cores
 * (wgmma tf32 with hi/lo error compensation, "3xTF32"); everything else uses the FP32/FP64 FMA kernel. */
int b200gf_tap_contract(int dtype, int64_t n_rows, int B, int P, int Q, int T,
                        const void* const* zs, const int64_t* z_ld, const void* W,
                        const void* bias, int bias_per_node,
                        void* out, int64_t out_ld, int accumulate,
                        void* scratch, size_t scratch_bytes, void* stream);
size_t b200gf_tap_contract_scratch_bytes(int T, int P, int Q);

/* tap gradient: dW[t][p][q] = sum_{n<n_rows, b} A[n, b*P + p] * Vs_t[n, b*Q + q]   (deterministic two-pass)
 * partial: device scratch of b200gf_tap_grad_scratch_bytes(...) bytes. */
int b200gf_tap_grad(int dtype, int64_t n_rows, int B, int P, int Q, int T,
                    const void* A, int64_t a_ld, const void* const* vs, const int64_t* v_ld,
                    void* dW, void* scratch, size_t scratch_bytes, void* stream);
size_t b200gf_tap_grad_scratch_bytes(int dtype, int64_t n_rows, int B, int P, int Q, int T);

/* ------------------------------------------------------------------------------------------------
 * Edge-variant graph filter, the variant of the path used by EdgeVariantGF (config "EdgeNet"):
 *   EVGF(S, x, b)   alegnn/utils/graphML.py:389-488,   EdgeVariantGF.forward  :2670-2698
 * One call per edge feature e, on a compact node set of NA nodes (the rows/columns of Phi that are not identically
 * zero).  Pattern: CSR (rowptr [NA+1], col [nnz]) shared by all (f, k, g).  w [F, K, G, nnz] = Phi^(k)_{f e g} on the
 * pattern (COLUMN convention u_k = Phi^(k) u_{k-1}, u_{-1} = x_g).  The batch index is innermost in every operand:
 *   xT [G, NA, B] (input on the compact set), states [n_states][F*G, NA, B] (u_k), Y [F, NA, B] = sum_g sum_k u_k
 *   (the caller sums over e and adds the bias).
 * diag (optional, int32 [NA]): index of row i's diagonal entry in the pattern, or -1 — when given, step k = 0 is the
 *   layer's "identity on the selected nodes" mask (graphML.py:2653-2663): u_0[i] = w_0[diag[i]] x[i]; NULL = k = 0 is
 *   an ordinary sparse step (functional EVGF with arbitrary matrices).
 * forward : n_states >= K-1 keeps u_0 .. u_{K-2} for the backward pass; n_states == 2 ping-pongs (inference).
 * backward: dY [F, NA, B] -> dw [F, K, G, nnz], dxT [G, NA, B]; needs the transposed pattern (rowptrT, colT) with
 *           perm[it] = index of that entry in the forward pattern, and lam = scratch of 2 * F*G*NA*B elements.
 *           Every element of dw is written, so it need not be zeroed first; with diag, the k = 0 slots other than
 *           the diagonal ones (and every k = 0 slot of a row with diag[i] = -1) are written with exactly 0.
 * ---------------------------------------------------------------------------------------------- */
int b200gf_ev_forward(int dtype, int64_t NA, int B, int G, int F, int K,
                      const int64_t* rowptr, const int32_t* col, const int32_t* diag, int64_t nnz,
                      const void* w, const void* xT, void* states, int n_states, void* Y, void* stream);
int b200gf_ev_backward(int dtype, int64_t NA, int B, int G, int F, int K,
                       const int64_t* rowptr, const int32_t* col,
                       const int64_t* rowptrT, const int32_t* colT, const int64_t* perm, const int32_t* diag, int64_t nnz,
                       const void* w, const void* xT, const void* states, const void* dY,
                       void* lam, void* dw, void* dxT, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Edge-gated recurrent layer (EdgeGatedHiddenState, alegnn/utils/graphML.py:4033-4209; E = 1): the reference's dense
 * B*T x N x N attention gates (learnAttentionGSO, :640-737) kept per non-zero of the mask |S + I| > 1e-9, and the hop
 * with a different gated GSO per sample (GatedGRNN's edge path, :1410-1451, :1474-1514).  Bs = number of samples.
 *   mask CSR: rowptr [N+1], col [nnz] (columns ascending); its transpose: rowptrT [N+1], permT [nnz] = position in the
 *   mask CSR of the k-th entry of column j.  s, dsig1, dsig2: [N, Bs]; alpha, dalpha, dlogit: [nnz, Bs] (sample
 *   innermost).  mixer: DEVICE pointer to the two mixer values (a1, a2).
 *
 * attention forward: alpha[q, b] = softmax over the mask row i of LeakyReLU_0.2(a1 s[j, b] + a2 s[i, b]), q = (i, j).
 * attention backward: dlogit = the softmax and LeakyReLU backward of dalpha (scratch, [nnz, Bs]);
 *   dsig2[i, b] = sum over row i of dlogit, dsig1[j, b] = sum over column j of dlogit (gather over the transpose);
 *   ds = a1 dsig1 + a2 dsig2, da1 = sum s dsig1, da2 = sum s dsig2 are left to the caller.
 * gated hop forward: dst[j, b*C + c] = sum_i S_ij gate[b, p(i, j)] src[i, b*C + c] over the CSR of S^T (rowptrT, colT,
 *   valT) with posT = p(i, j), the entry's position in the mask CSR (-1: outside the mask, contributes nothing).
 *   gate[b, p] is read at gate + b*gate_sb + p*gate_sp.  src / dst node-major, ld >= Bs*C.
 * gated hop backward: dsrc (NULL to skip) = the same hop over the CSR of S (rowptr, col, val, pos) applied to ddst;
 *   dgate (NULL to skip) [b, q] = m_sval[q] * sum_c src[i, b*C + c] ddst[j, b*C + c] for EVERY mask entry q = (i, j),
 *   m_sval [nnz] = S_ij in mask order (0 where S has no entry), written at dgate + b*dgate_sb + q*dgate_sp.
 * All four are deterministic (one writer per output element, fixed summation order).
 * ---------------------------------------------------------------------------------------------- */
int b200gf_egate_attention_forward(int dtype, int64_t N, int64_t nnz, int Bs,
                                   const int64_t* rowptr, const int32_t* col,
                                   const void* s, const void* mixer, void* alpha, void* stream);
int b200gf_egate_attention_backward(int dtype, int64_t N, int64_t nnz, int Bs,
                                    const int64_t* rowptr, const int32_t* col,
                                    const int64_t* rowptrT, const int32_t* permT,
                                    const void* s, const void* mixer, const void* alpha, const void* dalpha,
                                    void* dlogit, void* dsig1, void* dsig2, void* stream);
/* Graph attention layers (GraphAttentional, GraphFilterAttentional, EdgeVariantAttentional, graphML.py:739-969,
 * :2849-3270): the same attention on the same mask CSR, with the two ends of an edge scored by two arrays, s_src read at
 * the column node j and s_dst at the row node i (mixer: DEVICE pointer to (a1, a2); the layers pass (1, 1)):
 *   forward:  alpha[q, b] = softmax over the mask row i of LeakyReLU_0.2(a1 s_src[j, b] + a2 s_dst[i, b]), q = (i, j);
 *   backward: dlogit as above; dsig1[j, b] = sum over column j of dlogit (the gradient of the a1 s_src term),
 *             dsig2[i, b] = sum over row i of dlogit (of the a2 s_dst term).
 * s_src, s_dst, dsig1, dsig2 [N, Bs]; alpha, dalpha, dlogit [nnz, Bs].  b200gf_egate_attention_* are these with s
 * passed as both arrays. */
int b200gf_attention_forward(int dtype, int64_t N, int64_t nnz, int Bs,
                             const int64_t* rowptr, const int32_t* col,
                             const void* s_src, const void* s_dst, const void* mixer, void* alpha, void* stream);
int b200gf_attention_backward(int dtype, int64_t N, int64_t nnz, int Bs,
                              const int64_t* rowptr, const int32_t* col,
                              const int64_t* rowptrT, const int32_t* permT,
                              const void* s_src, const void* s_dst, const void* mixer, const void* alpha,
                              const void* dalpha, void* dlogit, void* dsig1, void* dsig2, void* stream);
int b200gf_gated_hop_forward(int dtype, int64_t N, int Bs, int C,
                             const int64_t* rowptrT, const int32_t* colT, const void* valT, const int32_t* posT,
                             const void* gate, int64_t gate_sb, int64_t gate_sp,
                             const void* src, int64_t src_ld, void* dst, int64_t dst_ld, void* stream);
int b200gf_gated_hop_backward(int dtype, int64_t N, int Bs, int C,
                              const int64_t* rowptr, const int32_t* col, const void* val, const int32_t* pos,
                              const int64_t* m_rowptr, const int32_t* m_col, const void* m_sval,
                              const void* gate, int64_t gate_sb, int64_t gate_sp,
                              const void* src, int64_t src_ld, const void* ddst, int64_t ddst_ld,
                              void* dsrc, int64_t dsrc_ld, void* dgate, int64_t dgate_sb, int64_t dgate_sp,
                              void* stream);

/* ------------------------------------------------------------------------------------------------
 * Node-variant graph filter (NVGF, alegnn/utils/graphML.py:293-387; NodeVariantGF :2317-2509), node-major only:
 *   y[n, b*F + f] = bias + sum_e sum_k sum_g h[f,e,k,g,node_tap[n]] (x_g S_e^k)[n]
 * Every node n reads the tap block m = node_tap[n] (int32 [N], 0 <= m < M; the layer's copyNodes), so the reference's
 * [F,E,K,G,N] index_select of the taps is never materialised.
 *
 * b200gf_nv_pack_taps: h [F,E,K,G,M] -> W [M][T][G][F], T = 1 + E*(K-1): W[m][0] = sum_e h[:,e,0,:,m]^T (k = 0 is the
 *   same x for every e), W[m][1 + e*(K-1) + (k-1)] = h[:,e,k,:,m]^T.  Each node's taps are one contiguous block.
 * b200gf_nv_forward: the E*(K-1) hops of b200gf_forward into the workspace, then one per-node contraction.  x [N, x_ld],
 *   y [N, y_ld] (ld >= B*G / B*F); bias NULL, [F] (bias_per_node = 0) or [F, N] (bias_per_node = 1).  Writes nothing at
 *   or past column B*F of y and no row at or past N.
 * b200gf_nv_backward: dy [N, dy_ld], x = the forward input.
 *   dx (NULL to skip) [N, dx_ld]: dz_t[n, b*G+g] = sum_f W[m][t][g][f] dy[n, b*F+f] and
 *     dx = dz_0 + sum_e BWD(dz_{e,1} + BWD(dz_{e,2} + ... BWD(dz_{e,K-1})));  nothing at or past column B*G is written.
 *   dh [F,E,K,G,M] (never NULL): dh[f,e,k,g,m] = sum over the nodes n of tap m, sum_b (x_g S_e^k)[n,b] dy[n,b,f]
 *     (k = 0: the merged term, the same value in every e).  Every dh element is written; taps that no node uses get
 *     exactly 0.  tap_rowptr (int64 [M+1]) / tap_nodes (int32 [N]) list the nodes of every tap in ascending order (the
 *     inverse of node_tap).  The sum is a deterministic two-pass reduction over fixed-size pieces of each member list,
 *     so a tap shared by every node (M = 1) is spread over many blocks.
 *   dbias (NULL to skip): as b200gf_backward.
 * workspace: b200gf_nv_workspace_bytes(plan, B, G, F, K, M, backward) bytes, 256-byte aligned.  T <= 48.
 * ---------------------------------------------------------------------------------------------- */
int b200gf_nv_pack_taps(int dtype, const void* h, void* W, int F, int E, int K, int G, int64_t M, void* stream);
int b200gf_nv_forward(const b200gf_plan* plan, const void* x, int64_t x_ld, const void* W, const int32_t* node_tap,
                      int64_t M, const void* bias, int bias_per_node, void* y, int64_t y_ld,
                      void* workspace, size_t workspace_bytes, int B, int G, int F, int K, void* stream);
int b200gf_nv_backward(const b200gf_plan* plan, const void* dy, int64_t dy_ld, const void* x, int64_t x_ld,
                       const void* W, const int32_t* node_tap, int64_t M,
                       const int64_t* tap_rowptr, const int32_t* tap_nodes,
                       void* dx, int64_t dx_ld, void* dh, void* dbias, int bias_per_node,
                       void* workspace, size_t workspace_bytes, int B, int G, int F, int K, void* stream);
size_t b200gf_nv_workspace_bytes(const b200gf_plan* plan, int B, int G, int F, int K, int64_t M, int backward);

/* ------------------------------------------------------------------------------------------------
 * ARMA graph filter by Jacobi iterations (jARMA, alegnn/utils/graphML.py:490-638; GraphFilterARMA :2714-2847), the
 * general-diagonal part (H1 + H2; the residue H3 = LSIGF(phi, S, x) + bias is b200gf_forward / b200gf_backward on the
 * plan of S).  Node-major only.  For every edge feature e of `plan`, with S~_e = S_e - diag(S_e), d_e = diag(S_e) and
 * r = 1 / (d_e - psi[f,e,p,g]) (per node), in the COLUMN convention S~ v:
 *   z_0 = r . x_g, z_t = r . (S~_e z_{t-1}) (t = 1..tMax);   y_0 = x_g, y_t = r . (S~_e y_{t-1}) (t = 1..tMax+1)
 *   out[n, b*F + f] += sum_{e,p,g} ( varphi[f,e,p,g] sum_t (-1)^t z_t + (-1)^(tMax+1) y_{tMax+1} )[n, b]
 * plan: built from S~_e^T (b200gf_plan_create), so its FWD hop is S~_e v and its BWD hop S~_e^T v.
 * d: [E, N] (the diagonals, row e for edge feature e).  psi, varphi: [F, E, P, G].  tMax >= 0.
 *
 * b200gf_arma_forward: x [N, x_ld] (ld >= B*G), out [N, out_ld] (ld >= B*F) is ADDED to (it normally holds the H3 term
 *   and the bias already); nothing at or past column B*F of out is written.  states: NULL (inference: two ping-pong
 *   states in the workspace) or a buffer of b200gf_arma_workspace_bytes(..., 3) bytes, 256-byte aligned, that receives
 *   the E*(tMax+1) wide states [N, ldw] the backward reads (ldw = B*F*P*G*2 padded to 32 bytes).
 * b200gf_arma_backward: dy [N, dy_ld] = dU, states = the forward's.
 *   dx (NULL to skip) [N, dx_ld]: ADDED to, dx_g += sum_{e,f,p} r . lambda_0 + sum_e S~_e^T sum_{f,p} (r . mu_1) with the
 *     adjoints lambda_tMax = (-1)^tMax varphi dU, lambda_t = (-1)^t varphi dU + S~^T (r . lambda_{t+1}),
 *     mu_{tMax+1} = (-1)^(tMax+1) dU, mu_t = S~^T (r . mu_{t+1}); nothing at or past column B*G is written.
 *   dpsi, dvarphi [F, E, P, G] (never NULL; every element written):
 *     dpsi = sum_{n,b} ( sum_t lambda_t . r . z_t + sum_{t>=1} mu_t . r . y_t ),  dvarphi = sum_{n,b} dU sum_t (-1)^t z_t,
 *     as deterministic two-pass column sums over fixed row pieces.
 * workspace: b200gf_arma_workspace_bytes(plan, B, G, F, P, tMax, what) bytes, 256-byte aligned; what = 0 forward without
 *   states, 1 forward with states, 2 backward, 3 the size of the forward's `states` buffer.  0 = invalid arguments.
 * ---------------------------------------------------------------------------------------------- */
int b200gf_arma_forward(const b200gf_plan* plan, const void* d, const void* psi, const void* varphi, int tMax,
                        int B, int G, int F, int P, const void* x, int64_t x_ld, void* out, int64_t out_ld,
                        void* states, void* workspace, size_t workspace_bytes, void* stream);
int b200gf_arma_backward(const b200gf_plan* plan, const void* d, const void* psi, const void* varphi, int tMax,
                         int B, int G, int F, int P, const void* dy, int64_t dy_ld, const void* states,
                         void* dx, int64_t dx_ld, void* dpsi, void* dvarphi,
                         void* workspace, size_t workspace_bytes, void* stream);
size_t b200gf_arma_workspace_bytes(const b200gf_plan* plan, int B, int G, int F, int P, int tMax, int what);

/* layout conversion between the reference's [C, N] (feature-major, C = B*G) and node-major [N, ld] */
int b200gf_to_node_major(int dtype, const void* src_cn, void* dst_nc, int64_t dst_ld,
                         int64_t N, int C, void* stream);
int b200gf_to_feature_major(int dtype, const void* src_nc, int64_t src_ld, void* dst_cn,
                            int64_t N, int C, void* stream);

/* taps h[F,E,K,G] -> W[T][G][F] with T = 1 + E*(K-1): W[0] = sum_e h[:,e,0,:]^T (k = 0 is the same x for
 * every e, graphML.py:154), W[1 + e*(K-1) + (k-1)] = h[:,e,k,:]^T.   transpose_taps != 0 gives the
 * backward-to-input form W[t][F][G] (no transpose). */
int b200gf_pack_taps(int dtype, const void* h, void* W, int F, int E, int K, int G,
                     int transpose_taps, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GF_H_ */
