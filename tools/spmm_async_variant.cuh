// cp.async-staged variant of the hop kernel — it was slower than the shipped spmm_hop_v2_kernel and is kept with the sweep
// tool as an alternative to re-measure (DESIGN.md §3.1).
//
// Gathered rows are staged in shared memory with cp.async (LDGSTS.128, L2-only), so the number of bytes in flight per SM
// is set by shared memory (2 x SLOTS neighbour rows per warp) instead of by registers, and the index chain
// rowptr -> col/val -> gather is software-pipelined three units deep:
//    iteration i:  issue the gathers of unit i+1 (its col/val arrived during iteration i-1)
//                  load col/val of unit i+2, (rowptr of the next 32-row block is fetched a block ahead, coalesced)
//                  wait for unit i's group, reduce it from shared memory, store the row
// A unit is a row (or a SLOTS-neighbour segment of a longer row).  Every lane reads back exactly the 16 bytes it copied
// itself, so no barrier is needed: cp.async.wait_group is the only synchronisation.
#pragma once
#include "../graph-neural-networks_b200/csrc/spmm_kernels.cuh"

namespace b200gf {

__device__ __forceinline__ void cp_async16(uint32_t saddr, const void* g, uint64_t pol, bool hint) {
  if (hint)
    asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(saddr), "l"(g), "l"(pol) : "memory");
  else
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(saddr), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// shared memory per warp: 2 * SLOTS * L * 16 bytes
template <typename T, typename IDX, int VEC, int L, int SLOTS, int THREADS, int MINB, int HINT, int SCATTER>
__global__ void __launch_bounds__(THREADS, MINB)
spmm_hop_async_kernel(const IDX* __restrict__ rowptr, const int32_t* __restrict__ col, const T* __restrict__ val,
                      const T* __restrict__ src, int src_ld, T* __restrict__ dst, int dst_ld, int n_rows, int C,
                      const ScatterParam<T, SCATTER> sp) {
  static_assert(SLOTS % 32 == 0 && SLOTS >= 32, "SLOTS is a multiple of the 32-entry col/val window");
  constexpr int NW = SLOTS / 32;             // col/val registers per unit
  constexpr int S = 32 / L;                  // neighbour rows per warp-wide copy
  constexpr int BUF_V = SLOTS * L;           // 16-byte vectors per buffer
  extern __shared__ __align__(16) unsigned char smem_async[];
  uint64_t pol = 0;
  if constexpr (HINT >= 2) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int sub = lane / L;
  const int cl = lane % L;
  using V16 = typename std::conditional<sizeof(T) == 4, float4, double2>::type;
  V16* const wbuf = reinterpret_cast<V16*>(smem_async) + (size_t)wib * 2 * BUF_V;
  const uint32_t wbuf_s = (uint32_t)__cvta_generic_to_shared(wbuf);

  const int n_warps = gridDim.x * (THREADS >> 5);
  const int n_vblk = (n_rows + 31) >> 5;     // 32-row blocks; the column chunk is blockIdx.y (chunk-major CTA order)
  const int vb0 = blockIdx.x * (THREADS >> 5) + wib;
  if (vb0 >= n_vblk) return;
  const int cbase = (int)blockIdx.y * (L * VEC) + cl * VEC;
  const bool col_ok = cbase < C;
  const T* __restrict__ srcc = src + cbase;

  // rowptr windows: A = the 32-row block the fetch cursor is in, B = this warp's next block (prefetched one block ahead,
  // coalesced: lane i holds row i of the block)
  int vbA = vb0;
  IDX rbA = 0, rbB = 0;
  int rlA = 0, rlB = 0;
  auto load_block = [&](int vb, IDX& rb, int& rl) {
    rb = 0; rl = 0;
    if (vb < n_vblk) {
      const int row = vb * 32 + lane;
      if (row < n_rows) { rb = __ldg(rowptr + row); rl = (int)(__ldg(rowptr + row + 1) - rb); }
    }
  };
  load_block(vbA, rbA, rlA);
  load_block(vbA + n_warps, rbB, rlB);

  // the fetch cursor walks units: (vb, r, off) = segment [off, off + SLOTS) of row r of virtual block vb (== vbA)
  struct Cur { int vb, r, off; };
  auto rows_in = [&](int vb) { return min(32, n_rows - vb * 32); };
  auto bounds = [&](const Cur& c, IDX& beg, int& len) {
    beg = __shfl_sync(FULL, rbA, c.r);
    len = __shfl_sync(FULL, rlA, c.r);
  };
  auto advance = [&](Cur& c, int len) {
    if (c.off + SLOTS < len) { c.off += SLOTS; return; }
    c.off = 0;
    if (++c.r == rows_in(c.vb)) {
      c.r = 0; c.vb += n_warps;
      vbA = c.vb; rbA = rbB; rlA = rlB;                 // roll the windows, prefetch the block after
      load_block(vbA + n_warps, rbB, rlB);
    }
  };

  // per-stage unit state
  struct Unit { int row, cnt; bool first, last, valid; };
  int32_t c1[NW], c2[NW];
  T v0[NW], v1[NW], v2[NW];
  Unit u0, u1, u2;
  auto fetch = [&](const Cur& cur, Unit& u, int32_t* c, T* v) {   // col/val loads of a unit (cursor must be valid)
    u.valid = cur.vb < n_vblk;
    u.cnt = 0; u.first = u.last = false; u.row = 0;
#pragma unroll
    for (int w = 0; w < NW; ++w) { c[w] = 0; v[w] = T(0); }
    if (!u.valid) return 0;
    IDX beg; int len;
    bounds(cur, beg, len);
    u.row = cur.vb * 32 + cur.r;
    u.cnt = min(len - cur.off, SLOTS);
    u.first = cur.off == 0;
    u.last = cur.off + SLOTS >= len;
#pragma unroll
    for (int w = 0; w < NW; ++w) {
      if (w * 32 + lane < u.cnt) {
        c[w] = ld_stream(col + beg + cur.off + w * 32 + lane);
        v[w] = ld_stream(val + beg + cur.off + w * 32 + lane);
      }
    }
    return len;
  };
  auto issue = [&](const Unit& u, const int32_t* c, int parity) {
    if (u.valid) {
      const uint32_t sb = wbuf_s + (uint32_t)(parity * BUF_V + lane) * 16u;
#pragma unroll
      for (int w = 0; w < NW; ++w) {
        const int cw = min(u.cnt - 32 * w, 32);          // entries of this 32-wide col/val window
#pragma unroll 4
        for (int j = 0; j * S < cw; ++j) {
          const int jj = j * S + sub;
          const int32_t cc = __shfl_sync(FULL, c[w], jj);
          if (jj < cw && col_ok)
            cp_async16(sb + (uint32_t)(w * L + j) * 512u, srcc + (int64_t)cc * src_ld, pol, HINT >= 2);
        }
      }
    }
    cp_async_commit();
  };

  Cur cur{vb0, 0, 0};
  // prologue: unit 0 and unit 1 fetched, unit 0 issued
  int len = fetch(cur, u0, c1, v0);
  issue(u0, c1, 0);
  if (u0.valid) advance(cur, len);
  len = fetch(cur, u1, c1, v1);
  if (u1.valid) advance(cur, len);

  Acc<T, VEC> acc;
  acc.zero();
  int parity = 0;
  while (u0.valid) {
    // (a) gathers of the next unit
    issue(u1, c1, parity ^ 1);
    // (b) col/val of the unit after that
    len = fetch(cur, u2, c2, v2);
    if (u2.valid) advance(cur, len);
    // (c) wait for this unit's copies (all but the most recent group) and reduce
    cp_async_wait<1>();
    {
      if (u0.first) acc.zero();
      const V16* b = wbuf + parity * BUF_V + lane;
#pragma unroll
      for (int w = 0; w < NW; ++w) {
        const int cw = min(u0.cnt - 32 * w, 32);
#pragma unroll 4
        for (int j = 0; j * S < cw; ++j) {
          const int jj = j * S + sub;
          const T wt = __shfl_sync(FULL, v0[w], jj);
          if (jj < cw && col_ok) {
            const V16 d = b[(w * L + j) * 32];
            if constexpr (VEC == 4) {
              acc.v[0] = fma(wt, d.x, acc.v[0]); acc.v[1] = fma(wt, d.y, acc.v[1]);
              acc.v[2] = fma(wt, d.z, acc.v[2]); acc.v[3] = fma(wt, d.w, acc.v[3]);
            } else {
              acc.v[0] = fma(wt, d.x, acc.v[0]); acc.v[1] = fma(wt, d.y, acc.v[1]);
            }
          }
        }
      }
      if (u0.last) {
        Acc<T, VEC> r = acc;
#pragma unroll
        for (int off = L; off < 32; off <<= 1) {
#pragma unroll
          for (int i = 0; i < VEC; ++i) r.v[i] += __shfl_xor_sync(FULL, r.v[i], off);
        }
        if (sub == 0 && col_ok) {
          if constexpr (SCATTER == EPI_BCAST) {
            bcast_store<T, VEC>(sp.a, u0.row, cbase, r);
          } else {
            store_vec<T, VEC, 0>(dst + (int64_t)u0.row * dst_ld + cbase, r);
            if constexpr (SCATTER == EPI_SCATTER) {
              if (sp.a.n_peers > 0) scatter_store<T, VEC>(sp.a, u0.row, cbase, r);
            }
          }
        }
      }
    }
    // (d) rotate the pipeline
    u0 = u1; u1 = u2;
#pragma unroll
    for (int w = 0; w < NW; ++w) { v0[w] = v1[w]; v1[w] = v2[w]; c1[w] = c2[w]; }
    parity ^= 1;
  }
  cp_async_wait<0>();
}

}  // namespace b200gf
