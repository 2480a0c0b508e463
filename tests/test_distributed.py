"""Node-partitioned / feature-partitioned LSIGF (graph-neural-networks_b200/distributed.py).

CPU: world_size-2 gloo runs with an oracle-backed `ops` (scipy / numpy stand-ins for the C-ABI building blocks) —
exercises the partitioning, padding, in-place all-gather and reduce-scatter choreography against the fp64 oracle.
GPU (-m gpu, needs >= 2 devices): the same through NCCL and the CUDA building blocks."""
import os
import pickle
import socket
import tempfile

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import lsigf_oracle as orc


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


class OracleOps:
    """CPU stand-ins with the CudaOps interface (test infrastructure: uses scipy, mirrors include/b200gf.h semantics)."""

    def __init__(self):
        self.device = torch.device("cpu")

    def make_plan_ops(self, fwd, bwd, n_rows, n_cols, dtype):
        import scipy.sparse as sp
        mk = lambda ops: [sp.csr_matrix((v, c, r), shape=(n_rows, n_cols)) for (r, c, v) in ops]  # noqa: E731
        return {"fwd": mk(fwd), "bwd": None if bwd is None else mk(bwd)}

    def make_plan_full(self, gso):
        import scipy.sparse as sp
        full = [sp.csr_matrix((v, c, r), shape=(gso.N, gso.N)) for (r, c, v) in gso.csr]
        return {"fwd": [m.T.tocsr() for m in full], "bwd": full}     # fwd gathers with rows of S^T, bwd with rows of S

    def hop(self, plan, e, direction, src, dst, C):
        A = plan["fwd" if direction == 0 else "bwd"][e]   # like b200gf_hop: reads n_cols rows of src, writes n_rows rows of dst
        out = A @ src[:A.shape[1], :C].numpy()
        dst[:A.shape[0], :C] = torch.from_numpy(np.ascontiguousarray(out))

    def pack_taps(self, h, transpose):
        F, E, K, G = h.shape
        W = [h[:, :, 0, :].sum(1).t()]
        for e in range(E):
            for k in range(1, K):
                W.append(h[:, e, k, :].t())
        W = torch.stack(W)                                     # [T, G, F]
        return (W.transpose(1, 2) if transpose else W).contiguous()

    def tap_grad(self, A, vs, n_rows, B, P, Q):
        a = A[:n_rows, :B * P].reshape(n_rows, B, P)
        return torch.stack([torch.einsum("nbp,nbq->pq", a, v[:n_rows, :B * Q].reshape(n_rows, B, Q)) for v in vs])

    def tap_contract(self, zs, W, bias, out, n_rows, B, P, Q, bias_per_node=0):
        acc = torch.zeros(n_rows, B, Q, dtype=out.dtype)
        for t, z in enumerate(zs):
            acc += torch.einsum("nbp,pq->nbq", z[:n_rows, :B * P].reshape(n_rows, B, P), W[t])
        if bias is not None:
            acc += bias.view(1, 1, Q)
        out[:n_rows, :B * Q] = acc.reshape(n_rows, B * Q)


def _case(N=203, B=2, G=6, F=8, K=4, E=2, seed=3):
    import scipy.sparse as sp
    rng = np.random.default_rng(seed)
    mats = []
    for e in range(E):
        m = sp.random(N, N, density=6.0 / N, format="csr", random_state=np.random.RandomState(seed + e),
                      data_rvs=lambda n: rng.standard_normal(n))
        mats.append(sp.csr_matrix(m / max(abs(m).sum(axis=1).max(), 1e-30)))
    x = rng.standard_normal((B, G, N))
    h = rng.uniform(-0.3, 0.3, (F, E, K, G))
    b = rng.uniform(-0.3, 0.3, (F, 1))
    return mats, x, h, b


def _worker(rank, world, port, backend, runs, out_path):
    """One rank: joins the process group, then runs every config of `runs` (keyword arguments of _partitioned) on it;
    rank 0 pickles the list of their gathered outputs to out_path (a file, not a queue: the parent reads it only after
    joining the ranks, and a pipe would block a writer of more than its buffer until then)."""
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    if backend == "nccl":
        torch.cuda.set_device(rank)
        dev = torch.device("cuda", rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    else:
        dev = torch.device("cpu")
        dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        outs = [_partitioned(rank, world, backend, dev, **cfg) for cfg in runs]
        if rank == 0:
            with open(out_path, "wb") as f:
                pickle.dump(outs, f)
    finally:
        dist.destroy_process_group()


def _partitioned(rank, world, backend, dev, mode, dtype_name, G=6, backward=True, F=8, grid=None, K=4, trace=False):
    """PartitionedLSIGF forward (twice: buffers are reused), its CUDA-graph replay where the fused path allows one, and
    backward through part.apply; returns (rank 0) the outputs gathered over the ranks as fp64 arrays in the oracle's
    layouts: y [B, F, N], and with backward dh [F, E, K, G], dx [B, G, N], db [F, 1].  trace: the hop kernels the first
    forward and the backward launched are returned too, with whether the fused path ran and its arenas' kinds."""
    import gnn_b200
    from gnn_b200.distributed import PartitionedLSIGF
    dtype = getattr(torch, dtype_name)
    ops = OracleOps() if backend != "nccl" else None
    mats, x, h, b = _case(G=G, F=F, K=K)
    B, G, N = x.shape
    F = h.shape[0]
    gso = gnn_b200.SparseGSO.from_scipy(mats, dtype=dtype)
    part = PartitionedLSIGF(gso, mode=mode, device=dev, ops=ops, grid=grid)
    R = part.rows_per_rank
    xn = torch.tensor(x, dtype=dtype).reshape(B * G, N).t().contiguous()       # node-major [N, B*G]
    ht = torch.tensor(h, dtype=dtype, device=dev)
    bt = torch.tensor(b, dtype=dtype, device=dev)
    if mode == "grid":
        x_local = part.grid_tile(xn, B, G).to(dev)
    elif mode == "nodes":
        xp = torch.zeros(part.n_pad, B * G, dtype=dtype)
        xp[:N] = xn
        x_local = xp[part.r0:part.r1].to(dev)
    else:
        g0, g1 = part.feature_slice(G)
        x_local = xn.view(N, B, G)[:, :, g0:g1].reshape(N, B * (g1 - g0)).contiguous().to(dev)
    if backend == "nccl":
        # default construction under NCCL = the kernels move their rows over NVLink themselves; a silent fall back to
        # the NCCL-collective path would leave the fused kernels untested
        assert part.fused, "default PartitionedLSIGF under NCCL must take the fused path"
    kernels = []

    def traced(fn):
        if not trace:
            return fn()
        from torch.profiler import ProfilerActivity, profile
        from dispatch_harness import _norm
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        kernels.extend(_norm(e.name).split("(")[0] for e in prof.events()
                       if e.device_type == torch.autograd.DeviceType.CUDA and "b200gf::" in e.name)
        return out

    y_local = traced(lambda: part.forward(ht, x_local, bt, B=B))
    y_local = part.forward(ht, x_local, bt, B=B)
    assert tuple(y_local.shape) == (R, B * F)
    if backend == "nccl" and G % (4 * world) == 0:
        # the same step replayed as CUDA graphs (peer-flag fence, no NCCL inside): must reproduce the eager result
        run = part.graphed(ht, x_local, bt, B=B)
        for _ in range(3):
            y_graph = run()
        torch.cuda.synchronize()
        assert torch.equal(y_graph, y_local), "graph replay differs from the eager fused step"
    out = {}
    if backward:
        # backward through the autograd wrapper (collective on every rank): dh, db summed over ranks, dx sharded like x
        dy = np.random.default_rng(99).standard_normal((B, F, N))
        dyp = torch.zeros(part.n_pad, B * F, dtype=dtype)
        dyp[:N] = torch.tensor(dy, dtype=dtype).reshape(B * F, N).t()
        hg, xg, bg = (t.clone().requires_grad_(True) for t in (ht, x_local, bt))
        traced(lambda: part.apply(hg, xg, bg, B).backward(dyp[part.r0:part.r1].to(dev)))
        if mode == "grid":
            tiles = [torch.empty_like(xg.grad) for _ in range(world)]      # [rows_per_group, B*(G/P_c)] of rank (rg, cg)
            dist.all_gather(tiles, xg.grad.contiguous())
            Rr, Gl = part.rows_per_group, G // part.Pc
            dx_full = torch.zeros(part.n_pad, B, G, dtype=dtype, device=dev)
            for p_, t_ in enumerate(tiles):
                r_, c_ = p_ // part.Pc, p_ % part.Pc
                dx_full[r_ * Rr:(r_ + 1) * Rr, :, c_ * Gl:(c_ + 1) * Gl] = t_.reshape(Rr, B, Gl)
            dx_nm = dx_full[:N]
        elif mode == "nodes":
            dxs = [torch.empty_like(xg.grad) for _ in range(world)]
            dist.all_gather(dxs, xg.grad.contiguous())
            dx_nm = torch.cat(dxs)[:N].reshape(N, B, G)
        else:
            per = (G + world - 1) // world
            mine = torch.zeros(N, B, per, dtype=dtype, device=dev)
            mine[:, :, :g1 - g0] = xg.grad.reshape(N, B, g1 - g0)
            dxs = [torch.empty_like(mine) for _ in range(world)]
            dist.all_gather(dxs, mine)
            dx_nm = torch.cat(dxs, dim=2)[:, :, :G] if G % world == 0 else \
                torch.cat([d[:, :, :max(0, min(G, (p + 1) * per) - min(G, p * per))] for p, d in enumerate(dxs)], dim=2)
        out.update(dh=hg.grad.cpu().double().numpy(), dx=dx_nm.cpu().double().numpy().transpose(1, 2, 0),
                   db=bg.grad.cpu().double().numpy())
    ys = [torch.empty_like(y_local) for _ in range(world)]
    dist.all_gather(ys, y_local.contiguous())
    out["y"] = torch.cat(ys)[:N].cpu().double().numpy().reshape(N, B, F).transpose(1, 2, 0)
    if trace:
        arenas = sorted({a.kind for a in part._arenas.values()} | ({"cuda-ipc"} if part._symm_by_width else set()))
        out.update(kernels=sorted(set(kernels)), fused=part.fused, arenas=arenas)
    return out if rank == 0 else None


def _spawn(backend, world, runs):
    for attempt in range(3):                     # the rendezvous port is picked by bind-and-release: retry if someone took it
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "outs.pkl")
            try:
                mp.spawn(_worker, args=(world, _free_port(), backend, runs, path), nprocs=world, join=True)
            except Exception as exc:
                if "EADDRINUSE" not in str(exc) or attempt == 2:
                    raise
                continue
            with open(path, "rb") as f:
                return pickle.load(f)


def _hold(out, dtype_name, G=6, backward=True, F=8, K=4):
    """Holds a run's gathered outputs to orc.lsigf_envelope componentwise (fp32: with the 3xTF32 tensor-core
    contraction's term) and returns their largest max-normalised error against the sparse fp64 oracle."""
    import scipy.sparse as sp
    mats, x, h, b = _case(G=G, F=F, K=K)
    B, _, N = x.shape
    npd = np.float32 if dtype_name == "float32" else np.float64
    r64 = lambda a: a.astype(npd).astype(np.float64)  # noqa: E731
    mr = [sp.csr_matrix((r64(m.data), m.indices, m.indptr), shape=m.shape) for m in mats]
    dy = r64(np.random.default_rng(99).standard_normal((B, h.shape[0], N)))
    env = orc.lsigf_envelope(r64(h), mr, r64(x), r64(b), dy, npd, tf32x3=npd == np.float32)
    refs = {"y": orc.lsigf_sparse(r64(h), mr, r64(x), r64(b))}
    if backward:
        refs.update(zip(("dh", "dx", "db"), orc.lsigf_grads_sparse(r64(h), mr, r64(x), dy, (h.shape[0], 1))))
    errs = []
    for name, ref in refs.items():
        v = orc.bound_violation(out[name], ref, env[name])
        print("%s: worst error / bound %.3g" % (name, v))
        assert v <= 1.0, "%s: error %.3g x its componentwise bound" % (name, v)
        errs.append(float(np.abs(out[name] - ref).max() / np.abs(ref).max()))
    return max(errs)


def _run(backend, mode, dtype_name, world=2, G=6, backward=True, F=8, grid=None, K=4):
    out, = _spawn(backend, world, [dict(mode=mode, dtype_name=dtype_name, G=G, backward=backward, F=F, grid=grid, K=K)])
    return _hold(out, dtype_name, G=G, backward=backward, F=F, K=K)


@pytest.mark.parametrize("mode,G", [("nodes", 6), ("features", 6), ("features", 5)])
def test_partitioned_gloo_world2(mode, G):
    """G = 6: all-to-all exchange of the shifted slices; G = 5 (not divisible by 2): reduce-scatter variant.
    Forward and backward (dh, dx, db) against the sparse oracle."""
    err = _run("gloo", mode, "float64", G=G)
    assert err < 1e-12, err


@pytest.mark.parametrize("mode,K", [("nodes", 2), ("nodes", 1), ("features", 2)])
def test_partitioned_gloo_world2_short_filters(mode, K):
    """K = 2: a single hop per chain (the last hop of a chain is never exchanged); K = 1: no hop at all."""
    err = _run("gloo", mode, "float64", K=K)
    assert err < 1e-12, err


@pytest.mark.parametrize("world,grid,K", [(4, (2, 2), 4), (2, (2, 1), 4), (2, (1, 2), 4), (4, (2, 2), 2), (4, (4, 1), 3), (4, (1, 4), 1)])
def test_partitioned_grid_gloo(world, grid, K):
    """The 2-D grid sharding with collectives in place of the fused epilogues (same tiles, same ownership, same operand
    layout): all-gather of every hop output inside the column group, all-to-all of the slices inside the row group.
    Forward and backward (dh, dx tiles, db) against the sparse oracle; G = 8 features split over the column groups."""
    err = _run("gloo", "grid", "float64", world=world, G=8, grid=grid, K=K)
    assert err < 1e-12, err


def test_row_slice_and_padding():
    from gnn_b200.distributed import row_slice
    rowptr = np.array([0, 2, 2, 5], dtype=np.int64)
    col = np.array([0, 2, 0, 1, 2], dtype=np.int32)
    val = np.arange(5, dtype=np.float64)
    rp, c, v = row_slice((rowptr, col, val), 1, 3)
    assert rp.tolist() == [0, 0, 3] and c.tolist() == [0, 1, 2] and v.tolist() == [2.0, 3.0, 4.0]
    rp, c, v = row_slice((rowptr, col, val), 2, 5)      # rows 3, 4 do not exist: empty padding rows
    assert rp.tolist() == [0, 3, 3, 3] and c.tolist() == [0, 1, 2]
    rp, c, v = row_slice((rowptr, col, val), 4, 6)      # entirely padding
    assert rp.tolist() == [0, 0, 0] and len(c) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("mode,G", [("nodes", 6), ("nodes", 48), ("features", 6), ("features", 16)])
@pytest.mark.parametrize("dtype_name,tol", [("float32", 1e-4), ("float64", 1e-11)])
def test_partitioned_nccl_world2(mode, G, dtype_name, tol):
    """nodes/G = 6: narrow rows, NCCL all-gather per hop; nodes/G = 48: the hop kernel with the fused all-gather epilogue
    (b200gf_hop_bcast: NVLink peer stores / NVSwitch multicast into symmetric memory, peer-flag fences, CUDA-graph replay);
    features/G = 6: NCCL all-to-all path; features/G = 16: the fused hop + NVLink scatter kernels (G/P = 8 columns per
    rank, 16-byte vectors) writing into CUDA-IPC symmetric operands."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    err = _run("nccl", mode, dtype_name, G=G, backward=False)    # backward over NCCL: tests/test_widen_distributed.py
    assert err < tol, err


@pytest.mark.gpu
@pytest.mark.parametrize("grid", [(2, 1), (1, 2)])
@pytest.mark.parametrize("dtype_name,tol", [("float32", 1e-4), ("float64", 1e-11)])
def test_partitioned_grid_nccl_world2(grid, dtype_name, tol):
    """The 2-D grid sharding on 2 GPUs in its two degenerate shapes: (2, 1) = two row groups, one column group — the
    all-gather epilogue carries the exchange, the scatter stays local; (1, 2) = one row group, two column groups — the
    other way round.  Forward (and CUDA-graph replay) against the sparse oracle."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    err = _run("nccl", "grid", dtype_name, G=48, backward=False, grid=grid)
    assert err < tol, err


@pytest.mark.gpu
def test_partitioned_nccl_world1_fused_paths():
    """NCCL with a single rank on one GPU takes the fused path of every sharding: the node sharding's all-gather
    (bcast_rows for the k = 0 rows, EPI_BCAST hops, the locally stored last hop, the peer-flag fence, forward and backward
    chains), the feature sharding's scatter (EPI_SCATTER) and the 2-D grid's (EPI_GRID), in fp32 and fp64, all in one
    spawned process.  Each runs forward twice (reused arenas), its CUDA-graph replay and backward through part.apply;
    the epilogue kernels must have launched, and y, dh, dx and db are held to the componentwise envelope.  One rank
    hides cross-rank offsets (one peer, row0 = 0): tests/test_peer_epilogues.py covers those with simulated peers."""
    runs = [dict(mode=m, dtype_name=d, G=48, F=24, K=4, backward=True, grid=(1, 1) if m == "grid" else None, trace=True)
            for m in ("nodes", "features", "grid") for d in ("float32", "float64")]
    want = {"nodes": [r"spmm_hop_v2_kernel<[\w,]*,2,1>", r"bcast_rows_kernel<"],
            "features": [r"spmm_hop_v2_kernel<[\w,]*,1,1>"],
            "grid": [r"spmm_hop_v2_kernel<[\w,]*,3,1>", r"bcast_rows_kernel<", r"scatter_rows_kernel<"]}
    import re
    for cfg, out in zip(runs, _spawn("nccl", 1, runs)):
        print("%s %s: arenas %s, kernels %s" % (cfg["mode"], cfg["dtype_name"], out["arenas"], out["kernels"]))
        assert out["fused"]
        for k in want[cfg["mode"]]:
            assert any(re.search(k, n) for n in out["kernels"]), "%s: %s did not launch" % (cfg["mode"], k)
        _hold(out, cfg["dtype_name"], G=48, F=24, K=4)


def test_unpack_tap_grads_is_the_adjoint_of_pack_taps():
    """dh = unpack(dW) must satisfy <dh, h'> = sum_t <dW_t, pack(h')_t> for every h' (the k = 0 tap is shared by all e)."""
    from gnn_b200.distributed import _unpack_tap_grads
    rng = np.random.default_rng(4)
    for (F, E, K, G) in [(3, 1, 1, 2), (2, 2, 3, 4), (4, 3, 2, 1), (1, 1, 5, 3)]:
        T = 1 + E * (K - 1)
        dW = torch.tensor(rng.standard_normal((T, F, G)))
        hp = torch.tensor(rng.standard_normal((F, E, K, G)))
        packed = OracleOps().pack_taps(hp, True)                     # [T, F, G]
        dh = _unpack_tap_grads(dW, E, K)
        assert dh.shape == hp.shape
        assert abs(float((dh * hp).sum() - (dW * packed).sum())) < 1e-10


def test_fused_default_resolution():
    """`fused=None` means: fused whenever the real CUDA ops run under NCCL with <= 16 ranks; explicit choices are kept."""
    from gnn_b200.distributed import resolve_fused
    assert resolve_fused(None, False, "nccl", 2) is True
    assert resolve_fused(None, False, "nccl", 16) is True
    assert resolve_fused(None, False, "nccl", 32) is False          # peer arrays of the kernels hold 16 pointers
    assert resolve_fused(None, False, "gloo", 2) is False
    assert resolve_fused(None, True, "nccl", 2) is False            # injected (CPU stand-in) ops
    assert resolve_fused(True, True, "gloo", 2) is True and resolve_fused(False, False, "nccl", 2) is False
    assert resolve_fused(0, False, "nccl", 2) is False


def test_grid_geometry_host_logic():
    """2-D grid bookkeeping that needs no GPU: the default factorisation, and that the tiles of all ranks tile x exactly
    (rows of the row group, zero padding, features of the column group)."""
    from gnn_b200.distributed import default_grid, PartitionedLSIGF
    assert default_grid(8) == (2, 4) and default_grid(4) == (2, 2) and default_grid(2) == (2, 1) and default_grid(3) == (3, 1)
    N, B, G, P = 203, 2, 16, 8
    Pr, Pc = default_grid(P)
    Rc = (N + P - 1) // P
    x = torch.arange(N * B * G, dtype=torch.float64).reshape(N, B * G)
    covered = torch.zeros(Rc * P, B, G)
    for rank in range(P):
        part = PartitionedLSIGF.__new__(PartitionedLSIGF)          # geometry only: no process group, no plan
        part.Pr, part.Pc, part.rg, part.cg = Pr, Pc, rank // Pc, rank % Pc
        part.rows_per_rank, part.rows_per_group, part.n_pad = Rc, Rc * Pc, Rc * P
        tile = part.grid_tile(x, B, G)
        Gl = G // Pc
        assert tuple(tile.shape) == (Rc * Pc, B * Gl)
        r0 = part.rg * Rc * Pc
        covered[r0:r0 + Rc * Pc, :, part.cg * Gl:(part.cg + 1) * Gl] += tile.view(Rc * Pc, B, Gl)
    assert torch.equal(covered[:N].reshape(N, B * G), x) and float(covered[N:].abs().max()) == 0.0
