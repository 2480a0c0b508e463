"""One CUDA graph for a whole inference call (SURVEY.md §8 f-2: the static-GSO GRNN time loop, graphML.py:1455-1527).

The reference's recurrent layers issue one small LSIGF per time step (graphML.py:1461); at N = 50..1000 nodes each step is
a handful of microsecond kernels, so a sequence of T steps is bound by launch latency and Python, not by the GPU.  Every
kernel of this library is enqueued on the caller's stream without host synchronisation or allocation
(include/b200gf.h) — so the complete T-step recursion, filters, gates and non-linearities included, can be captured once
and replayed as ONE graph launch.

    run = gnn_b200.graphed(layer, x_example, z0_example)      # warm-up + capture (inference: no autograd inside)
    z, zT = run(x, z0)                                        # copies into the static inputs, replays, returns the
                                                              # static outputs (valid until the next call)
Plumbing only (torch.cuda.CUDAGraph); the arithmetic is the same kernels in the same order as the eager call, so the
results are bit-identical (tests/test_widen_recurrent.py::test_graphed_grnn_matches_eager).
"""
import torch


class GraphedForward:
    def __init__(self, fn, *example_inputs, warmup=2):
        if not example_inputs or not all(isinstance(t, torch.Tensor) and t.is_cuda for t in example_inputs):
            raise RuntimeError("b200gf: graphed() needs CUDA tensor example inputs (there is no CPU path)")
        self.fn = fn
        self.static_in = [t.detach().clone() for t in example_inputs]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side), torch.no_grad():
            for _ in range(max(1, warmup)):                   # plans, function attributes, tensor-map encoder: all cached now
                fn(*self.static_in)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.no_grad(), torch.cuda.graph(self.graph):
            self.static_out = fn(*self.static_in)

    def __call__(self, *inputs):
        assert len(inputs) == len(self.static_in)
        for dst, src in zip(self.static_in, inputs):
            if dst.data_ptr() != src.data_ptr():
                dst.copy_(src)
        self.graph.replay()
        return self.static_out


def graphed(fn, *example_inputs, warmup=2):
    """Capture `fn(*example_inputs)` (any composition of this package's layers and element-wise torch ops, inference
    only) into one CUDA graph; returns a callable with the same signature that replays it."""
    return GraphedForward(fn, *example_inputs, warmup=warmup)
