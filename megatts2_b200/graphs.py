"""CUDA-graph replay of the device-only autoregressive drivers (MegaPLM.infer / MegaADM.infer).

One AR decode is ~3-7 thousand kernel launches whose arguments depend only on (weights, B, T) and on buffers this module
owns: the first call with a given key runs eagerly (it also builds the plans, descriptors and attributes), the second
captures the same enqueue sequence - programmatic-dependent-launch edges included - into a ``torch.cuda.CUDAGraph``, later
calls copy the input into the graph's static buffer and replay it.  The launch sequence is identical, so results are
bit-identical to the eager path (checked by tests/test_gpu_parity.py::test_graph_replay_matches_eager).

``MEGATTS2_GRAPHS=0`` or ``graphs.disabled()`` (profiling legs that record events between launches) keep everything eager."""
import contextlib
import os

import torch

_enabled = os.environ.get("MEGATTS2_GRAPHS", "1") != "0"
_off_depth = 0
replayed_launches = 0   # kernel nodes executed by graph replays (the library's own counter only sees eager enqueues)
MAX_GRAPHS = 8          # per owner: a graph pins its workspace (hundreds of MB at batch 64)


def enabled() -> bool:
    return _enabled and _off_depth == 0


@contextlib.contextmanager
def disabled():
    global _off_depth
    _off_depth += 1
    try:
        yield
    finally:
        _off_depth -= 1


class GraphedCall:
    """Per-owner cache: key -> ('warm',) after the first eager call, then (graph, static inputs, static outputs)."""

    def __init__(self):
        self.cache = {}

    def clear(self):
        self.cache.clear()

    def run(self, key, inputs, fn):
        """fn(*inputs) -> tuple of tensors; enqueues device work only (no host sync, no data-dependent host control)."""
        if not enabled() or torch.cuda.is_current_stream_capturing():
            return fn(*inputs)
        e = self.cache.get(key)
        if e is None:
            if len(self.cache) >= MAX_GRAPHS:
                self.cache.pop(next(iter(self.cache)))
            self.cache[key] = ("warm",)
            return fn(*inputs)
        if e[0] == "warm":
            static_in = tuple(t.clone() for t in inputs)
            g = torch.cuda.CUDAGraph()
            from . import ops
            n0 = ops._lib_launch_count()
            try:
                # thread_local: other threads of the process (an NCCL watchdog, a data loader) may call CUDA freely
                with torch.cuda.graph(g, capture_error_mode="thread_local"):
                    static_out = fn(*static_in)
            except Exception:
                self.cache[key] = ("eager",)      # capture not possible here (e.g. an allocator or driver restriction)
                torch.cuda.synchronize()
                return fn(*inputs)
            # the captured kernels address the scratch buffers ops.workspace handed out: the graph keeps them alive, since
            # a later, larger call replaces them there and the allocator would otherwise reuse their memory
            g.workspaces = ops.workspace_buffers()
            e = (g, static_in, static_out, ops._lib_launch_count() - n0)
            self.cache[key] = e
        elif e[0] == "eager":
            return fn(*inputs)
        global replayed_launches
        g, static_in, static_out, n_kernels = e
        for s, t in zip(static_in, inputs):
            if s.data_ptr() != t.data_ptr():
                s.copy_(t)
        g.replay()
        replayed_launches += n_kernels
        return tuple(o.clone() for o in static_out)
