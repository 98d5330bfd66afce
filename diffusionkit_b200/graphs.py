"""Per-input-shape state and CUDA-graph replay, shared by the MMDiT and the VAE decoder.

A captured graph bakes in the device pointers of every buffer its forward touched, so each input shape owns one state
dict holding its graph together with whatever buffers the forward keeps between calls (workspaces, tables).  The dicts
sit in an LRU bounded by DK_MAX_CACHED_SHAPES (default 4): evicting a shape drops its graph and its buffers together,
so a graph never outlives what it points at.  DK_CUDA_GRAPHS=0 runs every forward eagerly, kernel by kernel.
Both settings become attributes of each model (`use_cuda_graphs`, `max_cached_shapes`), which a caller may change
between calls.
"""
from __future__ import annotations

import os
from collections import OrderedDict

import torch

from . import ops


def default_settings():
    """(use CUDA graphs, number of input shapes to keep) from DK_CUDA_GRAPHS and DK_MAX_CACHED_SHAPES"""
    return os.environ.get("DK_CUDA_GRAPHS", "1") != "0", int(os.environ.get("DK_MAX_CACHED_SHAPES", "4"))


class ShapeCache:
    def __init__(self):
        self._states: "OrderedDict[tuple, dict]" = OrderedDict()

    def __len__(self) -> int:
        return len(self._states)

    def state(self, key: tuple, max_shapes: int) -> dict:
        """The state dict of input shape `key`, created empty if new (evicting least recently used shapes so that at
        most `max_shapes` remain)."""
        st = self._states.get(key)
        if st is None:
            while len(self._states) >= max(1, max_shapes):
                self._states.popitem(last=False)
            st = self._states[key] = {}
        else:
            self._states.move_to_end(key)
        return st

    def drop(self, name: str):
        """Forget entry `name` of every shape's state, and the entries "name.<part>" with it, and keep the rest."""
        for st in self._states.values():
            for key in [k for k in st if k == name or k.startswith(name + ".")]:
                del st[key]

    def drop_graphs(self):
        """Forget every captured graph but keep the buffers (for when an input the graphs read moves)."""
        self.drop("graph")

    def run(self, st: dict, use_graphs: bool, fn, *inputs: torch.Tensor, name: str = "graph",
            stateful: bool = False, device=None):
        """fn(*inputs), eagerly or by replaying the graph kept in `st[name]`.  With graphs on, the first call for a shape
        runs fn eagerly on static copies of the inputs (workspaces, tables, function attributes, allocator), then
        captures it; every replay copies the inputs into those copies and returns the same output tensor.
        stateful: fn updates buffers it also reads, so running it twice is not running it once; the first call returns
        the eager pass's output and the capture is not replayed until the next call.  A graph named "graph.<part>" is
        one part of a forward and is dropped with "graph".  device: where fn runs when it takes no inputs."""
        if not use_graphs:
            return fn(*inputs)
        entry = st.get(name)
        if entry is None:
            static = [t.clone() for t in inputs]
            first = fn(*static)
            torch.cuda.current_stream(static[0].device if static else device).synchronize()
            n0 = ops.launch_count()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                out = fn(*static)
            st[name] = (graph, static, out, ops.launch_count() - n0)
            if stateful:
                return first
            entry = st[name]
        graph, static, out, n_launch = entry
        for s, t in zip(static, inputs):
            s.copy_(t)
        graph.replay()
        ops.note_graph_launches(n_launch)
        return out
