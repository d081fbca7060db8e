"""CUDA-graph capture: one warm-up-then-capture sequence, and a tiny cache that replays a fixed-shape launch sequence with fresh inputs copied
into static buffers."""
from __future__ import annotations

import torch


def capture(step, device=None) -> torch.cuda.CUDAGraph:
    """Run step() once on a side stream, then capture it: lazy initialisation (function attributes, weight packing, workspaces) happens in the
    warm-up, so the captured launch sequence is the steady-state one.  The capture itself executes nothing."""
    s = torch.cuda.Stream(device=device)
    s.wait_stream(torch.cuda.current_stream(device))
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream(device).wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    return g


class GraphCache:
    def __init__(self):
        self._entries = {}

    def clear(self):
        self._entries.clear()

    def run(self, key, fn, *inputs):
        """fn(*static_inputs) -> tensor (or tuple of tensors) built only from stream-ordered work; inputs must keep shape/dtype per key."""
        ent = self._entries.get(key)
        if ent is None:
            static_in = [t.clone() for t in inputs]
            out = []
            g = capture(lambda: out.append(fn(*static_in)))
            ent = (g, static_in, out[-1])  # the captured call's outputs
            self._entries[key] = ent
        g, static_in, static_out = ent
        for dst, src in zip(static_in, inputs):
            dst.copy_(src)
        g.replay()
        if isinstance(static_out, (tuple, list)):
            return type(static_out)(o.clone() for o in static_out)
        return static_out.clone()
