"""The lifecycle every inference engine shares: when its packed copies of a module's weights are rebuilt, and what a deep copy keeps.

Packed copies are rebuilt before the next call after `load_state_dict`, `.to()` / `.cuda()`, or an in-place update of any parameter or buffer
(optimizer steps, EMA, in-place ops under `no_grad`): each of these changes a tensor's storage pointer or its version counter.  A write through
`.data` (`p.data.copy_(...)`) changes neither: call `engine.repack()` after one.
"""
from __future__ import annotations

import copy

import torch
from torch import nn


class PackedEngine:
    """Subclasses implement _pack(): build the packed copies from self.m and drop every workspace, captured graph and cached result."""

    settings = ()  # attributes a caller may change after construction; a deep copy keeps them

    def __init__(self, module, **options):
        self.m = module
        self.options = options  # the subclass's constructor arguments, so that a deep copy is built the same way
        self.packed = False
        self.generation = 0  # bumped by repack(): graphs captured outside the engine compare it to know they are stale
        self._sig = None

    def signature(self):
        """(storage pointer, version counter) of every parameter and buffer of the module."""
        return tuple((t.data_ptr(), t._version) for t in (*self.m.parameters(), *self.m.buffers()))

    def ensure_current(self) -> None:
        if not self.packed or self._sig != self.signature():
            self.repack()

    @torch.no_grad()
    def repack(self) -> None:
        """(Re)build the packed copies from the module's current weights."""
        self._pack()
        self._sig = self.signature()
        self.packed = True
        self.generation += 1

    def _pack(self) -> None:
        raise NotImplementedError

    def __deepcopy__(self, memo):
        """copy.deepcopy(module) (the reference EMA's shadow model) gets a fresh, unpacked engine bound to the copied module: packed weights,
        workspaces and captured CUDA graphs are per-instance caches, not state."""
        new = type(self)(memo.get(id(self.m), self.m), **self.options)
        for k in self.settings:
            setattr(new, k, copy.deepcopy(getattr(self, k), memo))
        return new


class EngineModule(nn.Module):
    """A module whose compute runs in PackedEngine attributes.  After `.to()` / `.cuda()` / `.cpu()` its engines repack: the caching allocator
    can hand a moved tensor the address it had before, with version 0, so the signature alone could miss the move."""

    def _apply(self, fn, *a, **k):
        out = super()._apply(fn, *a, **k)
        for v in vars(self).values():
            if isinstance(v, PackedEngine):
                v.packed = False
        return out
