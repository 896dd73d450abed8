"""Flat parameter storage: one fp32 master buffer (+ gradient, Adam moments and, in bf16 mode, a
bf16 shadow in the same element order) per module, with the reference's ``state_dict`` names as
views.  One buffer -> one fused Adam launch and one NCCL all-reduce bucket per module."""
import torch
import torch.nn as nn

import os
from collections import OrderedDict


class LRUCache(OrderedDict):
    """Bounded shape-keyed cache for workspaces / captured CUDA graphs.  Real data gives a different (batch, max formula
    length, image bucket) on nearly every batch; an unbounded per-shape cache would grow by tens to hundreds of MB per
    distinct key over an epoch.  Least-recently-used entries are dropped (their tensors return to torch's caching
    allocator, so a re-created workspace of a recurring shape costs no cudaMalloc)."""

    def __init__(self, maxsize=None):
        super().__init__()
        self.maxsize = int(maxsize if maxsize is not None else os.environ.get("LO_WS_CACHE", "4"))

    def get(self, key, default=None):
        if key in self:
            self.move_to_end(key)
            return super().__getitem__(key)
        return default

    def __setitem__(self, key, value):
        super().__setitem__(key, value)
        self.move_to_end(key)
        while len(self) > max(1, self.maxsize):
            self.popitem(last=False)


ALIGN = 8  # elements: 32 B in fp32, 16 B in bf16 (vector-load alignment of the kernels)


class FlatStore:
    def __init__(self, specs, device, bf16_shadow):
        """specs: list of (name, storage_shape)."""
        self.device = torch.device(device)
        self.specs = list(specs)
        self.offsets = {}
        off = 0
        for name, shape in self.specs:
            n = 1
            for s in shape:
                n *= s
            self.offsets[name] = (off, n, tuple(shape))
            off += (n + ALIGN - 1) // ALIGN * ALIGN
        self.numel = off
        self.master = torch.zeros(off, dtype=torch.float32, device=self.device)
        self.grad = torch.zeros(off, dtype=torch.float32, device=self.device)
        self.m = None
        self.v = None
        self.shadow = torch.zeros(off, dtype=torch.bfloat16, device=self.device) if bf16_shadow else None
        self.adam_state = None   # device float[2]: step, lr
        self._shadow_version = None   # master._version the shadow was last cast from (None: never, or stale)

    def view(self, buf, name):
        off, n, shape = self.offsets[name]
        return buf[off:off + n].view(shape)

    def w(self, name):
        """Kernel-facing weight storage (bf16 shadow in bf16 mode, the fp32 master otherwise)."""
        return self.view(self.shadow if self.shadow is not None else self.master, name)

    def f32(self, name):
        return self.view(self.master, name)

    def g(self, name):
        return self.view(self.grad, name)

    def ensure_adam(self, lr):
        if self.m is None:
            self.m = torch.zeros_like(self.master)
            self.v = torch.zeros_like(self.master)
            self.adam_state = torch.tensor([0.0, float(lr)], dtype=torch.float32, device=self.device)

    def set_lr(self, lr):
        self.adam_state[1] = float(lr)

    def sync_shadow(self):
        """Re-cast the bf16 shadow from the fp32 master (e.g. after the master was written behind torch's back by NCCL)."""
        if self.shadow is not None:
            self.shadow.copy_(self.master)   # plumbing cast (fp32 -> bf16, round-to-nearest-even)
        self._shadow_version = self.master._version

    def refresh_shadow(self):
        """Re-cast the shadow if the master changed since the last cast; every kernel-backed forward calls this.  In-place edits
        of the parameters (``p.mul_``, ``load_state_dict``, ``torch.optim`` steps) move the version counter that the parameter
        views share with ``master``.  The fused optimisers write the shadow themselves and leave the counter alone."""
        if self._shadow_version != self.master._version:
            self.sync_shadow()

    def mark_shadow_current(self):
        """Master and shadow were just written together (restored from a snapshot): the shadow needs no re-cast."""
        self._shadow_version = self.master._version

    def to_(self, device):
        device = torch.device(device)
        if device == self.device:
            return
        for k in ("master", "grad", "m", "v", "shadow", "adam_state"):
            t = getattr(self, k)
            if t is not None:
                setattr(self, k, t.to(device))
        self.device = device
        self._shadow_version = None


class ParamHolder(nn.Module):
    """A leaf with reference-named parameters that are views into a FlatStore."""

    def __init__(self):
        super().__init__()

    def bind(self, pname, store, sname, permute=None):
        v = store.view(store.master, sname)
        gv = store.view(store.grad, sname)
        if permute is not None:
            v = v.permute(*permute)
            gv = gv.permute(*permute)
        p = nn.Parameter(v, requires_grad=True)
        p.grad = gv
        p._lo_store = store
        p._lo_store_name = sname
        p._lo_permute = permute
        self.register_parameter(pname, p)


def grad_view(store, p):
    """The slice of ``store.grad`` that holds parameter ``p``'s gradient, in ``p``'s shape."""
    gv = store.view(store.grad, p._lo_store_name)
    return gv.permute(*p._lo_permute) if p._lo_permute is not None else gv


def bind_grads(module, store):
    """Point every parameter's ``.grad`` at its slice of ``store.grad``, which the fused train step overwrites: after that step
    ``p.grad`` reads its gradients.  A no-op when they already point there."""
    base = store.grad.data_ptr()
    for p in module.parameters():
        if p.grad is None or p.grad.data_ptr() != base + 4 * store.offsets[p._lo_store_name][0]:
            p.grad = grad_view(store, p)


def kernel_grads(params, need, backward):
    """Runs ``backward()``, whose kernels write the gradients of ``params`` (from one or several stores) into their stores' flat
    ``grad`` buffers, and returns (its result, [a copy of the gradient of each parameter, None where ``need`` is false]).  Every
    ``p.grad`` that aliases a store's buffer first gets memory of its own (same values), so what autograd has accumulated there
    survives the kernels."""
    for p in params:
        if p.grad is not None and p.grad.untyped_storage().data_ptr() == p._lo_store.grad.untyped_storage().data_ptr():
            p.grad = p.grad.clone()
    out = backward()
    return out, [grad_view(p._lo_store, p).clone() if n else None for p, n in zip(params, need)]
