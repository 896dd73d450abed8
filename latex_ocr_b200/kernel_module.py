"""The autograd bridge of the kernel-backed modules (EncoderCNN, Attention, DecoderWithAttention, tf_decoder.Decoder,
RowEncoder, TwoLayerDecoder): one autograd node for all of them, and the rule that makes the backward of an overwritten forward
refuse to run.

A module implements
  ``_forward_impl(*args, need_grad)`` -> (differentiable outputs (tuple), non-differentiable side outputs, saved)
      ``saved`` (None without ``need_grad``) is what the backward needs.  Its optional ``"entries"`` are the cache entries the
      forward wrote and stamped (``stamp``); its optional ``"tensors"`` go through ``ctx.save_for_backward``, so that torch
      refuses a backward after one of them was modified in place, and come back as ``saved["tensors"]``.
  ``_backward_impl(saved, *d_outputs, need)`` -> gradients of the differentiable inputs
      ``need``: which of the differentiable inputs, then which of the parameters, need a gradient.  The kernels write the
      parameter gradients into the flat ``store.grad`` buffers.  A ``d_output`` is None when the loss does not use that output.
"""
import itertools

import torch

from ._lib import LatexOcrB200Error
from .params import kernel_grads

_stamps = itertools.count(1)


def stamp(entry):
    """Mark a cache entry (a dict) as rewritten by a forward.  One counter serves every cache, so a re-created entry never
    repeats a stamp."""
    entry["gen"] = next(_stamps)
    return entry


class KernelFunction(torch.autograd.Function):
    """Autograd node of a kernel-backed module's forward.  Inputs: (module, dict receiving the side outputs, the forward's
    arguments, the number of differentiable inputs, the differentiable inputs, the module's parameters)."""

    @staticmethod
    def forward(ctx, mod, side, args, n_inputs, *tensors):
        outs, side["out"], saved = mod._forward_impl(*args, need_grad=True)
        ctx.mod, ctx.n_inputs, ctx.params = mod, n_inputs, tensors[n_inputs:]
        ctx.stamps = [(e, e["gen"]) for e in saved.pop("entries", ())]
        ctx.save_for_backward(*saved.pop("tensors", ()))
        ctx.saved = saved
        ctx.set_materialize_grads(False)          # an output the loss does not use arrives as None
        return outs

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, *douts):
        mod = ctx.mod
        if any(e["gen"] != g for e, g in ctx.stamps):
            raise LatexOcrB200Error("%s backward: the saved forward state was overwritten by a later forward of the same shape; "
                                    "run backward before the next such forward" % type(mod).__name__)
        need = ctx.needs_input_grad[4:]
        n = ctx.n_inputs
        saved = dict(ctx.saved, tensors=ctx.saved_tensors)
        dinputs, grads = kernel_grads(ctx.params, need[n:], lambda: mod._backward_impl(saved, *douts, need))
        return (None, None, None, None) + tuple(d if nd else None for d, nd in zip(dinputs, need[:n])) + tuple(grads)


def kernel_forward(mod, args, inputs):
    """``mod``'s forward on ``args``: returns (differentiable outputs, side outputs) of ``mod._forward_impl``.  ``inputs``: the
    differentiable ones among ``args``.  With grad mode on and one of them or a parameter requiring grad, an autograd graph is
    recorded (KernelFunction); otherwise the forward runs under ``no_grad``.  The outputs are the same either way."""
    if not inputs[0].is_cuda:
        raise LatexOcrB200Error("%s runs on CUDA tensors only (no CPU fallback)" % type(mod).__name__)
    params = list(mod.parameters())
    if torch.is_grad_enabled() and any(t.requires_grad for t in itertools.chain(inputs, params)):
        side = {}
        outs = KernelFunction.apply(mod, side, args, len(inputs), *inputs, *params)
        return outs, side["out"]
    with torch.no_grad():
        return mod._forward_impl(*args, need_grad=False)[:2]
