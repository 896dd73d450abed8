"""EncoderCNN — drop-in for model/components/seq2seq_torch.py:24-157 ('vanilla' stack) running on
hand-written sm_90a kernels through the C ABI.  Same constructor, ``forward(img[N,1,H,W]) ->
[N,H',W',512]``, ``fine_tune`` and ``state_dict`` keys ``cnn.{0,3,6,8,11,14}.{weight,bias}``.

Layout in HBM: feature maps NHWC, conv weights [Cout][3][3][Cin] (exposed to ``state_dict`` as OIHW
views of the same memory).  ``precision='fp32'`` runs every kernel in fp32 (tight-parity mode);
``'bf16'`` stores feature maps / weight shadows in bf16 with fp32 accumulation.
"""
import math

import torch
import torch.nn as nn

from . import _lib
from ._lib import check, dtype_code, impl_code, ptr, stream_ptr
from .kernel_module import kernel_forward, stamp
from .params import FlatStore, LRUCache, ParamHolder

# (sequential index, Cin, Cout, pad, pool after)    seq2seq_torch.py:35-56
_LAYERS = (("0", 1, 64, 1, (2, 2)), ("3", 64, 128, 1, (2, 2)), ("6", 128, 256, 1, None),
           ("8", 256, 256, 1, (2, 1)), ("11", 256, 512, 1, (1, 2)), ("14", 512, 512, 0, None))
# 'cnn' variant (seq2seq_torch.py:58-86): the two asymmetric pools are replaced by Conv2d(512,512,(2,4),stride 2,padding 1)+ReLU
# (index 12; a 6th tuple element gives kernel (R,S) and stride of a non-3x3 layer, run as im2col + GEMM)
_LAYERS_CNN = (("0", 1, 64, 1, (2, 2)), ("3", 64, 128, 1, (2, 2)), ("6", 128, 256, 1, None), ("8", 256, 256, 1, None),
               ("10", 256, 512, 1, None), ("12", 512, 512, 1, None, (2, 4, 2)), ("14", 512, 512, 0, None))


def _geom(layer):
    """(R, S, stride) of a layer tuple."""
    return layer[5] if len(layer) > 5 else (3, 3, 1)


def timing_signal_table(channels, height, width, device):
    """add_timing_signal_nd_torch (seq2seq_torch.py:115-157) as an [H][W][C] fp32 table.  Host-side
    constant built with the same torch ops as the reference (sin/cos of arange*inv_timescales)."""
    nts = channels // 4
    inc = math.log(1.0e4 / 1.0) / (float(nts) - 1)
    inv = 1.0 * torch.exp(torch.arange(nts).float() * (-inc))
    table = torch.zeros(channels, height, width)
    for dim, length in enumerate((height, width)):
        st = inv.unsqueeze(1) * torch.arange(length).float().unsqueeze(0)
        sig = torch.cat([torch.sin(st), torch.cos(st)], dim=0)
        lo = dim * 2 * nts
        table[lo:lo + 2 * nts] += sig[:, :, None] if dim == 0 else sig[:, None, :]
    return table.permute(1, 2, 0).contiguous().to(device)


class EncoderCNN(nn.Module):
    def __init__(self, config, training=False, device="cuda", precision=None, impl=None):
        super().__init__()
        self._config = config
        name = getattr(config, "encoder_cnn", "vanilla")
        if name not in ("vanilla", "cnn"):
            raise NotImplementedError("encoder_cnn=%r: 'vanilla' and 'cnn' are the reference's stacks" % name)   # seq2seq_torch.py:31-86
        self.layers = _LAYERS if name == "vanilla" else _LAYERS_CNN
        self.precision = precision or getattr(config, "precision", "bf16")
        if self.precision not in ("fp32", "bf16"):
            raise NotImplementedError("precision must be 'fp32' or 'bf16'")
        self.impl = impl if impl is not None else getattr(config, "conv_impl", "tc" if self.precision == "bf16" else "simt")
        self.tdtype = torch.float32 if self.precision == "fp32" else torch.bfloat16
        # pixel normalisation fused into conv1: None = raw 0..255 floats (torch flavour, img2seq_torch.py:115-117);
        # "tf" = (img - 128) / 128 (TF flavour, model/encoder.py:26-27)
        self.input_norm = getattr(config, "input_norm", None)
        if self.input_norm not in (None, "tf"):
            raise NotImplementedError("input_norm=%r" % (self.input_norm,))
        specs = []
        for l in self.layers:
            idx, cin, cout = l[:3]
            R, S_, _ = _geom(l)
            specs.append(("cnn.%s.weight" % idx, (cout, R, S_, cin)))
            specs.append(("cnn.%s.bias" % idx, (cout,)))
        self.store = FlatStore(specs, device, bf16_shadow=(self.precision == "bf16"))
        self.cnn = nn.ModuleDict()
        for idx in (l[0] for l in self.layers):
            h = ParamHolder()
            h.bind("weight", self.store, "cnn.%s.weight" % idx, permute=(0, 3, 1, 2))
            h.bind("bias", self.store, "cnn.%s.bias" % idx)
            self.cnn[idx] = h
        self.reset_parameters()
        self._ws = LRUCache()     # bounded: see params.LRUCache

    # nn.Conv2d default init (kaiming_uniform(a=sqrt(5)) == U(-1/sqrt(fan_in), 1/sqrt(fan_in)))
    def reset_parameters(self):
        with torch.no_grad():
            for l in self.layers:
                idx, cin = l[0], l[1]
                R, S_, _ = _geom(l)
                b = 1.0 / math.sqrt(cin * R * S_)
                self.cnn[idx].weight.uniform_(-b, b)
                self.cnn[idx].bias.uniform_(-b, b)

    def fine_tune(self, fine_tune=True):
        """seq2seq_torch.py:102-113."""
        for p in self.cnn.parameters():
            p.requires_grad = False
        for idx in list(self.cnn.keys())[2:]:      # children()[5:] of the Sequential == convs from index 6 on
            for p in self.cnn[idx].parameters():
                p.requires_grad = fine_tune

    def out_hw(self, H, W):
        h, w = H, W
        for l in self.layers:
            pad, pool = l[3], l[4]
            R, S_, stride = _geom(l)
            h, w = (h + 2 * pad - R) // stride + 1, (w + 2 * pad - S_) // stride + 1
            if pool:
                h, w = h // pool[0], w // pool[1]
        return h, w

    # ---------------------------------------------------------------------------------------------
    def _workspace(self, N, H, W, need_grad):
        key = (N, H, W)
        ws = self._ws.get(key)
        if ws is None:
            dev, td = self.store.device, self.tdtype
            ws = {"acts": {}, "grads": None}
            h, w = H, W
            shapes = {}
            for l in self.layers:
                idx, cin, cout, pad, pool = l[:5]
                R, S_, stride = _geom(l)
                if (R, S_, stride) != (3, 3, 1):
                    ws["col" + idx] = torch.empty(N * ((h + 2 * pad - R) // stride + 1) * ((w + 2 * pad - S_) // stride + 1), R * S_ * cin,
                                                  dtype=td, device=dev)
                h, w = (h + 2 * pad - R) // stride + 1, (w + 2 * pad - S_) // stride + 1
                if idx == "0":
                    h, w = h // 2, w // 2
                    shapes["P0"] = (N, h, w, cout)
                    continue
                shapes["Y" + idx] = (N, h, w, cout)
                if pool:
                    h, w = h // pool[0], w // pool[1]
                    shapes["P" + idx] = (N, h, w, cout)
            if h < 1 or w < 1:
                raise ValueError("image %dx%d too small for the vanilla encoder" % (H, W))
            ws["shapes"] = shapes
            for k, s in shapes.items():
                ws["acts"][k] = torch.empty(s, dtype=td, device=dev)
            ws["out"] = torch.empty(shapes["Y14"], dtype=td, device=dev)
            ws["table"] = timing_signal_table(512, shapes["Y14"][1], shapes["Y14"][2], dev)
            self._ws[key] = ws
        if need_grad and ws["grads"] is None:
            dev, td = self.store.device, self.tdtype
            ws["grads"] = {k: torch.empty(s, dtype=td, device=dev) for k, s in ws["shapes"].items()}
            ws["wflip"] = {l[0]: torch.empty(l[1] * _geom(l)[0] * _geom(l)[1] * l[2], dtype=td, device=dev)
                           for l in self.layers if l[0] != "0"}
        return ws

    def _impl(self):
        return impl_code(self.impl, self.precision)

    def forward_raw(self, img, need_grad=False):
        """img: CUDA float32 or uint8 [N,1,H,W] (raw 0..255 like img2seq_torch.py:115-117; uint8 = 4x less H2D traffic).  Returns the
        encoder output in storage dtype [N,H',W',512] (a workspace buffer, overwritten by the next call)."""
        L = _lib.lib()
        if img.dim() != 4 or img.size(1) != 1:
            raise ValueError("img must be [N,1,H,W]")
        if not img.is_cuda:
            raise _lib.LatexOcrB200Error("EncoderCNN runs on CUDA tensors only (no CPU fallback)")
        if img.dtype != torch.uint8:
            img = img.float()
        img = img.contiguous()
        N, _, H, W = img.shape
        ws = stamp(self._workspace(N, H, W, need_grad))     # this call overwrites the forward state of a pending backward
        self.store.refresh_shadow()
        st, dt, impl, S = stream_ptr(), dtype_code(self.precision), self._impl(), self.store
        A = ws["acts"]
        ws["img"] = img
        sc, of = (1.0 / 128.0, -1.0) if self.input_norm == "tf" else (1.0, 0.0)
        if need_grad:
            # training: conv1 also stores the pool arg-max / ReLU code per output (1 byte) for its weight-gradient kernel
            if ws.get("code0") is None:
                ws["code0"] = torch.empty(A["P0"].shape, dtype=torch.uint8, device=img.device)
            check(L.lo_conv1_pool_forward_code(ptr(img), int(img.dtype == torch.uint8), sc, of, ptr(S.f32("cnn.0.weight")),
                                               ptr(S.f32("cnn.0.bias")), ptr(A["P0"]), ptr(ws["code0"]), dt, N, H, W, st))
        elif self.input_norm == "tf":
            check(L.lo_conv1_pool_forward_norm(ptr(img), int(img.dtype == torch.uint8), 1.0 / 128.0, -1.0, ptr(S.f32("cnn.0.weight")),
                                               ptr(S.f32("cnn.0.bias")), ptr(A["P0"]), dt, N, H, W, st))
        else:
            conv1 = L.lo_conv1_pool_forward_u8 if img.dtype == torch.uint8 else L.lo_conv1_pool_forward
            check(conv1(ptr(img), ptr(S.f32("cnn.0.weight")), ptr(S.f32("cnn.0.bias")), ptr(A["P0"]), dt, N, H, W, st))
        x = A["P0"]
        for l in self.layers[1:]:
            idx, cin, cout, pad, pool = l[:5]
            R, S_, stride = _geom(l)
            y = A["Y" + idx]
            if (R, S_, stride) == (3, 3, 1):
                check(L.lo_conv3x3(ptr(x), ptr(S.w("cnn.%s.weight" % idx)), ptr(S.f32("cnn.%s.bias" % idx)), None, ptr(y), dt,
                                   N, x.shape[1], x.shape[2], cin, cout, pad, 1, impl, st))
            else:
                # general strided conv: im2col + GEMM with bias + ReLU in the epilogue
                col = ws["col" + idx]
                M, K = col.shape
                check(L.lo_im2col(ptr(x), ptr(col), dt, N, x.shape[1], x.shape[2], cin, R, S_, stride, pad, st))
                check(L.lo_gemm(ptr(col), dt, ptr(S.w("cnn.%s.weight" % idx)), dt, ptr(y), dt, M, cout, K, K, 1, 1, K, cout, 1, 0, 0, 0,
                                ptr(S.f32("cnn.%s.bias" % idx)), 0, 1, impl, st))
            x = y
            if pool:
                p = A["P" + idx]
                check(L.lo_maxpool_forward(ptr(y), ptr(p), dt, N, y.shape[1], y.shape[2], cout, pool[0], pool[1], st))
                x = p
        if getattr(self._config, "positional_embeddings", True):
            hwc = x.shape[1] * x.shape[2] * x.shape[3]
            check(L.lo_add_table(ptr(x), ptr(ws["table"]), ptr(ws["out"]), dt, N, hwc, st))
            return ws["out"]
        return x

    def grad_range(self, idx):
        """(offset, count) of layer ``idx``'s [weight, bias] gradient inside the flat store (contiguous by construction)."""
        ow, nw, _ = self.store.offsets["cnn.%s.weight" % idx]
        ob, nb, _ = self.store.offsets["cnn.%s.bias" % idx]
        return ow, ob + nb - ow

    def backward_raw(self, img_shape, denc, on_layer_grad=None, ws=None, dimg=None):
        """denc: fp32 [N,H',W',512] gradient w.r.t. the encoder output.  Fills self.store.grad.  ``on_layer_grad(idx)`` is
        called right after the kernels that complete layer idx's weight/bias gradient have been enqueued (last conv first):
        the data-parallel path fires that layer's gradient all-reduce there, overlapping the rest of the backward.  ``ws``: the
        workspace of the forward (default: the cached one of this image shape).  ``dimg``: an fp32 CUDA tensor of N*H*W
        elements that receives the gradient w.r.t. the image (written, not accumulated); it needs the arg-max codes of a training
        forward (``forward_raw(..., need_grad=True)``).  Without it, no image gradient is computed."""
        L = _lib.lib()
        N, _, H, W = img_shape
        ws = ws if ws is not None else self._workspace(N, H, W, True)
        if dimg is not None:
            if ws.get("code0") is None:
                raise _lib.LatexOcrB200Error("EncoderCNN.backward_raw: the image gradient needs the arg-max codes of a training "
                                             "forward (forward_raw(img, need_grad=True)); this workspace has none")
            if dimg.dtype != torch.float32 or not dimg.is_contiguous() or dimg.numel() != N * H * W:
                raise ValueError("dimg must be a contiguous float32 tensor of N*H*W elements")
        st, dt, impl, S = stream_ptr(), dtype_code(self.precision), self._impl(), self.store
        A, G = ws["acts"], ws["grads"]
        for l in self.layers[1:]:
            idx, cin, cout = l[:3]
            R, S_, stride = _geom(l)
            if (R, S_, stride) == (3, 3, 1):
                check(L.lo_conv_weight_flip(ptr(S.w("cnn.%s.weight" % idx)), ptr(ws["wflip"][idx]), dt, cin, cout, st))
            else:                                           # [Cout][K] -> [K][Cout] for dcol = dy @ W
                check(L.lo_transpose(ptr(S.w("cnn.%s.weight" % idx)), R * S_ * cin, ptr(ws["wflip"][idx]), cout, dt, cout, R * S_ * cin, st))
        last = "Y" + self.layers[-1][0]
        y6 = A[last]
        check(L.lo_relu_mask_cast(ptr(denc), ptr(y6), ptr(G[last]), dt, y6.numel(), st))
        # walk the stack backwards: (layer, key of its input activation = the previous layer's pooled or plain output)
        plan = []
        for i in range(len(self.layers) - 1, 0, -1):
            prev = self.layers[i - 1]
            plan.append((self.layers[i], ("P" if prev[4] else "Y") + prev[0]))
        cfg = {l[0]: l for l in self.layers}
        for l, xin in plan:
            idx, cin, cout, pad, pool = l[:5]
            R, S_, stride = _geom(l)
            x = A[xin]
            dy = G["Y" + idx]
            mask = A[xin] if xin.startswith("Y") else None   # ReLU mask fused when the producer is a conv
            if (R, S_, stride) == (3, 3, 1):
                check(L.lo_conv3x3_wgrad(ptr(x), ptr(dy), ptr(S.g("cnn.%s.weight" % idx)), ptr(S.g("cnn.%s.bias" % idx)), dt,
                                         N, x.shape[1], x.shape[2], cin, cout, pad, impl, st))
                # data gradient = conv3x3(dy, flipped weights, pad' = 2 - pad)
                check(L.lo_conv3x3(ptr(dy), ptr(ws["wflip"][idx]), None, ptr(mask), ptr(G[xin]), dt,
                                   N, dy.shape[1], dy.shape[2], cout, cin, 2 - pad, 0, impl, st))
            else:
                col = ws["col" + idx]                       # still holds im2col(x) from the forward
                M, K = col.shape
                check(L.lo_gemm(ptr(dy), dt, ptr(col), dt, ptr(S.g("cnn.%s.weight" % idx)), _lib.LO_F32, cout, K, M, 1, cout, K, 1, K, 1,
                                0, 0, 0, None, 0, 0, impl, st))                                    # dW = dy^T col
                check(L.lo_colsum(ptr(dy), dt, ptr(S.g("cnn.%s.bias" % idx)), M, cout, cout, 0, st))
                check(L.lo_gemm(ptr(dy), dt, ptr(ws["wflip"][idx]), dt, ptr(col), dt, M, K, cout, cout, 1, 1, cout, K, 1, 0, 0, 0, None,
                                0, 0, impl, st))                                                   # dcol = dy W  (col reused)
                check(L.lo_col2im(ptr(col), ptr(mask), ptr(G[xin]), dt, N, x.shape[1], x.shape[2], cin, R, S_, stride, pad, st))
            if on_layer_grad is not None:
                on_layer_grad(idx)
            if xin.startswith("P") and xin != "P0":
                src = "Y" + xin[1:]
                pool_k = cfg[xin[1:]][4]
                ysrc = A[src]
                check(L.lo_maxpool_backward(ptr(ysrc), ptr(A[xin]), ptr(G[xin]), ptr(G[src]), dt, N, ysrc.shape[1], ysrc.shape[2],
                                            ysrc.shape[3], pool_k[0], pool_k[1], st))
        sc, of = (1.0 / 128.0, -1.0) if self.input_norm == "tf" else (1.0, 0.0)
        if ws.get("code0") is not None:
            check(L.lo_conv1_pool_wgrad_code(ptr(ws["img"]), int(ws["img"].dtype == torch.uint8), sc, of, ptr(ws["code0"]), ptr(G["P0"]), dt,
                                             ptr(S.g("cnn.0.weight")), ptr(S.g("cnn.0.bias")), N, H, W, st))
        elif self.input_norm == "tf":
            check(L.lo_conv1_pool_wgrad_norm(ptr(ws["img"]), int(ws["img"].dtype == torch.uint8), 1.0 / 128.0, -1.0,
                                             ptr(S.f32("cnn.0.weight")), ptr(S.f32("cnn.0.bias")), ptr(G["P0"]), dt,
                                             ptr(S.g("cnn.0.weight")), ptr(S.g("cnn.0.bias")), N, H, W, st))
        else:
            wg1 = L.lo_conv1_pool_wgrad_u8 if ws["img"].dtype == torch.uint8 else L.lo_conv1_pool_wgrad
            check(wg1(ptr(ws["img"]), ptr(S.f32("cnn.0.weight")), ptr(S.f32("cnn.0.bias")), ptr(G["P0"]), dt,
                      ptr(S.g("cnn.0.weight")), ptr(S.g("cnn.0.bias")), N, H, W, st))
        if on_layer_grad is not None:
            on_layer_grad("0")
        if dimg is not None:
            # conv1's data gradient through its ReLU and max-pool, from the forward's codes and G["P0"] (complete above)
            check(L.lo_conv1_pool_dgrad_code(ptr(ws["code0"]), ptr(G["P0"]), dt, ptr(S.f32("cnn.0.weight")), sc, ptr(dimg),
                                             N, H, W, st))

    def forward(self, img):
        """Reference signature (seq2seq_torch.py:88-100): returns a new fp32 tensor [N,H',W',512].  With grad mode on and the
        image or a parameter requiring grad, an autograd graph is recorded whose backward runs ``backward_raw``; the output is
        the same either way.  The image gradient is returned in the image's shape and dtype."""
        return kernel_forward(self, (img,), (img,))[0][0]

    def _forward_impl(self, img, need_grad):
        """((encoder output,), None, what the backward of this call needs or None)."""
        out = self.forward_raw(img, need_grad=need_grad)
        if not need_grad:
            return (out.float(),), None, None
        N, _, H, W = img.shape
        ws = self._ws.get((N, H, W))
        # a copy, never the workspace buffer itself: each call's output has its own node
        return (out.to(torch.float32, copy=True),), None, {"entries": [ws], "ws": ws, "shape": tuple(img.shape), "dtype": img.dtype}

    def _backward_impl(self, saved, dout, need):
        """backward_raw on the workspace of the forward: returns (d img in the image's shape and dtype, or None,)."""
        dimg = torch.empty(saved["shape"], dtype=torch.float32, device=dout.device) if need[0] else None
        self.backward_raw(saved["shape"], dout.float().contiguous(), ws=saved["ws"], dimg=dimg)
        return (dimg.to(saved["dtype"]) if dimg is not None else None,)
