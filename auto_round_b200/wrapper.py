"""Tunable fake-quant linear for the SignRound loop -- host-side mirror of auto_round/wrapper.py.

`WrapperLinear` keeps the reference's parameter names (`value`, `min_scale`, `max_scale`, wrapper.py:184-190)
but the parameters are *views into one flat fp32 arena per block* (see quantizer.TuneArena) and the math runs in
hand-written sm_90a kernels behind the C ABI:

    forward   ar_gemm_bf16          Y = X · Wqᵀ on wgmma;  Wq = qdq(W; V, scales) is resident     (wrapper.py:517-565)
    backward  ar_gemm_bf16          dWq = dYᵀ·X  (bf16, like autograd of F.linear)  and  dX = dY · Wq
              ar_fq_update          ONE pass per layer: fake-quant backward from dWq (replaces autograd through
                                    wrapper.py:273-290), best-param snapshot, sign-SGD step, and the NEXT iteration's Wq
    (with micro-batches -- gradient_accumulate_steps, lm_head -- the quantizer sums the micro-batches' dWq in fp32 and
     runs ar_fq_update once per iteration)

There is no autograd graph over the weight and no eager fallback.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn

from . import ops
from .schemes import QuantizationScheme


class _FQLinearFn(torch.autograd.Function):
    """y = x · qdq(W)ᵀ (+bias).  `anchor` is a dummy fp32 scalar that requires grad so that backward runs even
    when x does not (q/k/v projections read the frozen block input)."""

    @staticmethod
    def forward(ctx, x, anchor, layer: "WrapperLinear"):
        k = layer.spec.k
        x2d = x.reshape(-1, k)
        if x2d.dtype != torch.bfloat16:
            x2d = x2d.to(torch.bfloat16)
        x2d = x2d.contiguous()
        y = ops.gemm(x2d, layer.wq, bias=layer.bias_bf16)          # layer.wq is kept current by ar_fq_update
        ctx.layer = layer
        ctx.x_dtype = x.dtype
        ctx.save_for_backward(x2d)
        return y.view(*x.shape[:-1], layer.spec.n)

    @staticmethod
    def backward(ctx, dy):
        layer = ctx.layer
        (x2d,) = ctx.saved_tensors
        dy2d = dy.reshape(-1, layer.spec.n)
        if dy2d.dtype != torch.bfloat16:
            dy2d = dy2d.to(torch.bfloat16)
        dy2d = dy2d.contiguous()
        # dWq[N,K] = dYᵀ·X: A = dY stored [T,N] (MN-major), B = X stored [T,K] (MN-major); bf16 like autograd of F.linear
        ops.gemm(dy2d, x2d, a_mn_major=True, b_mn_major=True, out=layer.gq)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = ops.fq_linear_bwd_dx(layer.spec, dy2d, layer.wq).view(*dy.shape[:-1], layer.spec.k)
            if dx.dtype != ctx.x_dtype:
                dx = dx.to(ctx.x_dtype)
        layer.got_grad = True
        if layer.on_grad is not None:          # the quantizer's per-layer exchange + fused update (after the dX GEMM:
            layer.on_grad(layer)               # the update overwrites layer.wq with the next iteration's weight)
        return dx, torch.zeros((), dtype=torch.float32, device=dy.device), None


class WrapperLinear(nn.Module):
    """Wraps an nn.Linear for tuning.  All tensors are CUDA; V / min_scale / max_scale and the bf16 dWq are slices of the
    block arena handed in by the quantizer."""

    def __init__(self, orig_layer: nn.Linear, scheme: QuantizationScheme, spec: ops.Spec, arena_views: dict,
                 global_scale=None, init_scale=None):
        super().__init__()
        # enable_alg_ext (SignRoundOptimizedWrapperLinear, sign_roundv2/quantizer.py:101-125): searched per-group initial
        # scale, fp32 [G]; the tunable max_scale (bound [0, 2]) multiplies it and min_scale is inert
        self.init_scale = init_scale
        self.orig_layer = orig_layer
        self.scheme = scheme
        self.spec = spec
        w = orig_layer.weight.data
        if not w.is_cuda:
            raise RuntimeError("WrapperLinear: the block must be on a CUDA device (no CPU tuning path)")
        if w.dtype != torch.bfloat16:
            raise RuntimeError(f"WrapperLinear: weights must be bf16 (amp dtype), got {w.dtype}")
        self.weight = w.contiguous()
        b = orig_layer.bias
        self.bias_bf16 = None if b is None else b.data.to(torch.bfloat16).contiguous()
        # wrapper.py:154-167 weight_min / weight_max (int types); nv: wrapper.py:108-114 global scale
        self.weight_min = self.weight_max = None
        if spec.is_int:
            self.weight_min, self.weight_max = ops.group_minmax(spec, self.weight)
        self.weight_global_scale = None
        if scheme.qdq_name == "nv_fp4":
            self.weight_global_scale = global_scale if global_scale is not None else ops.nv_global_scale(self.weight)
        self.value = arena_views["value"]
        self.max_scale = arena_views["max_scale"]
        self.min_scale = arena_views.get("min_scale")
        self.gq = arena_views.get("gq")                     # bf16 [N,K]: dL/dWq of the current iteration
        self.on_grad = None                                 # callback(layer) run at the end of this layer's backward
        self.got_grad = False
        self.wq = torch.empty_like(self.weight)            # fake-quant weight of the current iteration
        self.anchor = torch.zeros((), dtype=torch.float32, device=w.device, requires_grad=True)
        self.params = {"value": self.value, "max_scale": self.max_scale}
        if self.min_scale is not None:
            self.params["min_scale"] = self.min_scale

    def forward(self, x):
        return _FQLinearFn.apply(x, self.anchor, self)

    @torch.no_grad()
    def refresh_wq(self):
        """wq <- qdq(W; current V / scales): once before the loop; inside it ar_fq_update keeps wq current."""
        ops.qdq_fwd(self.spec, self.weight, self.value, self.min_scale, self.max_scale, self.weight_min, self.weight_max,
                    self.weight_global_scale, out_wq=self.wq, init_scale=self.init_scale)

    @torch.no_grad()
    def unwrapper(self, best: dict):
        """wrapper.py:345-468: qdq with the best params -> orig_layer.weight; attach scale / zp / global scale."""
        spec = self.spec
        # best == {} -> plain RTN (iters == 0): V = 0, scales = 1, range math in the weight dtype like the reference
        wq, scale, zp = ops.qdq_fwd(spec, self.weight, best.get("value"), best.get("min_scale"), best.get("max_scale"),
                                    self.weight_min, self.weight_max, self.weight_global_scale, out_wq=self.wq,
                                    want_scale=True, init_scale=self.init_scale)
        lin = self.orig_layer
        lin.weight.data.copy_(wq)
        n = spec.n
        lin.scale = scale.reshape(n, -1)
        if self.scheme.qdq_name == "int_sym":
            lin.zp = int(2 ** (self.scheme.bits - 1))
        elif self.scheme.qdq_name == "int_asym":
            lin.zp = zp.reshape(n, -1)
        else:
            lin.zp = None
        if self.weight_global_scale is not None:
            lin.weight_global_scale = self.weight_global_scale
        return lin

    @torch.no_grad()
    def unwrapper_opt_rtn(self, imatrix: Optional[torch.Tensor] = None):
        """iters == 0 without disable_opt_rtn (get_quant_func, data_type/utils.py:139-146): the imatrix-weighted scale
        search, then the qdq -- opt_rtn_int_sym (int.py:89-122), opt_rtn_nv_fp4 (nvfp.py:388-413), opt_rtn_mx_fp4
        (mxfp.py:172-230).  int_asym has no opt_rtn_* entry in the reference registry and takes the plain function."""
        name = self.scheme.qdq_name
        if name == "int_asym":
            return self.unwrapper({})
        spec, lin, n = self.spec, self.orig_layer, self.spec.n
        w = self.weight
        if name == "int_sym":
            qw = importance_weights(imatrix, w, self.scheme.bits, spec.group_size)
            scale, wq = ops.search_scale_int(spec, w, qw)
            lin.weight.data.copy_(wq)
            lin.scale = scale.to(w.dtype).reshape(n, -1)               # the reference keeps the searched scale in bf16
            lin.zp = int(2 ** (self.scheme.bits - 1))
            return lin
        if name == "nv_fp4":
            qw = importance_weights(imatrix, w, 4, spec.group_size)
            coeff = ops.search_scale_nv(spec, w, qw)
        else:
            qw = importance_weights(imatrix, w.to(torch.float32), 4, spec.group_size)
            coeff = ops.search_scale_mx(spec, w, qw)
        wq, scale, _ = ops.qdq_fwd(spec, w, None, None, coeff, None, None, self.weight_global_scale, out_wq=self.wq,
                                   want_scale=True)
        lin.weight.data.copy_(wq)
        lin.scale = scale.reshape(n, -1)
        lin.zp = None
        if self.weight_global_scale is not None:
            lin.weight_global_scale = self.weight_global_scale
        return lin


def importance_weights(imatrix: Optional[torch.Tensor], w: torch.Tensor, bits: int, group_size: int):
    """Per-element loss weights of the scale searches from the per-channel importance (int.py:107-115).  The common case
    returns the [K] vector untouched (the kernel broadcasts it over rows and pads K with 1e-5).  Channels whose importance
    is exactly zero take the reference's repair path (data_type/gguf.py:437-484), materialised here as [N, Kpad]."""
    if imatrix is None:
        return None
    im = imatrix.reshape(-1).to(torch.float32)
    if bool(torch.min(im) != 0):
        return im.contiguous()
    n, k = w.shape
    kpad = (k + group_size - 1) // group_size * group_size
    if kpad != k:
        im = torch.nn.functional.pad(im, (0, kpad - k), value=1e-5)
        w = torch.nn.functional.pad(w, (0, kpad - k), value=0.0)
    g = w.reshape(-1, group_size)
    qw = im.reshape(1, -1).expand(n, -1).reshape(-1, group_size).clone()
    zero_cnt = torch.sum(qw <= 1e-30, dim=-1)
    replace = zero_cnt > group_size // 2
    if bool(replace.any()):
        if bits <= 3:
            tmp = torch.abs(g)
        else:
            tmp = torch.abs(g) + torch.sqrt(torch.sum(torch.pow(g, 2), dim=-1, keepdim=True) / 32)
        qw[replace, :] = tmp.to(qw.dtype)[replace, :]
    mean_replace = (zero_cnt > 0) & (zero_cnt <= group_size // 2)
    if bool(mean_replace.any()):
        fill = (torch.sum(qw, dim=-1) / (qw.shape[1] - zero_cnt)).view(-1, 1).expand(-1, qw.shape[1])
        idx = qw == 0
        qw[idx] = fill[idx]
    return qw.reshape(n, kpad).contiguous()


def set_module(root: nn.Module, name: str, new: nn.Module):
    parts = name.split(".")
    parent = root
    for p in parts[:-1]:
        parent = getattr(parent, p)
    setattr(parent, parts[-1], new)
