"""Fused block glue for Llama-family decoder layers (RMSNorm / rotary embedding / SwiGLU), patched into the HF
block for the duration of the tuning loop and of the full-set forwards.

The reference runs these as chains of ATen elementwise kernels inside the HF layer (the layer is user code from
`transformers`, reached through compressors/utils.py:109-172 block_forward).  They are a visible share of an iteration's
device time, so each chain becomes one hand-written kernel forward and one backward (csrc/ar_block.cu).  Forward
values keep HF's rounding points; blocks that do not match the recognised patterns are left untouched.
"""
from __future__ import annotations

import sys
import types

import torch
import torch.nn as nn

from . import ops


class _RMSNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, eps):
        shape = x.shape
        x2d = x.reshape(-1, shape[-1])
        if x2d.dtype != torch.bfloat16:
            x2d = x2d.to(torch.bfloat16)
        x2d = x2d.contiguous()
        y, rstd = ops.rmsnorm_fwd(x2d, w, eps)
        ctx.save_for_backward(x2d, w, rstd)
        ctx.in_dtype = x.dtype
        return y.view(shape)

    @staticmethod
    def backward(ctx, dy):
        x2d, w, rstd = ctx.saved_tensors
        dy2d = dy.reshape(x2d.shape)
        if dy2d.dtype != torch.bfloat16:
            dy2d = dy2d.to(torch.bfloat16)
        dx = ops.rmsnorm_bwd(dy2d.contiguous(), x2d, w, rstd).view(dy.shape)
        return dx.to(ctx.in_dtype), None, None


class FusedRMSNorm(nn.Module):
    def __init__(self, orig: nn.Module):
        super().__init__()
        self.orig = orig
        self.eps = float(getattr(orig, "variance_epsilon", getattr(orig, "eps", 1e-6)))

    def forward(self, x):
        w = self.orig.weight
        if w.dtype != torch.bfloat16:
            w = w.to(torch.bfloat16)
        return _RMSNormFn.apply(x, w.contiguous(), self.eps)


class _RopeFn(torch.autograd.Function):
    """x: [B,H,S,D] view whose memory is [B,S,H,D] (projection output); cos/sin [1|B,S,D]."""

    @staticmethod
    def forward(ctx, x, cos, sin):
        xb = x.transpose(1, 2)
        if not xb.is_contiguous():
            xb = xb.contiguous()
        out = ops.rope(xb, cos, sin, backward=False)
        ctx.save_for_backward(cos, sin)
        return out.transpose(1, 2)

    @staticmethod
    def backward(ctx, g):
        cos, sin = ctx.saved_tensors
        gb = g.transpose(1, 2)
        if gb.dtype != torch.bfloat16:
            gb = gb.to(torch.bfloat16)
        if not gb.is_contiguous():
            gb = gb.contiguous()
        return ops.rope(gb, cos, sin, backward=True).transpose(1, 2), None, None


def _make_fused_rope(orig_fn):
    def apply_rotary_pos_emb(q, k, cos, sin, *args, **kwargs):
        plain = (not args) and (not kwargs or (set(kwargs) == {"unsqueeze_dim"} and kwargs["unsqueeze_dim"] == 1))
        ok = (plain and isinstance(q, torch.Tensor) and q.is_cuda and q.dtype == torch.bfloat16 and k.dtype == torch.bfloat16
              and q.dim() == 4 and k.dim() == 4 and cos.dim() == 3 and cos.dtype == torch.bfloat16
              and sin.dtype == torch.bfloat16 and cos.shape[-1] == q.shape[-1] and q.shape[-1] % 16 == 0
              and cos.shape[1] == q.shape[2] and k.shape[2] == q.shape[2] and cos.shape[0] in (1, q.shape[0]))
        if not ok:
            return orig_fn(q, k, cos, sin, *args, **kwargs)
        c, s = cos.contiguous(), sin.contiguous()
        return _RopeFn.apply(q, c, s), _RopeFn.apply(k, c, s)
    apply_rotary_pos_emb._ar_fused = True
    return apply_rotary_pos_emb


class _SwiGLUFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, gate, up):
        g, u = gate.contiguous(), up.contiguous()
        ctx.save_for_backward(g, u)
        return ops.swiglu_fwd(g, u)

    @staticmethod
    def backward(ctx, dh):
        g, u = ctx.saved_tensors
        if dh.dtype != torch.bfloat16:
            dh = dh.to(torch.bfloat16)
        return ops.swiglu_bwd(dh.contiguous(), g, u)


def _is_silu(act) -> bool:
    n = type(act).__name__.lower()
    return isinstance(act, nn.SiLU) or "silu" in n or "swish" in n


def _fused_mlp_forward(self, x):
    g, u = self.gate_proj(x), self.up_proj(x)
    if g.dtype == torch.bfloat16 and u.dtype == torch.bfloat16 and g.is_cuda and g.numel() % 8 == 0:
        return self.down_proj(_SwiGLUFn.apply(g, u))
    return self.down_proj(self.act_fn(g) * u)


# RMSNorm classes whose forward is exactly `w * (x * rsqrt(mean(x^2) + eps)).to(dtype)` (verified against the HF sources):
# an allowlist, because (1 + w) variants (Gemma, Qwen3-Next) share the class-name suffix but not the formula
_PLAIN_RMSNORM = {"LlamaRMSNorm", "Qwen2RMSNorm", "Qwen3RMSNorm", "MistralRMSNorm", "MixtralRMSNorm", "Qwen2MoeRMSNorm",
                  "Qwen3MoeRMSNorm", "Phi3RMSNorm"}


class fused_block_ops:
    """Context manager: patch RMSNorm modules, SwiGLU MLPs and the rotary helper of `block`; restore on exit."""

    def __init__(self, block: nn.Module, enabled: bool = True):
        self.block, self.enabled = block, enabled
        self.norms, self.mlps, self.rope = [], [], None

    def __enter__(self):
        if not self.enabled:
            return self
        from .wrapper import set_module
        for name, m in list(self.block.named_modules()):
            cls = type(m).__name__
            if cls in _PLAIN_RMSNORM and hasattr(m, "weight") and m.weight is not None and m.weight.dim() == 1 \
                    and m.weight.is_cuda and m.weight.shape[0] % 8 == 0 and m.weight.shape[0] <= 8192 \
                    and (hasattr(m, "variance_epsilon") or hasattr(m, "eps")):
                self.norms.append((name, m))
                set_module(self.block, name, FusedRMSNorm(m))
            elif all(hasattr(m, a) for a in ("gate_proj", "up_proj", "down_proj", "act_fn")) and _is_silu(m.act_fn) \
                    and "forward" not in m.__dict__:
                m.forward = types.MethodType(_fused_mlp_forward, m)
                self.mlps.append(m)
        # the rotary helper of the model file that defines the block: for a group of blocks tuned together (nblocks > 1)
        # that is the file of its members, the first modules of the walk that have one
        fn = None
        for m in self.block.modules():
            mod = sys.modules.get(type(m).__module__)
            fn = getattr(mod, "apply_rotary_pos_emb", None) if mod is not None else None
            if fn is not None:
                break
        if fn is not None and not getattr(fn, "_ar_fused", False):
            self.rope = (mod, fn)
            mod.apply_rotary_pos_emb = _make_fused_rope(fn)
        return self

    def __exit__(self, *a):
        from .wrapper import set_module
        for name, m in self.norms:
            set_module(self.block, name, m)
        for m in self.mlps:
            m.__dict__.pop("forward", None)
        if self.rope is not None:
            self.rope[0].apply_rotary_pos_emb = self.rope[1]
        self.norms, self.mlps, self.rope = [], [], None
        return False
