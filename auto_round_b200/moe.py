"""MoE experts on H100 -- replaces auto_round/modeling/fused_moe/moe_experts_interface.py:173-260 (the reference un-fuses
HF's fused 3-D expert parameters into per-expert nn.Linear modules and runs a python loop over the experts with
nonzero / index_select / index_copy_ per expert) by a device-side routing + grouped wgmma GEMM path:

    ar_moe_route      (token, slot) pairs sorted by expert, segments padded to the 256-row tile, tile tables   csrc/ar_moe.cu
    ar_moe_gather     Xp = X[token of row]                                                                       "
    grouped GEMMs     G = Xp·Wq_gateᵀ, U = Xp·Wq_upᵀ  ->  SwiGLU  ->  D = H·Wq_downᵀ   (ONE launch each for all experts)   csrc/ar_gemm.cu
    ar_moe_combine    out[token] = sum_slot D[row] * w[token, slot]                                              csrc/ar_moe.cu

All shapes are static (worst-case padded row capacity, tile counts read from device memory), nothing synchronises with the
host, so a MoE block's sign-SGD iteration is captured in a CUDA graph like a dense one.  The module keeps the reference's
layer names (`...experts.{e}.{gate,up,down}_proj`, SURVEY.md A.4): every projection is an nn.Linear whose weight is a VIEW
into one stacked [E, N, K] tensor per projection, which is what the grouped GEMMs read.

Data parallel runs use EXPERT PARALLELISM (SURVEY.md 8e): rank r owns experts [r E/W, (r+1) E/W) -- their rounding offsets,
scales and gradients never leave the rank.  Per iteration the ranks all-gather the (T/W)-token activations and routing, each
computes its experts' contribution for ALL tokens, and a reduce-scatter returns every rank the summed outputs of its own
tokens (backward: the same two collectives on the gradients).  4 x 134 MB per iteration instead of 2 x 2.9 GB of expert-weight
gradients for Mixtral-8x7B.  There is no CPU / eager fallback: the python loop lives in oracle/moe_loop.py as the test oracle.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import ops

PROJS = ("gate_proj", "up_proj", "down_proj")


class _ExpertContainer(nn.Module):
    def __init__(self, gate: nn.Linear, up: nn.Linear, down: nn.Linear):
        super().__init__()
        self.gate_proj, self.up_proj, self.down_proj = gate, up, down


def _view_linear(w_view: torch.Tensor) -> nn.Linear:
    n, k = w_view.shape
    lin = nn.Linear(k, n, bias=False, device="meta")
    lin.weight = nn.Parameter(w_view, requires_grad=False)
    return lin


class _GroupedExpertsFn(torch.autograd.Function):
    """hidden [T, H], top_k_index [T, k], top_k_weights [T, k] -> [T, H].  `anchor` makes backward run."""

    @staticmethod
    def forward(ctx, hidden, top_k_index, top_k_weights, anchor, mod: "GroupedExperts"):
        t_local, h = hidden.shape
        k = top_k_index.shape[-1]
        ep = mod.ep if (mod.tuning and mod.ep is not None and mod.ep.world > 1) else None
        x = hidden if hidden.dtype == torch.bfloat16 else hidden.to(torch.bfloat16)
        x = x.contiguous()
        ids = top_k_index.reshape(-1).to(torch.int64).contiguous()
        pw = top_k_weights.reshape(-1).to(torch.bfloat16).contiguous()
        e_begin, e_local, tokens = 0, mod.num_experts, t_local
        if ep is not None:
            w = ep.world
            e_local = mod.num_experts // w
            e_begin = ep.rank * e_local
            tokens = t_local * w
            x_all = torch.empty(tokens, h, dtype=torch.bfloat16, device=x.device)
            ids_all = torch.empty(tokens * k, dtype=torch.int64, device=x.device)
            pw_all = torch.empty(tokens * k, dtype=torch.bfloat16, device=x.device)
            ep.all_gather_(x_all, x)
            ep.all_gather_(ids_all, ids)
            ep.all_gather_(pw_all, pw)
            x, ids, pw = x_all, ids_all, pw_all
        route = mod.route_for(tokens * k, e_local, x.device)
        ops.moe_route(route, ids, e_begin)
        wg, wu, wd = (mod.stack(p, fake_quant=mod.tuning)[e_begin:e_begin + e_local] for p in PROJS)
        inter = wg.shape[1]
        xp = ops.moe_gather(x, route, k)
        g = ops.gemm_grouped_m(xp, wg, route, n=inter, k=h)
        u = ops.gemm_grouped_m(xp, wu, route, n=inter, k=h)
        hh = ops.swiglu_fwd(g, u)
        d = ops.gemm_grouped_m(hh, wd, route, n=h, k=inter)
        out = ops.moe_combine(d, route, tokens, k, pair_w=pw)
        if ep is not None:
            part = out
            out = torch.empty(t_local, h, dtype=torch.bfloat16, device=x.device)
            ep.reduce_scatter_(out, part)
        ctx.mod, ctx.route, ctx.k, ctx.ep, ctx.dims = mod, route, k, ep, (t_local, tokens, h, inter, e_begin, e_local)
        ctx.in_dtype, ctx.w_dtype, ctx.w_shape = hidden.dtype, top_k_weights.dtype, top_k_weights.shape
        ctx.save_for_backward(xp, g, u, hh, d, pw)
        return out if out.dtype == hidden.dtype else out.to(hidden.dtype)

    @staticmethod
    def backward(ctx, dout):
        mod, route, k, ep = ctx.mod, ctx.route, ctx.k, ctx.ep
        t_local, tokens, h, inter, e_begin, e_local = ctx.dims
        xp, g, u, hh, d, pw = ctx.saved_tensors
        go = dout.reshape(t_local, h)
        go = (go if go.dtype == torch.bfloat16 else go.to(torch.bfloat16)).contiguous()
        if ep is not None:
            go_all = torch.empty(tokens, h, dtype=torch.bfloat16, device=go.device)
            ep.all_gather_(go_all, go)
            go = go_all
        # combine backward: dD[row] = dOut[token] * w (bf16), d w[pair] = <dOut[token], D[row]>
        dd = ops.moe_gather(go, route, k, pair_w=pw)
        dw = ops.moe_rowdot(go, d, route, k)
        sl = slice(e_begin, e_begin + e_local)
        wg, wu, wd = (mod.stack(p, fake_quant=True)[sl] for p in PROJS)
        # down projection
        ops.gemm_grouped_k(dd, hh, route, mod.grad_stack("down_proj")[sl])
        dh = ops.gemm_grouped_m(dd, wd, route, n=inter, k=h, b_mn_major=True)
        dg, du = ops.swiglu_bwd(dh, g, u)
        ops.gemm_grouped_k(dg, xp, route, mod.grad_stack("gate_proj")[sl])
        ops.gemm_grouped_k(du, xp, route, mod.grad_stack("up_proj")[sl])
        dx = None
        if ctx.needs_input_grad[0]:
            dxg = ops.gemm_grouped_m(dg, wg, route, n=h, k=inter, b_mn_major=True)
            dxu = ops.gemm_grouped_m(du, wu, route, n=h, k=inter, b_mn_major=True)
            dx = ops.moe_combine(dxg, route, tokens, k, pair_w=None, d2=dxu)
        if ep is not None:
            part = dw
            dw = torch.empty(t_local * k, dtype=torch.bfloat16, device=go.device)
            ep.reduce_scatter_(dw, part)
            if dx is not None:
                part = dx
                dx = torch.empty(t_local, h, dtype=torch.bfloat16, device=go.device)
                ep.reduce_scatter_(dx, part)
        # fused update of every local expert's three layers; an expert no token was routed to (count == 0) gets no gradient
        # and is left untouched on the device (SignSGD skips grad-is-None parameters, sign_sgd.py:274-276)
        for e in range(e_begin, e_begin + e_local):
            flag = route.counts[e - e_begin:e - e_begin + 1]
            for p in PROJS:
                wl = mod.layer(e, p)
                wl.got_grad = True
                if wl.on_grad is not None:
                    wl.on_grad(wl, flag)
        if dx is not None and dx.dtype != ctx.in_dtype:
            dx = dx.to(ctx.in_dtype)
        return dx, None, dw.view(ctx.w_shape).to(ctx.w_dtype), torch.zeros((), dtype=torch.float32, device=dout.device), None


class GroupedExperts(nn.Module):
    """Per-expert nn.Linear containers "0".."E-1" (weights = views of one stacked tensor per projection) + the grouped
    forward.  While a block is tuned the linears are WrapperLinear (`bind_wrapped`): the grouped GEMMs then read the stacked
    fake-quant weights the fused update kernel keeps current, and write the stacked weight gradients it consumes."""

    def __init__(self, fused: nn.Module):
        super().__init__()
        gu, dn = fused.gate_up_proj.data, fused.down_proj.data
        e, two_i, h = gu.shape
        inter = two_i // 2
        name = type(fused.act_fn).__name__.lower()
        if not (isinstance(fused.act_fn, nn.SiLU) or "silu" in name or "swish" in name):
            raise NotImplementedError("grouped experts: only SiLU-gated (SwiGLU) experts are built")
        if e > 32:
            raise NotImplementedError("grouped experts: at most 32 experts per routing launch (ar_moe_route)")
        self.num_experts, self.hidden, self.inter, self.act_fn = e, h, inter, fused.act_fn
        self._stacks = {"gate_proj": gu[:, :inter].contiguous(), "up_proj": gu[:, inter:].contiguous(), "down_proj": dn.contiguous()}
        for i in range(e):
            self.add_module(str(i), _ExpertContainer(*(_view_linear(self._stacks[p][i]) for p in PROJS)))
        self._fq, self._grads, self._routes = {}, {}, {}
        self.tuning = False
        self.ep = None                              # quantizer.DataParallel when the experts are sharded over the ranks
        self.anchor = None

    def layer(self, e: int, proj: str):
        return getattr(getattr(self, str(e)), proj)

    def stack(self, proj: str, fake_quant: bool = False) -> torch.Tensor:
        """[E, N, K] weights of one projection: the fake-quant weights of the current iteration while tuning, else the
        linears' own weights (re-stacked if `.to()` / load_state_dict broke the aliasing)."""
        if fake_quant:
            return self._fq[proj]
        st = self._stacks.get(proj)
        lins = [self.layer(e, proj) for e in range(self.num_experts)]
        ws = [(l.orig_layer.weight if hasattr(l, "orig_layer") else l.weight) for l in lins]
        if st is None or st.device != ws[0].device or any(w.data_ptr() != st[e].data_ptr() for e, w in enumerate(ws)):
            st = torch.stack([w.data for w in ws]).contiguous()
            for e, w in enumerate(ws):
                w.data = st[e]
            self._stacks[proj] = st
        return st

    def grad_stack(self, proj: str) -> torch.Tensor:
        return self._grads[proj]

    def route_for(self, pairs: int, e_local: int, device) -> ops.MoeRoute:
        key = (pairs, e_local, str(device))
        if key not in self._routes:
            self._routes[key] = ops.MoeRoute(pairs, e_local, device)
        return self._routes[key]

    def bind_wrapped(self, ep=None):
        """Called after wrapper_block: point every expert WrapperLinear's fake-quant weight / weight gradient at slices of
        stacked [E, N, K] buffers."""
        dev = self.layer(0, PROJS[0]).weight.device
        for p in PROJS:
            n, k = self.layer(0, p).weight.shape
            self._fq[p] = torch.empty(self.num_experts, n, k, dtype=torch.bfloat16, device=dev)
            pitch = (n + 255) // 256 * 256          # row pitch of an expert's gradient slab: whole 256-row GEMM tiles
            self._grads[p] = torch.zeros(self.num_experts, pitch, k, dtype=torch.bfloat16, device=dev)
            for e in range(self.num_experts):
                wl = self.layer(e, p)
                wl.wq, wl.gq = self._fq[p][e], self._grads[p][e, :n]
        self.anchor = torch.zeros((), dtype=torch.float32, device=dev, requires_grad=True)
        self.ep = ep if (ep is not None and ep.world > 1) else None
        if self.ep is not None and self.num_experts % self.ep.world:
            raise NotImplementedError(f"expert parallelism needs num_experts ({self.num_experts}) divisible by the world size")
        self.tuning = True

    def release(self):
        """After unwrapper_block: drop the tuning buffers (stacked fake-quant weights, gradients, routing tables)."""
        self._fq, self._grads, self._routes, self.anchor, self.ep, self.tuning = {}, {}, {}, None, None, False

    def owner_of(self, e: int) -> int:
        return 0 if self.ep is None else e // (self.num_experts // self.ep.world)

    def forward(self, hidden_states, top_k_index, top_k_weights):
        if not hidden_states.is_cuda:
            raise RuntimeError("GroupedExperts: CUDA tensors only (auto_round_b200 has no CPU path; the reference's expert loop is "
                               "restated in oracle/moe_loop.py for the tests)")
        lead = hidden_states.shape
        x = hidden_states.reshape(-1, lead[-1])
        ids = top_k_index.reshape(x.shape[0], -1)
        w = top_k_weights.reshape(x.shape[0], -1)
        anchor = self.anchor if self.tuning else torch.zeros((), dtype=torch.float32, device=x.device)
        out = _GroupedExpertsFn.apply(x, ids, w, anchor, self)
        return out.view(lead)


def is_fused_experts(m: nn.Module) -> bool:
    gu, dn = getattr(m, "gate_up_proj", None), getattr(m, "down_proj", None)
    return isinstance(gu, nn.Parameter) and isinstance(dn, nn.Parameter) and gu.dim() == 3 and dn.dim() == 3 \
        and hasattr(m, "act_fn") and gu.shape[0] == dn.shape[0]


def unfuse_experts(block: nn.Module) -> int:
    """Replace every fused-experts module of `block` in place; returns how many were replaced."""
    from .wrapper import set_module
    n = 0
    for name, m in list(block.named_modules()):
        if is_fused_experts(m):
            set_module(block, name, GroupedExperts(m))
            n += 1
    return n
