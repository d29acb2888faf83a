"""Block-wise SignRound tuning on H100 -- host-side mirror of
auto_round/algorithms/quantization/sign_round/quantizer.py:311-552 (SignRoundQuantizer.quantize_block).

Same call contract as the reference's plug point (SURVEY.md 8b #1): `quantize_block(block, fp_inputs, input_others,
fp_outputs, q_inputs, block_ctx, input_ids=None)` mutates `block` in place (qdq weights, `.scale/.zp/
.weight_global_scale` attributes on every quantised nn.Linear) and returns the best parameters.

What is different from the reference (H100-first):
  * all tunables of a block live in ONE flat fp32 arena [V of every layer | scales of every layer] with a matching
    best-snapshot arena; the weight gradient of every layer is the bf16 dWq of a plain wgmma GEMM, and ONE fused kernel
    per layer turns it into (fake-quant backward -> snapshot -> sign-SGD step -> next iteration's fake-quant weight);
  * under data parallelism a layer's dWq is reduce-scattered over the ranks as soon as its backward GEMMs are issued
    (overlapping the rest of the backward), each rank updates its row shard of V / scales and the new fake-quant weight
    is all-gathered: weight-sized work and memory traffic shrink with the number of GPUs;
  * loss, best-iteration selection, snapshot and sign-SGD update run on the device without any host
    synchronisation inside the 200-iteration loop (the reference calls loss.item() every iteration);
  * the sampler's batch sequence is drawn up-front (same python `random` stream, compressors/utils.py:388-438) and
    uploaded once; samples are gathered on the device;
  * calibration samples shard across ranks (rank r takes batch[r::world]); gradients are summed BEFORE the sign.
"""
from __future__ import annotations

import random
from dataclasses import dataclass, field
from typing import Optional

import numpy as np
import torch
import torch.nn as nn

from . import ops
from .schemes import QuantizationScheme
from .fused import fused_block_ops
from .wrapper import WrapperLinear, set_module

SHARED_CACHE_KEYS = ("position_ids", "cache_position", "position_embeddings", "cu_seqlens")  # utils/common.py:676


class IndexSampler:
    """auto_round/compressors/utils.py:388-438 -- cyclic shuffled batches from the GLOBAL python `random` state."""

    def __init__(self, nsamples: int, batch_size: int):
        if batch_size <= 0 or batch_size > nsamples:
            raise ValueError("batch_size must be > 0 and <= nsamples")
        self.nsamples, self.batch_size, self.index = nsamples, batch_size, 0
        self.indices = list(range(nsamples))
        random.shuffle(self.indices)

    def next_batch(self):
        if self.index + self.batch_size > self.nsamples:
            random.shuffle(self.indices)
            self.index = 0
        batch = self.indices[self.index:self.index + self.batch_size]
        self.index += self.batch_size
        return batch


def lr_schedule_table(iters: int, lr: float, minmax_lr: float) -> np.ndarray:
    """LinearLR(start 1.0 -> end 0.0 over `iters`) applied to fp32 lr tensors, chainable form
    (quantizer.py:426-429, torch.optim.lr_scheduler.LinearLR.get_lr): lr_{t+1} = fp32(lr_t * fp32(1 - 1/(iters-t))).
    Returns [iters, 2] float32: column 0 rounding lr, column 1 minmax lr."""
    tab = np.zeros((max(iters, 1), 2), dtype=np.float32)
    a, b = np.float32(lr), np.float32(minmax_lr)
    for t in range(iters):
        tab[t, 0], tab[t, 1] = a, b
        f = np.float32(1.0 + (0.0 - 1.0) / (iters * 1.0 + t * (0.0 - 1.0)))
        a, b = np.float32(a * f), np.float32(b * f)
    return tab


class TuneArena:
    """Flat storage for every tunable of one block: fp32 [ V_0 | V_1 | ... | scales ... ] (+ the best snapshot) and the bf16
    weight gradients `gq` [ dWq_0 | dWq_1 | ... ] written by the grad-w GEMMs."""

    def __init__(self, specs: dict, device):
        off = 0
        self.views = {}
        for name, spec in specs.items():
            n = spec.n * spec.kpad
            self.views[name] = {"value": (off, n, (spec.n, spec.kpad))}
            off += n
        self.clamp_begin = off                       # first scale parameter (multiple of 16: kpad % 16 == 0)
        for name, spec in specs.items():
            g = spec.groups
            self.views[name]["max_scale"] = (off, g, (g,))
            off += (g + 3) // 4 * 4
            if spec.is_int:                           # mx/nv ignore min_scale (it never receives a gradient)
                self.views[name]["min_scale"] = (off, g, (g,))
                off += (g + 3) // 4 * 4
        self.numel = off
        self.params = torch.zeros(off, dtype=torch.float32, device=device)
        self.params[self.clamp_begin:] = 1.0          # min/max_scale start at 1, V at 0 (wrapper.py:184-190)
        self.best = self.params.clone()               # (a layer that never gets a gradient keeps its initial parameters)
        self.gq_views, goff = {}, 0
        for name, spec in specs.items():
            self.gq_views[name] = (goff, spec.n * spec.k, (spec.n, spec.k))
            goff += (spec.n * spec.k + 7) // 8 * 8    # 16-byte aligned segments (TMA store target)
        self.gq = torch.zeros(goff, dtype=torch.bfloat16, device=device)

    def layer_views(self, name: str) -> dict:
        out = {key: self.params[o:o + n].view(shape) for key, (o, n, shape) in self.views[name].items()}
        o, n, shape = self.gq_views[name]
        out["gq"] = self.gq[o:o + n].view(shape)
        return out

    def best_views(self, name: str) -> dict:
        return {key: self.best[o:o + n].view(shape) for key, (o, n, shape) in self.views[name].items()}


@dataclass
class DataParallel:
    """Calibration-sample sharding over the ranks of one NVSwitch box (SURVEY.md 8e).  The data path uses NCCL
    (reduce-scatter / all-gather / all-reduce over NVLink); with a `gloo` group -- the CPU tests of the host logic and the
    single-GPU two-process test of the sharded update -- the same calls are emulated with gloo's all-reduce / all-gather."""
    rank: int = 0
    world: int = 1
    group: object = None

    def shard(self, batch):
        return list(batch)[self.rank::self.world]

    def row_shard(self, n_rows: int):
        """Rows [r0, r1) of a layer's weight this rank owns in the sharded update, or None when the rows do not split
        evenly (the layer then stays replicated: all-reduce of dWq + full update on every rank)."""
        if self.world == 1 or n_rows % self.world:
            return None
        per = n_rows // self.world
        return self.rank * per, (self.rank + 1) * per

    def _nccl(self) -> bool:
        import torch.distributed as dist
        return dist.get_backend(self.group) == "nccl"

    def all_reduce_(self, *tensors):
        if self.world == 1:
            return
        import torch.distributed as dist
        for t in tensors:
            if t.dtype == torch.bfloat16 and not self._nccl():      # gloo: no bf16 reduction
                f = t.float()
                dist.all_reduce(f, op=dist.ReduceOp.SUM, group=self.group)
                t.copy_(f)
            else:
                dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)

    def reduce_scatter_(self, out, full):
        """out (this rank's contiguous 1/world slice of `full`) <- sum over ranks."""
        import torch.distributed as dist
        if self._nccl():
            dist.reduce_scatter_tensor(out, full, group=self.group)
        else:
            f = full.float()
            dist.all_reduce(f, op=dist.ReduceOp.SUM, group=self.group)
            out.copy_(f.reshape(self.world, -1)[self.rank].view_as(out))

    def all_gather_(self, out, local):
        """out [world * len(local)] <- every rank's `local` (which may be the rank's own slice of `out`)."""
        import torch.distributed as dist
        if self._nccl():
            dist.all_gather_into_tensor(out, local, group=self.group)
        else:                                                       # gloo has no all_gather on CUDA tensors: sum of
            dt = torch.float32 if out.dtype == torch.bfloat16 else out.dtype      # zero-padded slices (exact)
            buf = torch.zeros(out.numel(), dtype=dt, device=out.device)
            buf.view(self.world, -1)[self.rank].copy_(local.reshape(-1))
            dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=self.group)
            out.reshape(-1).copy_(buf)


@dataclass
class TuneResult:
    losses: list = field(default_factory=list)
    best_iter: int = 0
    best_loss: float = float("inf")
    init_loss: float = float("nan")
    batches: list = field(default_factory=list)
    quantized_layers: list = field(default_factory=list)
    used_cuda_graph: bool = False


def accumulate_gq(acc: torch.Tensor, gq: torch.Tensor, first: bool, final: bool):
    """Gradient accumulation over the micro-batches of one iteration: `acc` (fp32) sums the micro-batches' bf16 dWq `gq`
    (the reference accumulates V.grad in fp32; dV is linear in dWq for fixed parameters), and after the last one the sum
    is rounded to bf16 once, into `gq`, for the fused update."""
    if first:
        acc.copy_(gq)
    else:
        acc.add_(gq)
    if final:
        gq.copy_(acc)


def default_layer_filter(name: str, module: nn.Module) -> bool:
    return type(module) is nn.Linear


def valid_token_masks(input_ids, device, stacked: bool = False):
    """Per-sample masks of the tokens that count in the loss (label id != -100, base.py:257-280), or None when every
    token counts.  `input_ids`: list of [1, S] label ids (or None).  Returns a list of [S] bool tensors on `device`, or
    with `stacked` one contiguous uint8 [n, S] tensor."""
    if input_ids is None:
        return None
    masks = [(ids != -100).reshape(-1) for ids in input_ids]
    if all(bool(m.all()) for m in masks):
        return None
    if stacked:
        return torch.stack(masks).to(device=device, dtype=torch.uint8).contiguous()
    return [m.to(device) for m in masks]


def _causal_equivalent(masks, token_masks) -> bool:
    """True if every cached attention mask is plain causal except, at most, entries in the LAST query row whose
    token is excluded from the loss.  The reference builds exactly that mask for tensor datasets (last key masked,
    calibration/llm.py:375-398; last position -100, :359-360), and the last row of a causal block influences no
    other row, so the fast is_causal attention path is numerically identical on every row that matters."""
    if masks is None:
        return True
    if token_masks is None:
        return False
    for m, tm in zip(masks, token_masks):
        if m is None:
            continue
        if m.dim() != 4 or m.shape[-1] != m.shape[-2]:
            return False
        s = m.shape[-1]
        allowed = (m != 0) if m.dtype == torch.bool else (m == 0)
        causal = torch.ones(s, s, dtype=torch.bool, device=m.device).tril()
        diff = (allowed.reshape(-1, s, s) != causal).any(-1).any(0)        # rows that differ
        if bool(diff[:-1].any()):
            return False
        if bool(diff[-1]) and int(tm.reshape(-1)[-1]) != 0:
            return False
    return True


def _causal_when_unmasked(block: Optional[nn.Module]) -> bool:
    """True if every attention module of `block` runs causal attention when it gets attention_mask=None (HF sdpa and
    flash-attention integrations derive is_causal from the module); False for `eager` (or unknown) implementations."""
    if block is None:
        return False
    impls = set()
    for m in block.modules():
        cfg = getattr(m, "config", None)
        impl = getattr(cfg, "_attn_implementation", None) if cfg is not None else None
        if impl is not None:
            impls.add(impl)
    return bool(impls) and impls <= {"sdpa", "flash_attention_2", "flash_attention_3"}


class SignRoundQuantizer:
    """Tuning loop driver.  Hyper-parameters follow SignRoundConfig (sign_round/config.py:21-178)."""

    def __init__(self, scheme: QuantizationScheme, iters: int = 200, lr: Optional[float] = None,
                 minmax_lr: Optional[float] = None, batch_size: int = 8, enable_minmax_tuning: bool = True,
                 enable_quanted_input: bool = True, not_use_best_mse: bool = False, amp_dtype=torch.bfloat16,
                 layer_config: Optional[dict] = None, layer_filter=default_layer_filter,
                 dp: Optional[DataParallel] = None, gradient_accumulate_steps: int = 1, use_cuda_graph: bool = True,
                 fuse_block_ops: bool = True, enable_alg_ext: bool = False):
        self.scheme = scheme
        # sign_roundv2 (SignRoundV2Quantizer.prepare_run, sign_roundv2/quantizer.py:330-357): symmetric int / mx / nv layers
        # get a searched init scale with max_scale in [0, 2]; bits < 4 additionally switches to the outlier-suppressed loss
        self.enable_alg_ext = bool(enable_alg_ext)
        self.iters = iters
        self.lr_is_auto = lr is None
        self.lr = lr
        self.minmax_lr = minmax_lr
        self.batch_size = batch_size
        self.enable_minmax_tuning = enable_minmax_tuning
        self.enable_quanted_input = enable_quanted_input
        self.not_use_best_mse = not_use_best_mse
        self.amp_dtype = amp_dtype
        self.layer_config = layer_config or {}
        self.layer_filter = layer_filter
        self.dp = dp or DataParallel()
        self.use_cuda_graph = use_cuda_graph
        self.fuse_block_ops = fuse_block_ops
        self.gradient_accumulate_steps = max(1, int(gradient_accumulate_steps or 1))
        self.last_result: Optional[TuneResult] = None
        self.last_arena = None

    # sign_round/config.py:107-136
    def compute_lr(self, bits: int) -> float:
        if not self.lr_is_auto:
            return float(self.lr)
        if self.iters >= 1000 and bits <= 3:
            return 2.0 / self.iters
        return 1.0 / max(self.iters, 1)

    def _lr_table(self, bits: int, device) -> torch.Tensor:
        """Flat device copy of lr_schedule_table for this run: (rounding lr, minmax lr) of every iteration."""
        lr0 = self.compute_lr(bits)
        mm_lr0 = float(self.minmax_lr) if self.minmax_lr is not None else lr0
        if not self.enable_minmax_tuning:
            mm_lr0 = 0.0
        return torch.from_numpy(lr_schedule_table(self.iters, lr0, mm_lr0)).to(device).reshape(-1)

    def _read_losses(self, res: TuneResult, state: torch.Tensor, hist: torch.Tensor):
        """Device loss state of a finished tuning loop -> `res` (the only host sync of the loop).  With not_use_best_mse
        the last iteration is the one applied."""
        st = state.cpu().tolist()
        res.losses = hist.cpu().tolist()[:self.iters]
        res.best_loss, res.best_iter = st[0], int(st[2])
        res.init_loss = res.losses[0]
        if self.not_use_best_mse:
            res.best_iter, res.best_loss = self.iters - 1, res.losses[-1]

    def layer_names(self, name: str):
        """(full module name or None, name inside its own decoder block) of a layer named `name` relative to the module being
        tuned.  `self.block_prefix`, set by AutoRound before each block, is the block's full name ("model.layers.3"), or
        for a group of blocks tuned together (nblocks > 1) the prefix map of its `BlockGroup` ({"layers.0":
        "model.layers.2", "layers.1": "model.layers.3"}), which sends "layers.1.mlp.down_proj" to
        ("model.layers.3.mlp.down_proj", "mlp.down_proj")."""
        prefix = getattr(self, "block_prefix", None)
        if not prefix:
            return None, name
        if isinstance(prefix, str):
            return f"{prefix}.{name}", name
        head, j, rel = name.split(".", 2)
        return f"{prefix[f'{head}.{j}']}.{rel}", rel

    def scheme_for(self, name: str, module: nn.Module) -> Optional[QuantizationScheme]:
        """Per-layer override: `layer_config` keys are FULL module names as in the reference
        ("model.layers.3.mlp.down_proj": {"bits": 8}); `layer_names` turns the block-relative `name` into one.  A bare
        block-relative key ("mlp.down_proj") applies to that layer of every block."""
        cfg = None
        full, rel = self.layer_names(name)
        if full:
            cfg = self.layer_config.get(full)
        if cfg is None:
            cfg = self.layer_config.get(rel)
        if cfg is None:
            return self.scheme
        if isinstance(cfg, QuantizationScheme):
            return cfg
        from dataclasses import replace
        s = replace(self.scheme)
        for k, v in cfg.items():
            if hasattr(s, k):
                setattr(s, k, v)
        return s

    # ---------------------------------------------------------------------------------------------
    def _optimized(self, sc: QuantizationScheme) -> bool:
        return self.enable_alg_ext and sc.qdq_name in ("int_sym", "mx_fp4", "nv_fp4")

    def search_init_scale(self, spec, sc: QuantizationScheme, w: torch.Tensor, imatrix):
        """search_optimized_init_scale (data_type/utils.py:223-254) -> fp32 [G].  The importance vector is broadcast over
        rows and padded with 1e-5 inside the kernel; unlike the RTN route there is no zero repair here
        (reshape_imatrix_for_weight, data_type/utils.py:269-282)."""
        qw = None if imatrix is None else imatrix.reshape(-1).to(torch.float32).contiguous()
        if sc.qdq_name == "int_sym":
            return ops.search_scale_int(spec, w, qw, want_wq=False)[0]
        if sc.qdq_name == "mx_fp4":
            return ops.search_scale_mx(spec, w, qw)
        return ops.search_scale_nv(spec, w, qw)

    def wrapper_block(self, block: nn.Module, nv_global_scales: Optional[dict] = None, imatrices: Optional[dict] = None):
        """wrapper.py:774-828: every eligible nn.Linear (bits <= 8) -> WrapperLinear on the block arena."""
        todo = {}
        for name, mod in block.named_modules():
            if self.layer_filter(name, mod):
                sc = self.scheme_for(name, mod)
                if sc is None or sc.bits > 8:
                    continue
                n, k = mod.weight.shape
                thr = 1e-5
                todo[name] = (mod, sc, ops.make_spec(sc.qdq_name, sc.bits, sc.group_size, n, k, thr, 1.0))
        if not todo:
            return {}, None
        device = next(iter(todo.values()))[0].weight.device
        arena = TuneArena({n: t[2] for n, t in todo.items()}, device)
        wrapped = {}
        for name, (mod, sc, spec) in todo.items():
            gs = None if nv_global_scales is None else nv_global_scales.get(name)
            init = None
            if self._optimized(sc):
                init = self.search_init_scale(spec, sc, mod.weight.data.contiguous(), (imatrices or {}).get(name))
            wl = WrapperLinear(mod, sc, spec, arena.layer_views(name), gs, init)
            set_module(block, name, wl)
            wrapped[name] = wl
        return wrapped, arena

    def unwrapper_block(self, block: nn.Module, wrapped: dict, arena: TuneArena, use_best: bool = True):
        for name, wl in wrapped.items():
            views = arena.best_views(name) if use_best else {k: v for k, v in wl.params.items()}
            lin = wl.unwrapper(views)
            set_module(block, name, lin)

    def rtn_block(self, block: nn.Module, wrapped: Optional[dict] = None, nv_global_scales: Optional[dict] = None,
                  imatrices: Optional[dict] = None, is_moe: bool = False):
        """iters == 0: round-to-nearest of every eligible linear (algorithms/quantization/base.py:202-255).
        `imatrices is None` is the zero-shot route (`disable_opt_rtn=True` -> quant_tensor_rtn_sym / the plain dtype
        function); a dict {layer name: importance [K] or None} selects the optimized RTN (rtn/quantizer.py:108-140), except
        for routed MoE experts, which the reference sends through plain RTN (base.py:213-226)."""
        if wrapped is None:
            wrapped, _ = self.wrapper_block(block, nv_global_scales)
        with torch.no_grad():
            for name, wl in wrapped.items():
                plain = imatrices is None or (is_moe and "expert" in name and "shared_expert" not in name)
                set_module(block, name, wl.unwrapper({}) if plain else wl.unwrapper_opt_rtn(imatrices.get(name)))
        return list(wrapped)

    # ---------------------------------------------------------------------------------------------
    def _stack(self, samples, device):
        if isinstance(samples, torch.Tensor):
            return samples.to(device).contiguous()
        t = torch.cat([s.to(device, non_blocking=True) for s in samples], dim=0)
        return t.contiguous()

    def _prepare_others(self, input_others: dict, token_masks, device, block: Optional[nn.Module] = None):
        """Split block kwargs into (static kwargs, per-sample stacked tensors); drop a causal-equivalent mask -- but only
        when the block's attention takes the `is_causal` path for a missing mask (sdpa / flash); HF's eager attention applies
        NO mask at all when attention_mask is None, so there the cached mask is kept."""
        static, per_sample = {}, {}
        others = dict(input_others or {})
        others.pop("positional_inputs", None)
        am = others.get("attention_mask")
        if isinstance(am, (list, tuple)) and len(am) and isinstance(am[0], torch.Tensor):
            if _causal_when_unmasked(block) and _causal_equivalent(am, token_masks):
                others["attention_mask"] = None          # -> is_causal fast path inside the HF attention
        for key, val in others.items():
            if key in SHARED_CACHE_KEYS:
                # the calibrator stores shared kwargs either raw (tensor / (cos, sin) tuple) or as a LIST with one raw
                # value per calibration batch (calibration/llm.py:507-545): take the first copy
                v = val[0] if isinstance(val, list) and len(val) >= 1 else val
                static[key] = _to_device(v, device)
            elif isinstance(val, (list, tuple)) and len(val) and isinstance(val[0], torch.Tensor):
                per_sample[key] = torch.cat([v.to(device) for v in val], dim=0)
            elif isinstance(val, torch.Tensor):
                per_sample[key] = val.to(device)
            else:
                static[key] = val
        return static, per_sample

    def block_forward(self, block, x, kwargs):
        """compressors/utils.py:109-172: HF decoder layer under autocast(amp dtype); first output."""
        with torch.autocast(device_type="cuda", dtype=self.amp_dtype):
            out = block(x, **kwargs)
        return out[0] if isinstance(out, (tuple, list)) else out

    # ---------------------------------------------------------------------------------------------
    def quantize_block(self, block: nn.Module, fp_inputs, input_others, fp_outputs, q_inputs=None, block_ctx=None,
                       input_ids=None, nv_global_scales: Optional[dict] = None, **kwargs) -> dict:
        # the C ABI launches on the CURRENT device's current stream: make the block's device current for the whole call
        with torch.cuda.device(next(block.parameters()).device):
            return self._quantize_block(block, fp_inputs, input_others, fp_outputs, q_inputs, block_ctx, input_ids,
                                        nv_global_scales, **kwargs)

    def _quantize_block(self, block: nn.Module, fp_inputs, input_others, fp_outputs, q_inputs=None, block_ctx=None,
                        input_ids=None, nv_global_scales: Optional[dict] = None, **kwargs) -> dict:
        dp = self.dp
        active = q_inputs if (q_inputs is not None and self.enable_quanted_input) else fp_inputs
        device = next(block.parameters()).device
        if device.type != "cuda":
            raise RuntimeError("quantize_block: block must be on a CUDA device (auto_round_b200 has no CPU path)")
        x_all = self._stack(active, device)
        ref_all = self._stack(fp_outputs, device)
        nsamples = x_all.shape[0]
        seq, hidden = x_all.shape[1], x_all.shape[-1]

        token_masks = valid_token_masks(input_ids, device, stacked=True)
        valid_per_sample = None if token_masks is None else token_masks.sum(dim=1).cpu().tolist()

        wrapped, arena = self.wrapper_block(block, nv_global_scales, kwargs.get("imatrices"))
        self.last_arena = arena if kwargs.get("keep_arena") else None
        res = TuneResult(quantized_layers=list(wrapped))
        self.last_result = res
        if not wrapped or self.iters <= 0:
            if wrapped:                                   # iters == 0: plain RTN (data_type/int.py:125-162)
                self.rtn_block(block, wrapped)
            return {}

        static_kw, per_sample_kw = self._prepare_others(
            input_others, None if token_masks is None else list(token_masks), device, block)

        # ---- schedules drawn up-front (same python-random stream as the reference's IndexSampler)
        iters = self.iters
        # gradient_accumulate_steps = A > 1 (quantizer.py:437-452): an iteration draws batch_size * A samples and runs them
        # as A micro-batches of batch_size; MSELoss(reduction="sum"), gradients accumulate, ONE sign-SGD step
        accum = self.gradient_accumulate_steps
        mbs = min(nsamples, self.batch_size)
        gbs = min(nsamples, mbs * accum)
        accum = (gbs + mbs - 1) // mbs
        sampler = kwargs.get("sampler") or IndexSampler(nsamples, gbs)
        batches = [list(sampler.next_batch()) for _ in range(iters)]
        res.batches = batches
        micro = [[dp.shard(b[j * mbs:(j + 1) * mbs]) for j in range(accum)] for b in batches]
        lbs = len(micro[0][0])
        if lbs == 0 or any(len(m) != lbs for it_m in micro for m in it_m):
            raise RuntimeError(f"micro-batches of {mbs} samples (global batch {gbs}) cannot be sharded evenly over {dp.world} ranks")
        idx_dev = torch.tensor(micro, dtype=torch.int32, device=device).reshape(iters, accum * lbs)
        lr_tab = self._lr_table(min(wl.scheme.bits for wl in wrapped.values()), device)

        loss_sum = torch.zeros(1, dtype=torch.float64, device=device)
        state = torch.zeros(4, dtype=torch.float64, device=device)
        flag = torch.zeros(1, dtype=torch.int32, device=device)
        hist = torch.zeros(iters, dtype=torch.float32, device=device)
        # MSELoss('mean') over the GLOBAL batch; with accumulation the reference switches to reduction='sum'
        inv_numel = 1.0 / float(gbs * seq * hidden) if accum == 1 else 1.0
        x_buf = torch.empty((lbs,) + tuple(x_all.shape[1:]), dtype=x_all.dtype, device=device)
        ref_buf = torch.empty_like(x_buf)

        # ---- device-side schedule: iteration counter, current batch indices, 1/num_elm of the current batch
        it_dev = torch.zeros(1, dtype=torch.int32, device=device)
        cur32 = torch.zeros(accum * lbs, dtype=torch.int32, device=device)
        cur64 = torch.zeros(accum * lbs, dtype=torch.int64, device=device)
        cur_inv = torch.ones(1, dtype=torch.float64, device=device)
        if token_masks is not None:
            inv_tab = torch.tensor([1.0 / max(1, sum(valid_per_sample[i] for i in b)) for b in batches],
                                   dtype=torch.float64, device=device)
        elif accum > 1:           # num_elm = elements of the first global batch's inputs (quantizer.py:445-449)
            inv_tab = torch.full((iters,), 1.0 / float(gbs * seq * hidden), dtype=torch.float64, device=device)
        else:
            inv_tab = torch.ones(iters, dtype=torch.float64, device=device)

        from .moe import GroupedExperts
        moe_mods = [m for m in block.modules() if isinstance(m, GroupedExperts)]
        for m in moe_mods:          # expert WrapperLinears read / write slices of stacked [E, N, K] buffers; under data
            m.bind_wrapped(dp)      # parallelism the experts are sharded over the ranks (expert parallelism)
        ep_owned = {}               # id(expert WrapperLinear) -> this rank owns it (full local update, no exchange)
        for m in moe_mods:
            for e in range(m.num_experts):
                for pj in ("gate_proj", "up_proj", "down_proj"):
                    ep_owned[id(m.layer(e, pj))] = (m.owner_of(e) == dp.rank) if dp.world > 1 else True

        # enable_alg_ext loss (SignRoundV2Quantizer._get_loss, sign_roundv2/quantizer.py:362-399): bits < 4 -> the numel/1000
        # largest |pred - ref| are dropped; otherwise it falls back to the base MSE WITHOUT forwarding the valid-token mask
        # (sign_roundv2/quantizer.py:399).  That fallback also applies to int asym, which keeps the plain wrapper: with
        # enable_alg_ext its loss runs over every token (pinned by tests/golden/block_algext_w2a16_asym_g32.pt).
        optimized = [wl for wl in wrapped.values() if wl.init_scale is not None]
        outlier_loss = bool(optimized) and self.scheme.sym and self.scheme.bits < 4
        unmasked_loss = self.enable_alg_ext and not outlier_loss
        clamp_hi = 2.0 if optimized else 1.0                        # minmax_scale_bound (sign_roundv2/quantizer.py:102)
        if optimized and len(optimized) != len(wrapped):
            raise NotImplementedError("enable_alg_ext with mixed optimized / plain layers in one block (per-layer bounds)")
        outlier_scratch = ops.OutlierSelect(device) if outlier_loss else None

        # ---- per-layer exchange + fused update.  One GPU: the update kernel follows the layer's backward GEMMs on the compute
        # stream.  Data parallel: the layer's bf16 dWq is reduce-scattered on the communication stream while the backward
        # continues, this rank updates its row shard (fake-quant backward, snapshot, sign-SGD, next Wq) and the new Wq rows
        # are all-gathered; layers whose rows do not split evenly stay replicated (all-reduce + full update).
        compute_stream = lambda: torch.cuda.current_stream(device)          # noqa: E731 (the capture stream while capturing)
        comm = torch.cuda.Stream(device=device) if dp.world > 1 else None
        best_of = {n: arena.best_views(n) for n in wrapped}
        shards, gq_shard, wire_full, wire_seg = {}, {}, {}, {}
        for n, wl in wrapped.items():
            wl.refresh_wq()                                         # iteration 0 runs on qdq(W; V = 0, scales = 1)
            shards[n] = None if id(wl) in ep_owned else dp.row_shard(wl.spec.n)
            if shards[n] is not None:
                r0, r1 = shards[n]
                gq_shard[n] = torch.empty(r1 - r0, wl.spec.k, dtype=torch.bfloat16, device=device)
                if ops.wire_supported(wl.spec):
                    # the new fake-quant rows travel as 4-bit codes + per-group {a, off} (a quarter of the bf16 bytes);
                    # every rank rebuilds the identical bf16 weight with ar_wq_decode
                    wire_seg[n] = ops.wire_segment_bytes(wl.spec, r1 - r0)
                    wire_full[n] = torch.zeros(dp.world * wire_seg[n], dtype=torch.uint8, device=device)
        name_of = {id(wl): n for n, wl in wrapped.items()}

        def update_layer(wl, grad_flag=None):
            n = name_of[id(wl)]
            bv = best_of[n]
            kw = dict(best_v=bv["value"], best_min=bv.get("min_scale"), best_max=bv["max_scale"], flag=flag, it_dev=it_dev,
                      clamp_hi=clamp_hi, init_scale=wl.init_scale, has_grad=grad_flag)
            args = (wl.spec, wl.weight, wl.value, wl.min_scale, wl.max_scale, wl.weight_min, wl.weight_max, wl.weight_global_scale)
            owned = ep_owned.get(id(wl))
            if dp.world == 1 or owned is not None:
                # one GPU, or an expert layer under expert parallelism: its owner saw every token routed to it, so the
                # gradient is complete locally (no exchange); the other ranks leave it alone
                if owned is None or owned:
                    ops.fq_update(*args, wl.gq, wl.wq, lr_tab, **kw)
                return
            comm.wait_stream(compute_stream())                      # this layer's dWq and dX GEMMs are enqueued
            with torch.cuda.stream(comm):
                if shards[n] is None:
                    dp.all_reduce_(wl.gq)
                    ops.fq_update(*args, wl.gq, wl.wq, lr_tab, **kw)
                else:
                    r0, r1 = shards[n]
                    dp.reduce_scatter_(gq_shard[n], wl.gq)
                    if n in wire_full:
                        seg = wire_seg[n]
                        own = wire_full[n][dp.rank * seg:(dp.rank + 1) * seg]
                        ops.fq_update(*args, gq_shard[n], None, lr_tab, row0=r0, row1=r1, gq_row0=r0, wire=own, **kw)
                        dp.all_gather_(wire_full[n], own)
                        ops.wq_decode(wl.spec, wire_full[n], dp.world, wl.wq)
                    else:
                        ops.fq_update(*args, gq_shard[n], wl.wq, lr_tab, row0=r0, row1=r1, gq_row0=r0, **kw)
                        dp.all_gather_(wl.wq, wl.wq[r0:r1])

        for wl in wrapped.values():
            wl.on_grad = update_layer

        acc_state = {"first": True, "final": True}
        gq_acc = {}
        if accum > 1:
            if moe_mods:
                raise NotImplementedError("gradient_accumulate_steps > 1 with grouped MoE experts")
            if outlier_loss:
                raise NotImplementedError("gradient_accumulate_steps > 1 with the outlier-suppressed loss (enable_alg_ext, bits < 4)")
            gq_acc = {n: torch.zeros(wl.spec.n, wl.spec.k, dtype=torch.float32, device=device) for n, wl in wrapped.items()}

            def accumulate_then_update(wl, grad_flag=None):
                accumulate_gq(gq_acc[name_of[id(wl)]], wl.gq, acc_state["first"], acc_state["final"])
                if acc_state["final"]:
                    update_layer(wl, grad_flag)

            for wl in wrapped.values():
                wl.on_grad = accumulate_then_update

        def iteration(last: bool):
            ops.sched_load(idx_dev, inv_tab, it_dev, accum * lbs, cur32, cur64, cur_inv)
            for wl in wrapped.values():
                wl.got_grad = False
            for j in range(accum):
                c32, c64 = cur32[j * lbs:(j + 1) * lbs], cur64[j * lbs:(j + 1) * lbs]
                acc_state["first"], acc_state["final"] = (j == 0), (j == accum - 1)
                ops.gather_rows(x_all, c32, out=x_buf)
                ops.gather_rows(ref_all, c32, out=ref_buf)
                kw = dict(static_kw)
                for key, val in per_sample_kw.items():
                    kw[key] = val.index_select(0, c64)
                mask_rows = None
                if token_masks is not None:
                    mask_rows = token_masks.index_select(0, c64).reshape(-1)
                pred = self.block_forward(block, x_buf, kw)
                pred2d = pred.reshape(-1, hidden)
                if pred2d.dtype != torch.bfloat16:
                    pred2d = pred2d.to(torch.bfloat16)
                pred2d, ref2d = pred2d.contiguous(), ref_buf.reshape(-1, hidden)
                if outlier_loss:
                    dpred = ops.mse_outlier_fwd_bwd(pred2d, ref2d, mask_rows, 1000.0, loss_sum, outlier_scratch,
                                                    numel_global=gbs * seq * hidden if dp.world > 1 else None,
                                                    all_gather=dp.all_gather_, rank=dp.rank, world=dp.world)
                else:
                    dpred = ops.mse_fwd_bwd(pred2d, ref2d, None if unmasked_loss else mask_rows, inv_numel, 1000.0, loss_sum)

                def bookkeeping():                                  # loss -> best flag (read by every update kernel)
                    ops.best_update(loss_sum, inv_numel, 1.0, 0, state, flag, hist, inv_num_elm_dev=cur_inv, it_dev=it_dev)
                    if self.not_use_best_mse:
                        flag.fill_(1 if last else 0)

                if j == accum - 1:                                  # the iteration's loss is complete
                    if dp.world > 1:
                        comm.wait_stream(compute_stream())
                        with torch.cuda.stream(comm):
                            dp.all_reduce_(loss_sum)               # the best iteration is chosen on the GLOBAL loss
                            bookkeeping()
                    else:
                        bookkeeping()
                pred.backward(dpred.view_as(pred).to(pred.dtype))
            if dp.world > 1:
                compute_stream().wait_stream(comm)
            ops.iter_advance(it_dev)

        with fused_block_ops(block, self.fuse_block_ops):
            # ---- CUDA graph: the iteration has static shapes and a device-side schedule, so (after two eager iterations
            # that also serve as warm-up) it is captured once -- forward, backward, the per-layer collectives on the
            # communication stream and the fused updates -- and replayed.
            n_eager = min(iters, 2)
            use_graph = self.use_cuda_graph and not self.not_use_best_mse and iters > n_eager + 1
            graph = None
            if use_graph:
                side = torch.cuda.Stream(device=device)
                side.wait_stream(torch.cuda.current_stream(device))
                with torch.cuda.stream(side):
                    for it in range(n_eager):
                        iteration(False)
                torch.cuda.current_stream(device).wait_stream(side)
                for wl in wrapped.values():
                    wl.anchor.grad = None
                launches_before = ops.LAUNCHES[0]
                try:
                    graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(graph, capture_error_mode="thread_local" if dp.world > 1 else "global"):
                        iteration(False)
                except Exception as e:  # noqa: BLE001 -- capture is an optimisation; the eager loop is the same kernels
                    import warnings
                    warnings.warn(f"CUDA graph capture of the SignRound iteration failed ({e!r}); running eagerly")
                    graph = None
                    torch.cuda.synchronize(device)
                    if dp.world > 1:
                        raise
            else:
                n_eager = 0
            res.used_cuda_graph = graph is not None
            if graph is not None:       # launches recorded once at capture are issued at every replay
                per_graph = ops.LAUNCHES[0] - launches_before
                ops.LAUNCHES[0] += per_graph * (iters - n_eager) - per_graph
            for it in range(n_eager if use_graph else 0, iters):
                if graph is None:
                    iteration(it == iters - 1)
                else:
                    graph.replay()
        for wl in wrapped.values():
            wl.on_grad = None
        if dp.world > 1:            # every rank snapshotted its own row shard: rebuild the full best parameters
            import torch.distributed as dist
            for m in moe_mods:      # expert layers: the owner's best parameters go to everybody
                for e in range(m.num_experts):
                    for pj in ("gate_proj", "up_proj", "down_proj"):
                        for t in best_of[name_of[id(m.layer(e, pj))]].values():
                            dist.broadcast(t, src=m.owner_of(e), group=dp.group)
            for n, wl in wrapped.items():
                if shards[n] is None or id(wl) in ep_owned:
                    continue
                r0, r1 = shards[n]
                kp, gpr = wl.spec.kpad, wl.spec.kpad // wl.spec.group_size
                for key, t in best_of[n].items():
                    flat = t.reshape(-1)
                    per = kp if key == "value" else gpr
                    dp.all_gather_(flat, flat[r0 * per:r1 * per])

        self._read_losses(res, state, hist)
        with torch.no_grad():
            self.unwrapper_block(block, wrapped, arena)
        for m in moe_mods:
            m.release()
        return {n: arena.best_views(n) for n in wrapped}


    # ---------------------------------------------------------------------------------------------
    def quantize_layer(self, layer: nn.Linear, fp_inputs, q_inputs=None, input_ids=None, name: str = "lm_head", **kwargs):
        """A linear OUTSIDE the block list (lm_head with `quant_lm_head=True`) -- mirror of
        SignRoundQuantizer.quantize_layer_outside_block (sign_round/quantizer.py:554-759), on the block loop's gradient path:
        bf16 grad-w GEMM, then one fused update (ar_fq_update) per iteration.  Differences from the block loop, all the
        reference's: micro-batches of one sample with the gradient accumulated over the `batch_size` samples of an
        iteration (the `accumulate_gq` rule of gradient_accumulate_steps), MSELoss(reduction="sum"), the target is the FP
        weight applied to the FP input (recomputed each step: 128 x [2048, 128256] bf16 targets would be 67 GB for
        Llama-3), the tuning forward reads the quantised-chain input when there is one, and `num_elm` is fixed before the
        loop from the first `batch_size` samples.  `fp_inputs` / `q_inputs`: lists of [1, S, K] tensors.  Mutates `layer`
        in place."""
        device = layer.weight.device
        if not layer.weight.is_cuda:
            raise RuntimeError("quantize_layer: the layer must be on a CUDA device (no CPU tuning path)")
        torch.cuda.set_device(device)                              # the C ABI launches on the current device's stream
        # Under data parallelism every rank holds the full chained inputs (they were all-gathered) and runs this layer's
        # tuning REPLICATED: identical inputs, identical deterministic kernels, identical result on every rank, no exchange.
        # (Sharding the micro-batches would need a 1 GB bf16 gradient all-reduce per iteration for Llama-3's lm_head.)
        sc = self.scheme_for(name, layer)
        n, k = layer.weight.shape
        spec = ops.make_spec(sc.qdq_name, sc.bits, sc.group_size, n, k, 1e-5, 1.0)
        arena = TuneArena({name: spec}, device)
        gs = kwargs.get("nv_global_scale")
        wl = WrapperLinear(layer, sc, spec, arena.layer_views(name), gs)
        nsamples = len(fp_inputs)
        fp_all = self._stack(fp_inputs, device).to(torch.bfloat16)
        seq = fp_all.shape[1]
        fp_all = fp_all.reshape(nsamples, seq, k).contiguous()
        q_all = None if q_inputs is None else self._stack(q_inputs, device).to(torch.bfloat16).reshape(nsamples, seq, k).contiguous()
        token_masks = valid_token_masks(input_ids, device, stacked=True)
        iters = self.iters
        gbs = min(nsamples, self.batch_size)                       # gradient_accumulate_steps = batch_size (:660-662)
        if self.batch_size != 1:
            if token_masks is not None:
                num_elm = int(token_masks[:gbs].sum())
            else:
                num_elm = gbs * seq * k                            # _count_layer_input_elements over the first gbs samples
            inv_numel = 1.0                                        # reduction="sum"
        else:
            num_elm, inv_numel = 1, 1.0 / float(seq * n)
        num_elm = 1 if num_elm <= 0 else num_elm
        sampler = kwargs.get("sampler") or IndexSampler(nsamples, gbs)
        batches = [list(sampler.next_batch()) for _ in range(iters)]
        res = TuneResult(quantized_layers=[name], batches=batches)
        self.last_result = res
        lr_tab = self._lr_table(sc.bits, device)
        loss_sum = torch.zeros(1, dtype=torch.float64, device=device)
        state = torch.zeros(4, dtype=torch.float64, device=device)
        flag = torch.zeros(1, dtype=torch.int32, device=device)
        hist = torch.zeros(max(iters, 1), dtype=torch.float32, device=device)
        w, bias = wl.weight, wl.bias_bf16
        best = arena.best_views(name)
        target = torch.empty(seq, n, dtype=torch.bfloat16, device=device)
        pred = torch.empty_like(target)
        dpred = torch.empty_like(target)
        gq_acc = torch.empty(n, k, dtype=torch.float32, device=device) if gbs > 1 else None
        wl.refresh_wq()                                             # iteration 0 runs on qdq(W; V = 0, scales = 1)
        for it in range(iters):
            batch = batches[it]
            for j, i in enumerate(batch):
                cur = (q_all if q_all is not None else fp_all)[i]
                ops.gemm(fp_all[i], w, bias=bias, out=target)                                   # layer(org_input), no grad
                ops.gemm(cur, wl.wq, bias=bias, out=pred)                  # wl.wq is kept current by ar_fq_update
                ops.mse_fwd_bwd(pred, target, None if token_masks is None else token_masks[i], inv_numel, 1000.0, loss_sum,
                                dpred=dpred)
                ops.gemm(dpred, cur, a_mn_major=True, b_mn_major=True, out=wl.gq)          # dWq = dYᵀ·X, bf16
                if gq_acc is not None:
                    accumulate_gq(gq_acc, wl.gq, j == 0, j == len(batch) - 1)
            ops.best_update(loss_sum, inv_numel, 1.0 / float(num_elm), it, state, flag, hist)
            if self.not_use_best_mse:
                flag.fill_(1 if it == iters - 1 else 0)
            # after the flag: the update snapshots the pre-update parameters when it is set; `it` selects the lr row
            ops.fq_update(spec, w, wl.value, wl.min_scale, wl.max_scale, wl.weight_min, wl.weight_max, wl.weight_global_scale,
                          wl.gq, wl.wq, lr_tab, best_v=best["value"], best_min=best.get("min_scale"),
                          best_max=best["max_scale"], flag=flag, it=it, clamp_hi=1.0)
        if iters > 0:
            self._read_losses(res, state, hist)
            with torch.no_grad():
                lin = wl.unwrapper(arena.best_views(name))
        else:
            with torch.no_grad():
                lin = wl.unwrapper({})
        return lin


def _to_device(v, device):
    if isinstance(v, torch.Tensor):
        return v.to(device)
    if isinstance(v, (list, tuple)):
        return type(v)(_to_device(i, device) for i in v)
    return v
