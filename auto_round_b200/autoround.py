"""`AutoRound(...)` entry point -- keeps the reference's Python surface for the block-wise tuning path
(auto_round/autoround.py:722-788; compressors/base.py:202-486, :1925-2021; compressors/orchestrator.py:176-388,
:525-816; algorithms/composer.py:360-483) while every kernel of the hot path is hand-written sm_90a CUDA.

    ar = AutoRound(model, tokenizer, scheme="W4A16", iters=200, nsamples=128, seqlen=2048, batch_size=8,
                   dataset=[LongTensor[b, seqlen], ...], device_map=0, seed=42)
    model, layer_config = ar.quantize()
    ar.quantize_and_save("out_dir", format="auto_round")

Checkpoint formats: "auto_round" (default), "auto_gptq", "auto_awq" (export.resolve_format).
Out of scope (rejected loudly, never silently emulated): activation quantisation, GGUF / MLX / llm-compressor formats,
AutoScheme, MLLM / diffusion calibration, torch.compile, CPU execution.
"""
from __future__ import annotations

import json
import logging
import os
import random
import time
from typing import Optional

import numpy as np
import torch
import torch.nn as nn

from . import export, ops
from . import resume as resume_mod
from .fused import fused_block_ops
from .moe import unfuse_experts
from .quantizer import DataParallel, SignRoundQuantizer, valid_token_masks
from .schemes import QuantizationScheme, parse_scheme
from .wrapper import set_module

logger = logging.getLogger(__name__)

_SCHEME_KW = ("bits", "group_size", "sym", "data_type", "act_bits", "act_group_size", "act_sym", "act_data_type",
              "act_dynamic", "super_bits", "super_group_size")
_SIGNROUND_KW = ("lr", "minmax_lr", "enable_minmax_tuning", "enable_quanted_input", "not_use_best_mse",
                 "enable_norm_bias_tuning", "dynamic_max_gap", "momentum", "enable_alg_ext", "disable_opt_rtn",
                 "enable_lfq", "nblocks", "quant_lm_head", "scale_dtype", "amp", "to_quant_block_names",
                 "reference_mask_cast", "use_cuda_graph", "fuse_block_ops")


class _StopForward(Exception):
    pass


def set_seed(seed: int):
    """transformers.set_seed (compressors/base.py:360): python random, numpy, torch."""
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed_all(seed)


def find_blocks(model: nn.Module):
    """utils/model.py:1380 get_block_names: the first ModuleList of decoder layers -> (prefix, ModuleList)."""
    for name, mod in model.named_modules():
        if isinstance(mod, nn.ModuleList) and len(mod) > 0 and all(isinstance(m, nn.Module) for m in mod):
            if any(isinstance(sub, nn.Linear) for sub in mod[0].modules()):
                return name, mod
    raise RuntimeError("no transformer block list found in the model")


def block_groups(nblk: int, nblocks: int) -> list:
    """Indices of the blocks tuned together: [i, min(i + nblocks, nblk)) for i = 0, nblocks, 2 nblocks, ...; the last
    group may be short (compressors/orchestrator.py:227-241)."""
    return [list(range(i, min(i + nblocks, nblk))) for i in range(0, nblk, nblocks)]


class BlockGroup(nn.Module):
    """Consecutive decoder blocks tuned as one unit (nblocks > 1): the forward feeds each member's first output to the
    next member, every member with the same kwargs, and returns the last member's output.  The members stay where they are
    in the model; the group only holds them, as `layers.<j>`."""

    def __init__(self, blocks, names):
        super().__init__()
        self.layers = nn.ModuleList(blocks)
        self.names = list(names)

    def prefix_map(self) -> dict:
        """{"layers.<j>": full name of member j}: the group-relative name of a layer -> its full module name
        (SignRoundQuantizer.layer_names)."""
        return {f"layers.{j}": n for j, n in enumerate(self.names)}

    def forward(self, hidden_states, *args, **kwargs):
        for blk in self.layers:
            out = blk(hidden_states, *args, **kwargs)
            hidden_states = out[0] if isinstance(out, (tuple, list)) else out
        return hidden_states


def repeated_tail(input_ids: torch.Tensor) -> torch.Tensor:
    """bool [b, s]: in each row, the run of positions just before the last one that hold the row's last token.  Without
    a pad token the reference takes that run for padding (calibration/llm.py:351-358, :375-389)."""
    same = input_ids[:, :-1] == input_ids[:, -1:]
    run = same.flip(1).cumprod(1).flip(1).bool()              # stays true back from the end until the first other token
    return torch.cat([run, run.new_zeros(run.shape[0], 1)], dim=1)


def label_ids_and_mask(input_ids: torch.Tensor, tokenizer):
    """One token batch [b, s] -> (label ids with -100 at every position excluded from the loss, long attention mask), the
    reference's conventions for tensor datasets (calibration/llm.py:346-398).  Padding is the pad id, or the repeated
    tail when the tokenizer has no pad id (labels) or no pad token (mask); the last position is always excluded."""
    pad_id = getattr(tokenizer, "pad_token_id", None)
    ids = input_ids.masked_fill((input_ids == pad_id) if pad_id is not None else repeated_tail(input_ids), -100)
    ids[:, -1] = -100
    if pad_id is not None and getattr(tokenizer, "pad_token", None) is not None:
        am = (input_ids != pad_id).to(torch.long)
    else:
        am = (~repeated_tail(input_ids)).to(torch.long)
    am[:, -1] = 0
    return ids, am


class _GemmLinear(nn.Module):
    """nn.Linear forward on the wgmma GEMM (used for the no-grad full-set block forwards)."""

    def __init__(self, lin: nn.Linear):
        super().__init__()
        self.lin = lin

    def forward(self, x):
        w = self.lin.weight
        x2d = x.reshape(-1, w.shape[1]).to(torch.bfloat16).contiguous()
        acc = getattr(self.lin, "_ar_imatrix", None)
        if acc is not None:
            acc.add(x, x2d)
        b = None if self.lin.bias is None else self.lin.bias.to(torch.bfloat16).contiguous()
        y = ops.gemm(x2d, w.contiguous(), bias=b)
        return y.view(*x.shape[:-1], w.shape[0])


class _ImatrixAcc:
    """Per-layer importance accumulator: sum over tokens of x^2 per input channel + the sample count
    (collect_imatrix, algorithms/quantization/rtn/quantizer.py:86-105)."""

    def __init__(self, k: int, device):
        self.sum = torch.zeros(k, dtype=torch.float32, device=device)
        self.count = torch.zeros(1, dtype=torch.float32, device=device)

    def add(self, x, x2d=None):
        if x2d is None:
            x2d = x.reshape(-1, x.shape[-1]).to(torch.bfloat16).contiguous()
        ops.imatrix_accum(x2d, self.sum)
        self.count += float(x.shape[0])                      # the reference counts input.shape[0] per call


class _collect_imatrix:
    """Context manager: while active, every listed nn.Linear of the block accumulates its importance matrix during the
    full-precision forward (register_fp_input_forward_hooks, rtn/quantizer.py:80-105)."""

    def __init__(self, block: nn.Module, names, device):
        self.lins = {n: block.get_submodule(n) for n in names}
        self.device = device
        self.handles = []

    def __enter__(self):
        for n, lin in self.lins.items():
            lin._ar_imatrix = _ImatrixAcc(lin.weight.shape[1], self.device)
            # linears that _swap_linears leaves alone (odd shapes) are reached through a regular forward hook
            self.handles.append(lin.register_forward_hook(
                lambda mod, inp, out: mod._ar_imatrix.add(inp[0] if isinstance(inp, (tuple, list)) else inp)))
        return self

    def __exit__(self, *a):
        for h in self.handles:
            h.remove()
        return False

    def finish(self, dp, normalise: bool) -> dict:
        """-> {name: importance [K] fp32}; summed over data-parallel ranks; divided by the sample count for the optimized
        RTN (rtn/quantizer.py:135-138), left as the raw sum for alg_ext (sign_roundv2/quantizer.py:413-428)."""
        out = {}
        for n, lin in self.lins.items():
            acc = lin._ar_imatrix
            del lin._ar_imatrix
            dp.all_reduce_(acc.sum, acc.count)
            if float(acc.count) == 0:
                out[n] = None                                 # never reached (e.g. an expert no token was routed to)
                continue
            out[n] = acc.sum / acc.count if normalise else acc.sum
        return out


class _swap_linears:
    """Context manager: route every bf16 nn.Linear of a block through ops.gemm, then restore."""

    def __init__(self, block: nn.Module):
        self.block = block
        self.saved = []

    def __enter__(self):
        from .moe import GroupedExperts
        grouped = tuple(n + "." for n, m in self.block.named_modules() if isinstance(m, GroupedExperts))
        for name, m in list(self.block.named_modules()):
            if name.startswith(grouped) and grouped:
                continue                     # expert linears are never called: the grouped GEMMs read their stacked weights
            if type(m) is nn.Linear and m.weight.is_cuda and m.weight.dtype == torch.bfloat16 \
                    and m.weight.shape[1] % 8 == 0 and m.weight.shape[0] % 8 == 0:
                self.saved.append((name, m))
                set_module(self.block, name, _GemmLinear(m))
        return self

    def __exit__(self, *a):
        for name, m in self.saved:
            set_module(self.block, name, m)
        return False


class AutoRound:
    def __init__(self, model, tokenizer=None, platform: str = "hf", scheme="W4A16", layer_config: Optional[dict] = None,
                 dataset=None, iters: Optional[int] = None, seqlen: int = 2048, nsamples: int = 128, batch_size: int = 8,
                 gradient_accumulate_steps: Optional[int] = None, low_gpu_mem_usage: bool = False, device_map=0,
                 enable_torch_compile: Optional[bool] = None, seed: int = 42, low_cpu_mem_usage: bool = True,
                 alg_configs=None, algorithm=None, **kwargs):
        if isinstance(model, str):
            from transformers import AutoModelForCausalLM, AutoTokenizer
            tokenizer = tokenizer or AutoTokenizer.from_pretrained(model)
            model = AutoModelForCausalLM.from_pretrained(model, torch_dtype="auto")
        if not isinstance(model, nn.Module):
            raise TypeError("model must be an nn.Module or a checkpoint path")
        if tokenizer is None:
            raise ValueError("a tokenizer object is required when `model` is a module (context/model.py:270-271)")
        if platform != "hf":
            raise NotImplementedError("only platform='hf'")
        if algorithm not in (None, "signround") or alg_configs is not None:
            raise NotImplementedError("only the default SignRound algorithm is built on H100")
        if enable_torch_compile:
            raise NotImplementedError("torch.compile is not part of the H100 path (hand-written kernels instead)")
        unknown = set(kwargs) - set(_SCHEME_KW) - set(_SIGNROUND_KW)
        if unknown:
            raise TypeError(f"unsupported AutoRound arguments for the H100 hot path: {sorted(unknown)}")
        for k in ("enable_norm_bias_tuning", "enable_lfq"):
            if kwargs.get(k):
                raise NotImplementedError(f"{k}=True is outside the H100 hot path")
        # quant_lm_head: SURVEY.md 8 f4 (quantize_layer_outside_block).  Oracle pinned against a reference run
        # (tests/golden/lm_head_*.pt); CUDA loop: quantizer.quantize_layer, GPU parity in tests/test_gpu_lm_head.py
        self.quant_lm_head = bool(kwargs.get("quant_lm_head"))
        if kwargs.get("dynamic_max_gap", -1) not in (-1, None) or kwargs.get("momentum") not in (None, 0, 0.0):
            raise NotImplementedError("dynamic_max_gap / momentum: only the reference defaults (-1 / 0)")
        nblocks = kwargs.get("nblocks", 1)
        if nblocks is None:
            nblocks = 1
        if isinstance(nblocks, bool) or not isinstance(nblocks, int) or nblocks <= 0:
            raise ValueError(f"`nblocks` must be a positive int, got {nblocks!r}")
        # nblocks > 1: SignRound tunes each run of `nblocks` consecutive blocks as one BlockGroup (one loss at the group's
        # output, one arena, one best iteration); the RTN modes (iters == 0) ignore it
        self.nblocks = nblocks
        self.model = model.eval()
        self.tokenizer = tokenizer
        self.scheme: QuantizationScheme = parse_scheme(scheme, {k: kwargs.get(k) for k in _SCHEME_KW})
        # enable_alg_ext (sign_roundv2): int asym keeps the plain wrapper in the reference (sign_roundv2/quantizer.py:334-357);
        # symmetric int / MXFP4 / NVFP4 get the searched init scale, max_scale in [0,2] and (bits < 4) the outlier-suppressed
        # loss.  For int asym the only effect is the loss: SignRoundV2Quantizer._get_loss falls back to the base MSE without
        # the valid-token mask (sign_roundv2/quantizer.py:399), which the fixtures confirm.  GPU parity: tests/test_gpu_alg_ext.py
        self.enable_alg_ext = bool(kwargs.get("enable_alg_ext"))
        self.layer_config = layer_config or {}
        self.dataset = dataset
        self.iters = 200 if iters is None else int(iters)
        self.seqlen, self.nsamples = int(seqlen), int(nsamples)
        self.batch_size = min(int(batch_size), self.nsamples)            # compressors/base.py:234-241
        self.gradient_accumulate_steps = gradient_accumulate_steps or 1
        self.low_gpu_mem_usage = low_gpu_mem_usage
        self.seed = seed
        self.sign_kw = {k: kwargs[k] for k in ("lr", "minmax_lr", "enable_minmax_tuning", "enable_quanted_input",
                                               "not_use_best_mse", "use_cuda_graph", "fuse_block_ops")
                        if k in kwargs and kwargs[k] is not None}
        # The reference casts EVERY cached non-integer block kwarg to the amp dtype (calibration/inputs.py:96-107,
        # utils/model.py:1972-2000).  Under transformers >= 5 the 4-D attention mask is boolean, so that cast turns it
        # into an additive +1/0 bias (future tokens become visible).  Default: keep the boolean mask (intended causal
        # semantics, and it enables the is_causal attention path); reference_mask_cast=True reproduces the reference
        # bit-for-bit for parity runs.
        self.reference_mask_cast = bool(kwargs.get("reference_mask_cast", False))
        self._orig_disable_opt_rtn = kwargs.get("disable_opt_rtn")
        self.disable_opt_rtn = bool(kwargs.get("disable_opt_rtn", False))
        self.device = self._resolve_device(device_map)
        if torch.cuda.is_available():
            torch.cuda.set_device(self.device)       # the C ABI launches on the current device's current stream
        self.amp_dtype = torch.bfloat16
        self.dp = self._resolve_dp()
        set_seed(seed)
        self.quantized = False
        self.block_results = []
        self.timings = {}
        self._pack_on_the_fly = False
        self._packed = False
        self._fmt = None                        # export.ResolvedFormat the layers are (to be) packed in
        self._lm_head_extra = None              # {name: extra_config entry} of layers quantized outside the blocks

    # -------------------------------------------------------------------------------------------
    @staticmethod
    def _resolve_device(device_map):
        if isinstance(device_map, torch.device):
            dev = device_map
        elif isinstance(device_map, int):
            dev = torch.device("cuda", device_map)
        elif isinstance(device_map, str):
            s = device_map.strip()
            if s in ("auto", "cuda"):
                dev = torch.device("cuda", torch.cuda.current_device() if torch.cuda.is_available() else 0)
            elif s.isdigit():
                dev = torch.device("cuda", int(s))
            else:
                dev = torch.device(s)
        else:
            raise TypeError(f"device_map {device_map!r} not supported (one GPU per process; use torchrun for DP)")
        if dev.type != "cuda":
            raise RuntimeError("auto_round_b200 runs on CUDA (sm_90a) only; there is no CPU path")
        return dev

    @staticmethod
    def _resolve_dp() -> DataParallel:
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            return DataParallel(dist.get_rank(), dist.get_world_size(), None)
        return DataParallel()

    # ------------------------------------------------------------------------------ calibration
    def _token_batches(self):
        """dataset = list of LongTensor [b, seqlen] (calibration/llm.py:305-317)."""
        ds = self.dataset
        if ds is None or isinstance(ds, str):
            raise NotImplementedError("pass `dataset` as a list of token tensors [b, seqlen]; hub datasets need network")
        if isinstance(ds, torch.Tensor):
            ds = [ds]
        total = 0
        for data in ds:
            if not isinstance(data, torch.Tensor):
                raise TypeError("dataset entries must be LongTensor [b, seqlen]")
            if data.dim() == 1:
                data = data.unsqueeze(0)
            if data.shape[-1] < self.seqlen:
                continue
            data = data[:, :self.seqlen]
            if total + data.shape[0] > self.nsamples:
                data = data[: self.nsamples - total]
            if data.shape[0] == 0:
                break
            total += data.shape[0]
            yield data
            if total >= self.nsamples:
                break

    @torch.no_grad()
    def cache_block_inputs(self, first_block: nn.Module):
        """LLMCalibrator.calib (calibration/llm.py:283-451): run the token batches through the model, capture the
        first block's inputs per sample and stop.  Reproduces the reference's mask conventions for tensor datasets:
        last key masked, trailing repeated tokens masked, and -100 at every position excluded from the loss."""
        model, dev = self.model, self.device
        captured = {"hidden": [], "kwargs": None, "per_sample": {}}
        shared = ("position_ids", "cache_position", "position_embeddings", "cu_seqlens")

        def hook(mod, args, kwargs):
            hs = args[0] if args else kwargs.get("hidden_states")
            captured["hidden"].extend(torch.split(hs.detach(), 1, dim=0))
            kw = {k: v for k, v in kwargs.items() if k != "hidden_states"}
            if captured["kwargs"] is None:
                captured["kwargs"] = {}
                for k, v in kw.items():
                    if k in shared or not isinstance(v, torch.Tensor):
                        captured["kwargs"][k] = v
            for k, v in kw.items():
                if isinstance(v, torch.Tensor) and k not in shared:
                    captured["per_sample"].setdefault(k, []).extend(torch.split(v.detach(), 1, dim=0))
            raise _StopForward

        # only what runs before the first block needs the device: everything except the other blocks
        blocks = getattr(self, "_blocks", None)
        if blocks is None:
            _, blocks = find_blocks(model)
        block_ids = {id(b) for b in blocks}
        for mod in model.modules():
            if id(mod) in block_ids:
                continue
            for p in mod.parameters(recurse=False):
                p.data = p.data.to(dev)
            for bname, b in mod.named_buffers(recurse=False):
                mod._buffers[bname] = b.to(dev)
        first_block.to(dev)
        handle = first_block.register_forward_pre_hook(hook, with_kwargs=True)
        ids_cache = []
        try:
            for data in self._token_batches():
                input_ids = data.to(dev)
                ids, am = label_ids_and_mask(input_ids, self.tokenizer)
                ids_cache.extend(torch.split(ids.cpu(), 1, dim=0))
                try:
                    with torch.autocast(device_type="cuda", dtype=self.amp_dtype):
                        model(input_ids, attention_mask=am, use_cache=False)
                except _StopForward:
                    pass
        finally:
            handle.remove()
        others = dict(captured["kwargs"] or {})
        for k, v in captured["per_sample"].items():
            if self.reference_mask_cast:
                v = [t if t.dtype in (torch.int32, torch.int64) else t.to(self.amp_dtype) for t in v]
            others[k] = v
        hidden = [h.to(self.amp_dtype) for h in captured["hidden"]]       # calibration/inputs.py:88-92
        if len(hidden) == 0:
            raise RuntimeError("no calibration samples: dataset sequences shorter than seqlen?")
        return hidden, others, ids_cache

    # ----------------------------------------------------------------------------------- forwards
    @torch.no_grad()
    def _forward_all(self, quantizer: SignRoundQuantizer, block, inputs, others, token_masks):
        """BlockForwardRunner.forward over every sample in batches of `batch_size` (algorithms/block_runner.py:171)."""
        dev = self.device
        static_kw, per_sample_kw = quantizer._prepare_others(others, token_masks, dev, block)
        outs = []
        bs = self.batch_size
        n = len(inputs)
        dp = self.dp
        # data parallel: rank r forwards its contiguous share of the samples, one all-gather rebuilds the full set
        per = (n + dp.world - 1) // dp.world
        lo, hi = (dp.rank * per, min(n, (dp.rank + 1) * per)) if dp.world > 1 else (0, n)
        with _swap_linears(block), fused_block_ops(block, quantizer.fuse_block_ops):
            for i in range(lo, hi, bs):
                j = min(i + bs, hi)
                x = torch.cat([t.to(dev) for t in inputs[i:j]], dim=0)
                kw = dict(static_kw)
                for k, v in per_sample_kw.items():
                    kw[k] = v[i:j]
                y = quantizer.block_forward(block, x, kw)
                outs.append(y.to(self.amp_dtype))
        if dp.world == 1:
            return [t for y in outs for t in torch.split(y, 1, dim=0)]
        import torch.distributed as dist
        local = torch.cat(outs, dim=0) if outs else torch.empty((0,) + tuple(inputs[0].shape[1:]), dtype=self.amp_dtype, device=dev)
        if local.shape[0] < per:                                   # last rank may own fewer samples: pad
            pad = local.new_zeros((per - local.shape[0],) + tuple(local.shape[1:]))
            local = torch.cat([local, pad], dim=0)
        full = torch.empty((per * dp.world,) + tuple(local.shape[1:]), dtype=local.dtype, device=dev)
        dist.all_gather_into_tensor(full, local.contiguous(), group=dp.group)
        return list(torch.split(full[:n], 1, dim=0))

    def _block_mse(self, outs, refs, token_masks):
        """mean over valid tokens of (out - ref)^2, fp32 accumulate (ar_mse_fwd_bwd without the gradient) -> device scalar."""
        loss = torch.zeros(1, dtype=torch.float64, device=self.device)
        hidden = outs[0].shape[-1]
        for i in range(0, len(outs), self.batch_size):
            o = torch.cat([t.to(self.device) for t in outs[i:i + self.batch_size]], dim=0).reshape(-1, hidden).contiguous()
            r = torch.cat([t.to(self.device) for t in refs[i:i + self.batch_size]], dim=0).reshape(-1, hidden).contiguous()
            m = None
            if token_masks is not None:
                m = torch.cat([t.reshape(-1) for t in token_masks[i:i + self.batch_size]]).to(torch.uint8).contiguous()
            ops.mse_fwd_bwd(o, r, m, 1.0, 1.0, loss, want_grad=False)
        if token_masks is not None:
            n_valid = torch.stack([t.sum() for t in token_masks]).sum().to(torch.float64)      # device count
        else:
            n_valid = torch.tensor(float(len(outs) * outs[0].shape[-2]), dtype=torch.float64, device=self.device)
        return (loss / (n_valid * hidden)).reshape(())

    @staticmethod
    def _fuse_nv_global_scales(block: nn.Module, names) -> dict:
        """NVFP4: q/k/v and gate/up (w1/w3) share min(global_scale) (data_type/utils.py:433-530)."""
        gs = {}
        lin = {n: block.get_submodule(n) for n in names}
        for n, m in lin.items():
            gs[n] = ops.nv_global_scale(m.weight.data.contiguous())
        groups = [("q_proj", "k_proj", "v_proj"), ("gate_proj", "up_proj"), ("w1", "w3")]
        by_parent = {}
        for n in names:
            parent, _, leaf = n.rpartition(".")
            by_parent.setdefault(parent, {})[leaf] = n
        for parent, leaves in by_parent.items():
            for grp in groups:
                members = [leaves[g] for g in grp if g in leaves]
                if len(members) >= 2:
                    shared = torch.stack([gs[m] for m in members]).min(dim=0).values
                    for m in members:
                        gs[m] = shared.clone()
        return gs

    def _hook(self, bi: int, phase: str):
        cb = getattr(self, "block_hook", None)
        if cb is not None:
            cb(bi, phase)

    # ---------------------------------------------------------------------------------- quantize
    def quantize(self):
        """Quantize the blocks one after the other.  `iters > 0` tunes every block with SignRound; `iters == 0` runs the
        RTN mode `_rtn_mode` selects.  Tuning and the calibrated optimized RTN cache the first block's inputs once and
        feed each block's full-precision outputs to the next one."""
        model = self.model
        prefix, blocks = find_blocks(model)
        self.block_prefix, self._blocks = prefix, blocks
        if self._pack_on_the_fly and self._fmt is None:
            self._fmt = self._resolve_format("auto_round")
        mode = "tune" if self.iters > 0 else self._rtn_mode()
        tune = mode == "tune"
        fp_inputs = others = ids_cache = token_masks = None
        if mode in ("tune", "calibrated_opt"):
            t_cache0 = time.time()
            fp_inputs, others, ids_cache = self.cache_block_inputs(blocks[0])
            if tune:
                torch.cuda.synchronize(self.device)
                self.timings["cache_inputs_s"] = time.time() - t_cache0
            token_masks = valid_token_masks(ids_cache, self.device)

        tune_kw = dict(enable_alg_ext=self.enable_alg_ext, gradient_accumulate_steps=self.gradient_accumulate_steps,
                       **self.sign_kw) if tune else {}                    # RTN ignores the tuning options
        quantizer = SignRoundQuantizer(self.scheme, iters=self.iters, batch_size=self.batch_size, amp_dtype=self.amp_dtype,
                                       layer_config=self.layer_config, dp=self.dp, **tune_kw)
        self.quantizer = quantizer
        t0 = time.time()                                                  # orchestrator.py:631
        q_inputs = None
        nblk = len(blocks)
        # AR_RESUME_DIR (utils/resume.py, orchestrator.py:634-676): skip the blocks a previous process finished, restore
        # their results and the two chain values, and persist the same after every block of this run
        resume, start = self._open_resume(prefix, blocks) if tune else (None, 0)
        if resume is not None and start > 0:
            fp_chain, q_chain, rng = resume.load_input_ids(), resume.load_q_input(), None
            if fp_chain is None:
                raise RuntimeError(f"AR_RESUME_DIR: manifest lists {start} finished blocks but the chained inputs are missing")
            for bj in range(start):
                snap = resume.load_block(f"{prefix}.{bj}")
                rng = snap.pop("__rng__", rng)
                quantizer.block_prefix = f"{prefix}.{bj}"
                unfuse_experts(blocks[bj])                                # snapshots hold per-expert names
                self._freeze(blocks[bj])                                  # same normalisation as the live path
                resume_mod.restore_block(blocks[bj], snap, quantizer.scheme_for)
                self.block_results.append({"block": f"{prefix}.{bj}", "resumed": True})
            fp_inputs = [t.to(self.device) for t in fp_chain]
            q_inputs = None if q_chain is None else [t.to(self.device) for t in q_chain]
            if rng is not None:                                           # the sampler continues where the dead run was
                random.setstate(rng["python"])
                torch.set_rng_state(rng["torch"])
        # The zero-shot RTN modes list every linear the layer filter accepts, so there a layer that layer_config lifts
        # above 8 bits still joins the shared NVFP4 global scale of its q/k/v or gate/up group; the calibrated modes
        # list only the layers they quantize.
        all_linears = mode in ("plain", "zero_shot_opt")
        for group in block_groups(nblk, self.nblocks if tune else 1):
            bi = group[0]
            if bi < start:
                continue
            tb = time.time()
            if self.nblocks == 1 or not tune:
                block = blocks[bi]
                quantizer.block_prefix = f"{prefix}.{bi}"                 # layer_config keys are full module names
            else:                                                         # the group is tuned as one module
                block = BlockGroup([blocks[j] for j in group], [f"{prefix}.{j}" for j in group])
                quantizer.block_prefix = block.prefix_map()
            self._hook(bi, "h2d0")
            block.to(self.device)                                         # H2D of this block's (group's) weights
            unfuse_experts(block)                                         # MoE: fused 3-D experts -> per-expert nn.Linear
            self._freeze(block)
            self._hook(bi, "compute0")
            names = [n for n, m in block.named_modules() if quantizer.layer_filter(n, m) and (all_linears or (
                     quantizer.scheme_for(n, m) is not None and quantizer.scheme_for(n, m).bits <= 8))]
            nv_gs = self._fuse_nv_global_scales(block, names) if self.scheme.qdq_name == "nv_fp4" else None
            if tune:
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
                ev[0].record()
                # (3) reference outputs of the FP block on the FP inputs  (composer.py:423-429)
                imatrices = None
                if self.enable_alg_ext and self.scheme.qdq_name != "int_asym":   # imatrix hooks on the FP-input forward,
                    # raw sums (sign_roundv2/quantizer.py:401-428); the reference collects them for asym too but never reads them
                    with _collect_imatrix(block, names, self.device) as col:
                        ref_out = self._forward_all(quantizer, block, fp_inputs, others, token_masks)
                    imatrices = col.finish(self.dp, normalise=False)
                else:
                    ref_out = self._forward_all(quantizer, block, fp_inputs, others, token_masks)
                ev[1].record()
                eff = q_inputs if (q_inputs is not None and quantizer.enable_quanted_input) else fp_inputs
                quantizer.quantize_block(block, eff, others, ref_out, q_inputs, None, input_ids=ids_cache,
                                         nv_global_scales=nv_gs, imatrices=imatrices)
                res = quantizer.last_result
                done = res.quantized_layers
                ev[2].record()
                # (6) outputs of the quantised block feed the next block (composer.py:476-481)
                if quantizer.enable_quanted_input and (group[-1] + 1 < nblk or self.quant_lm_head):
                    q_inputs = self._forward_all(quantizer, block, eff, others, token_masks)
                else:
                    q_inputs = None
                # per-block output MSE of the tuned block against the FP block over ALL samples (valid tokens only) -- the
                # second half of the headline metric; a device scalar, read back after the last block (no host sync here)
                blk_mse = self._block_mse(q_inputs, ref_out, token_masks) if q_inputs is not None else None
                fp_inputs = ref_out
                ev[3].record()
            else:
                # OptimizedRTNQuantizer (rtn/quantizer.py:72-140): the FP forward over the calibration set collects each
                # linear's importance (sum x^2 per input channel / #samples) for the weighted scale search; iters == 0
                # implies enable_quanted_input=False, so the FP outputs feed the next block (composer.py:423-429, 476-483)
                imatrices = {} if mode == "zero_shot_opt" else None
                if mode == "calibrated_opt":
                    with _collect_imatrix(block, names, self.device) as col:
                        fp_inputs = self._forward_all(quantizer, block, fp_inputs, others, token_masks)
                    imatrices = col.finish(self.dp, normalise=True)
                done = quantizer.rtn_block(block, None, nv_gs, imatrices=imatrices,
                                           is_moe=any("experts" in n for n in names))
            if self._pack_on_the_fly:                                     # immediate_pack (orchestrator.py:327-337)
                for n in done:
                    export.pack_layer(n, block, quantizer.scheme_for(n, block.get_submodule(n)), self.device,
                                      out_device=self.device, fmt=self._fmt)
            if tune:
                ev[4].record()
            self._hook(bi, "d2h0")
            block.to("cpu")                                               # packed tensors (or qdq weights) -> host
            self._hook(bi, "done")
            if tune:
                torch.cuda.synchronize(self.device)
                if resume is not None and self.dp.rank == 0:              # one writer; every rank holds identical results
                    snap = resume_mod.snapshot_block(block)
                    snap["__rng__"] = {"python": random.getstate(), "torch": torch.get_rng_state()}
                    resume.mark_block_done(f"{prefix}.{bi}", snap, q_inputs, fp_inputs)
                phases = {k: ev[i].elapsed_time(ev[i + 1])
                          for i, k in enumerate(("ref_forward_ms", "tune_ms", "q_forward_ms", "pack_ms"))}
                rec = {"block": f"{prefix}.{bi}", "init_loss": res.init_loss, "best_loss": res.best_loss,
                       "best_iter": res.best_iter, "seconds": time.time() - tb, "losses": res.losses,
                       "phases_ms": phases, "cuda_graph": res.used_cuda_graph, "batches": res.batches, "block_mse": blk_mse}
                if isinstance(block, BlockGroup):
                    rec["blocks"] = list(block.names)
                self.block_results.append(rec)
            elif mode == "calibrated_opt":
                rec = {"block": f"{prefix}.{bi}", "imatrix_layers": len(imatrices)}
                if getattr(self, "keep_imatrix", False):                  # inspection hook for the parity tests
                    rec["imatrix"] = {n: (None if t is None else t.detach().cpu()) for n, t in imatrices.items()}
                self.block_results.append(rec)
        if tune and self.quant_lm_head:
            self._quantize_lm_head(quantizer, fp_inputs, q_inputs, ids_cache)
        if not tune:
            torch.cuda.synchronize(self.device)                           # the RTN loop never waits on the device
        self.timings["tuning_s"] = time.time() - t0                      # "quantization tuning time" (orchestrator.py:792)
        for r in self.block_results:                                      # device scalars -> python floats
            if isinstance(r.get("block_mse"), torch.Tensor):
                r["block_mse"] = float(r["block_mse"])
        if resume is not None and self.dp.rank == 0:
            resume.clear()                                                # a finished run leaves no state behind
        self.quantized = True
        self._packed = self._pack_on_the_fly
        layer_cfg = {}
        if tune:                                                          # the RTN modes report no per-layer config
            quantized = lambda m: hasattr(m, "scale") or isinstance(m, export.QuantLinear)    # noqa: E731
            layer_cfg = {full: sc.to_dict() for _, _, full, sc in self._block_layers(quantized)}
        self.layer_config_out = layer_cfg
        return model, layer_cfg

    def _freeze(self, *modules: nn.Module):
        """Prepare modules for quantization: no autograd on their parameters, fp32/fp16 parameters cast to the amp dtype."""
        for mod in modules:
            for p in mod.parameters():
                p.requires_grad_(False)
                if p.dtype in (torch.float32, torch.float16):
                    p.data = p.data.to(self.amp_dtype)

    def _block_layers(self, keep):
        """(block, block-relative name, full name, resolved scheme) of every module of every block that `keep(module)`
        accepts.  While a block is walked `quantizer.block_prefix` names it, so that layer_config keys given as full
        module names resolve; the walk clears it at the end.  Modules may be replaced while the walk is suspended."""
        q = self.quantizer
        try:
            for bi, block in enumerate(self._blocks):
                q.block_prefix = f"{self.block_prefix}.{bi}"
                for n, m in list(block.named_modules()):
                    if keep(m):
                        yield block, n, f"{q.block_prefix}.{n}", q.scheme_for(n, m)
        finally:
            q.block_prefix = None

    def _find_tail(self):
        """(final norm module, output projection, its name) of a causal LM: the layers between the last block and the
        logits.  The reference discovers them with hooks on a full-model forward (orchestrator.py:549-592); here the
        block chain already holds the last block's outputs, so only the norm in between has to be applied."""
        model = self.model
        if getattr(getattr(model, "config", None), "tie_word_embeddings", False):
            raise NotImplementedError("quant_lm_head with tied input/output embeddings")
        head = getattr(model, "lm_head", None)
        if not isinstance(head, nn.Linear):
            raise NotImplementedError("quant_lm_head: the model has no nn.Linear `lm_head`")
        for path in ("model.norm", "model.final_layernorm", "transformer.ln_f", "model.decoder.final_layer_norm"):
            try:
                return model.get_submodule(path), head, "lm_head"
            except AttributeError:
                continue
        raise NotImplementedError("quant_lm_head: cannot locate the final normalisation layer of this architecture")

    def _quantize_lm_head(self, quantizer, fp_chain, q_chain, ids_cache):
        """orchestrator.py:840-930 -> quantize_layer_outside_block: tune lm_head on (norm(q chain), norm(FP chain))."""
        norm, head, name = self._find_tail()
        quantizer.block_prefix = None                 # `name` is already a full module name
        norm.to(self.device)
        head.to(self.device)
        self._freeze(norm, head)
        with torch.no_grad(), torch.autocast(device_type="cuda", dtype=self.amp_dtype):
            fp_h = [norm(t.to(self.device)).to(self.amp_dtype) for t in fp_chain]
            q_h = None if q_chain is None else [norm(t.to(self.device)).to(self.amp_dtype) for t in q_chain]
        sc = quantizer.scheme_for(name, head)
        gs = ops.nv_global_scale(head.weight.data.contiguous()) if sc.qdq_name == "nv_fp4" else None
        quantizer.quantize_layer(head, fp_h, q_h, input_ids=ids_cache, name=name, nv_global_scale=gs)
        res = quantizer.last_result
        self.block_results.append({"block": name, "init_loss": res.init_loss, "best_loss": res.best_loss,
                                   "best_iter": res.best_iter, "losses": res.losses})
        if self._pack_on_the_fly:
            export.pack_layer(name, self.model, sc, self.device, out_device=self.device, fmt=self._fmt)
        self._lm_head_extra = {name: export.extra_config_entry(sc)}
        norm.to("cpu")
        self.model.get_submodule(name).to("cpu")

    def _open_resume(self, prefix: str, blocks):
        """-> (ResumeState | None, index of the first block still to do).  Active only when AR_RESUME_DIR is set."""
        rd = os.environ.get("AR_RESUME_DIR")
        if not rd:
            return None, 0
        if self.nblocks != 1:              # orchestrator.py:226, :696-701: no resume inside or across groups
            logger.warning("AR_RESUME_DIR is set but nblocks=%d: resume state is kept only for nblocks=1, so this run "
                           "starts from block 0 and writes none", self.nblocks)
            return None, 0
        names = [f"{prefix}.{i}" for i in range(len(blocks))]
        model_id = getattr(getattr(self.model, "config", None), "_name_or_path", None)
        scheme_desc = (json.dumps(self.scheme.to_dict(), sort_keys=True, default=str) + "|"
                       + resume_mod.layer_config_fingerprint(self.layer_config)
                       + f"|iters={self.iters}|bs={self.batch_size}|seed={self.seed}|alg_ext={getattr(self, 'enable_alg_ext', False)}"
                       + f"|pack={self._pack_on_the_fly}|{sorted(self.sign_kw.items())}")
        if self._pack_on_the_fly and self._fmt is not None and self._fmt.is_new_layout:
            scheme_desc += f"|layout={self._fmt.writer}/{self._fmt.layout}"      # a resumed run cannot mix layouts
        sig = resume_mod.compute_run_signature(model_id, scheme_desc, resume_mod.dataset_fingerprint(self.dataset), self.nsamples,
                                               self.seqlen, names)
        st = resume_mod.ResumeState(os.path.join(rd, "group_0"), sig, names)
        return st, st.resume_index

    def _rtn_mode(self) -> str:
        """Which RTN the reference runs for iters == 0 (`_select_rtn_compressor_base_cls`, autoround.py:250-318, and
        get_quant_func, data_type/utils.py:139-158), pinned by tests/golden/rtn_export_*.pt:
          plain           `disable_opt_rtn=True`; int asym (no opt_rtn_* function registered); W8 int unless the user
                          passed disable_opt_rtn=False explicitly (autoround.py:269-276)
          calibrated_opt  int sym < 8 bit: calibration forward -> imatrix -> weighted scale search.  NVFP4 too: the
                          reference's routing preview still sees the preset's act_bits=4, asks for activation calibration and
                          so runs the OptimizedRTN quantizer with its imatrix hooks
          zero_shot_opt   MXFP4: no calibration, opt_rtn_mx_fp4 with imatrix=None"""
        name = self.scheme.qdq_name
        if self.disable_opt_rtn or name == "int_asym":
            return "plain"
        if name == "int_sym":
            if self.scheme.bits >= 8 and self._orig_disable_opt_rtn is None:
                return "plain"
            return "calibrated_opt"
        return "calibrated_opt" if name == "nv_fp4" else "zero_shot_opt"

    def _resolve_format(self, format: Optional[str]):
        """export.resolve_format for this run: host-only checks of `format` against the scheme, `layer_config` and the
        shapes of the linears that will be quantised (the blocks', and lm_head with quant_lm_head)."""
        base = self.scheme.to_dict()
        layers = []
        try:
            prefix, blocks = find_blocks(self.model)
        except RuntimeError:
            prefix, blocks = None, []
        named = [(f"{prefix}.{bi}.{n}", n, m) for bi, blk in enumerate(blocks) for n, m in blk.named_modules()]
        if self.quant_lm_head and isinstance(getattr(self.model, "lm_head", None), nn.Linear):
            named.append(("lm_head", "lm_head", self.model.lm_head))
        for full, rel, m in named:
            if type(m) is not nn.Linear:
                continue
            cfg = self.layer_config.get(full, self.layer_config.get(rel))
            sc = cfg if isinstance(cfg, QuantizationScheme) else QuantizationScheme.from_dict({**base, **(cfg or {})})
            if sc.bits <= 8:
                layers.append((full, m, sc))
        return export.resolve_format(format, self.scheme, self.layer_config, layers)

    def save_quantized(self, output_dir: Optional[str] = None, format: str = "auto_round", inplace: bool = True):
        fmt = self._resolve_format(format) if not self._packed else self._resolve_format_packed(format)
        if not self.quantized:
            raise RuntimeError("call quantize() first")
        if not self._packed:
            for block, n, _, sc in self._block_layers(lambda m: type(m) is nn.Linear and hasattr(m, "scale")):
                export.pack_layer(n, block, sc, self.device, fmt=fmt)
            for n in (self._lm_head_extra or {}):                           # layers tuned outside the blocks (lm_head)
                m = self.model.get_submodule(n)
                if type(m) is nn.Linear and hasattr(m, "scale"):
                    export.pack_layer(n, self.model, self.quantizer.scheme_for(n, m), self.device, fmt=fmt)
            self._packed, self._fmt = True, fmt
        tuning = dict(self.sign_kw)
        lr_used = self.quantizer.compute_lr(self.scheme.bits) if self.iters > 0 else None
        if lr_used is not None and "lr" not in tuning and lr_used != 1.0 / self.iters:
            tuning["lr"] = lr_used                    # the auto rule gave 2/iters: the reference serialises the resolved lr
            tuning.setdefault("minmax_lr", lr_used)
        if fmt.writer == "auto_round":
            extra = dict(self._lm_head_extra or {})
            extra.update(self._layer_config_overrides())
            qcfg = export.build_quantization_config(self.scheme, self.block_prefix, extra or None, self.iters,
                                                    self.nsamples, self.seqlen, self.batch_size, tuning=tuning,
                                                    packing_format=fmt.packing_format)
        elif fmt.writer == "auto_awq":
            qcfg = export.build_awq_config(self.scheme, self.block_prefix, self._unquantized_linears(), self.iters, tuning)
        else:
            qcfg = self._gptq_config(tuning)
        self.quantization_config = qcfg
        if output_dir is None:
            self.model.config.quantization_config = qcfg
            return self.model
        export.save_quantized(self.model, output_dir, qcfg, self.tokenizer, fp16=fmt.writer != "auto_round")
        return self.model

    def _resolve_format_packed(self, format: Optional[str]):
        """The layers are packed already (quantize_and_save, or an earlier save): `format` must resolve to that layout;
        packed words are not re-packed into another one."""
        fmt = self._resolve_format(format)
        have = self._fmt if self._fmt is not None else self._resolve_format("auto_round")
        if (fmt.writer == "auto_gptq") != (have.writer == "auto_gptq") or fmt.layout != have.layout:
            raise RuntimeError(f"the model is already packed for {have.writer} ({have.layout} layout); format {format!r} "
                               f"needs the {fmt.layout} layout of {fmt.writer}.  Choose the format before packing: "
                               "quantize_and_save(format=...), or quantize() then save_quantized(format=...)")
        return fmt

    def _unquantized_linears(self) -> list:
        """Full names of the nn.Linear layers the run left in 16 bit (`modules_to_not_convert` of the AWQ config,
        export_to_awq/export.py:60-111)."""
        return [n for n, m in self.model.named_modules() if type(m) is nn.Linear]

    def _gptq_config(self, tuning: dict) -> dict:
        """export_to_autogptq/export.py:232-310: per-layer overrides become `dynamic` rules, a quantised lm_head sets
        `lm_head`, and when a block layer stays unquantised the block-relative names of the quantised ones are listed."""
        base = self.scheme.to_dict()
        overrides, quantized, all_quantized = {}, set(), True
        both = lambda m: type(m) is nn.Linear or isinstance(m, export.QuantLinear)           # noqa: E731
        for block, n, full, sc in self._block_layers(both):
            if isinstance(block.get_submodule(n), export.QuantLinear):
                quantized.add(n)
            else:
                all_quantized = False
            if sc is not None and any(base.get(k) != v for k, v in sc.to_dict().items()):
                overrides[full] = sc
        for n in (self._lm_head_extra or {}):
            overrides[n] = self.quantizer.scheme_for(n, self.model.get_submodule(n))
        return export.build_gptq_config(self.scheme, overrides, bool(self._lm_head_extra),
                                        None if all_quantized else [sorted(quantized)],
                                        self.iters, tuning)

    def _layer_config_overrides(self) -> dict:
        """`extra_config` entries for block layers whose resolved scheme differs from the global one
        (export_to_autoround/export.py:303-318): full layer name -> the differing fields."""
        out = {}
        if not self.layer_config:
            return out
        base = self.scheme.to_dict()
        for _, _, full, sc in self._block_layers(lambda m: type(m) is nn.Linear or isinstance(m, export.QuantLinear)):
            if sc is None:
                continue
            diff = {k: v for k, v in sc.to_dict().items() if base.get(k) != v}
            if diff:
                out[full] = diff
        return out

    def quantize_and_save(self, output_dir: str = "tmp_autoround", format: Optional[str] = None, inplace: bool = True):
        fmt = format or "auto_round"
        self._fmt = self._resolve_format(fmt)             # rejects an unsupported combination before any GPU work
        self._pack_on_the_fly = True
        model, _ = self.quantize()
        self.save_quantized(output_dir, fmt, inplace)
        return model, [output_dir]
