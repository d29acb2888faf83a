"""Low-bit pack + `auto_round` checkpoint writer -- host-side mirror of
  auto_round/export/formats/backends/autoround.py:134-170      (pack_layer dispatch by scheme)
  auto_round/export/export_to_autogptq/export.py:133-185        (int sym  -> qlinear_torch_zp, zp-1 layout)
  auto_round/export/export_to_autoround/export.py:143-239       (int asym -> qlinear_torch, plain layout)
  auto_round/export/export_to_autoround/export_to_nvfp_mx.py:60-134  (fp4 -> qlinear_fp)
  auto_round/export/export_to_awq/export.py:114-227, utils.py:197-273  (int4 -> AWQ GEMM layout, `auto_awq` config)
  auto_round/export/export_to_autogptq/export.py:133-323        (int -> zp-1 layout + g_idx, `auto_gptq` config)
  auto_round/export/formats/backends/{autoround,auto_gptq,auto_awq}.py  (which layout a format + scheme resolves to)
The packing arithmetic runs in the CUDA kernels of csrc/ar_pack.cu; buffer names, dtypes and shapes are the
checkpoint wire format of the reference (SURVEY.md A.5) so that its loaders read our output unchanged.
"""
from __future__ import annotations

import json
import logging
import os
import re
from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn as nn

from . import ops
from .schemes import QuantizationScheme
from .wrapper import set_module

AUTOROUND_VERSION = "0.15.0"      # format version of the reference this writer mirrors
logger = logging.getLogger(__name__)


class QuantLinear(nn.Module):
    """Packed replacement of an nn.Linear (holder of the wire-format buffers; inference is out of scope)."""

    def __init__(self, in_features: int, out_features: int, scheme: QuantizationScheme, buffers: dict, bias=None,
                 persist_g_idx: bool = False):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        self.bits, self.group_size, self.sym, self.data_type = scheme.bits, scheme.group_size, scheme.sym, scheme.data_type
        for k, v in buffers.items():
            # g_idx is rebuilt by the loader (k // group_size): the reference's auto_round checkpoints do not carry it,
            # its auto_gptq checkpoints do (tests/golden/rtn_export_fmt_*__auto_gptq.pt)
            self.register_buffer(k, v, persistent=(k != "g_idx" or persist_g_idx))
        if bias is not None:
            self.register_buffer("bias", bias)
        else:
            self.bias = None

    def extra_repr(self):
        return f"in={self.in_features}, out={self.out_features}, bits={self.bits}, g={self.group_size}, {self.data_type}"


def packing_format_of(scheme: QuantizationScheme) -> str:
    """export_to_autoround/export.py:275-280, formats/backends/autoround.py:62-75."""
    if scheme.data_type == "int" and scheme.sym:
        return "auto_round:auto_gptq"
    if scheme.data_type in ("nv_fp", "mx_fp", "nv_fp4", "mx_fp4"):
        return "auto_round:llm_compressor"             # what v0.15.0 writes for FP4 (tests/golden/rtn_export_*.pt)
    return "auto_round"


@dataclass(frozen=True)
class ResolvedFormat:
    """What a `format=` argument means for one scheme: which writer builds the `quantization_config`, which layout the
    integer layers are packed in, and the `packing_format` an auto-round config carries."""
    writer: str                           # "auto_round" | "auto_gptq" | "auto_awq"
    layout: str                           # "auto": zp-1 words for sym, plain words for asym, FP4 bytes | "gptq" | "awq"
    packing_format: Optional[str] = None  # auto_round writer only

    @property
    def is_new_layout(self) -> bool:
        """A layout no run could produce before the AWQ / GPTQ writers existed (part of the resume signature)."""
        return self.writer != "auto_round" or self.layout != "auto"


SUPPORTED_FORMATS = ("auto_round", "auto_gptq", "gptqmodel", "auto_awq", "auto_round:auto_gptq", "auto_round:gptqmodel",
                     "auto_round:auto_awq")
GPTQ_ASYM_WARNING = ("the asymmetrical kernel of the GPTQ format may result in a noticeable accuracy drop,"
                     " particularly for 2-bit quantization and smaller models."
                     " We recommend exporting to either the AutoAWQ format ( only 4 bits) or "
                     "the AutoRound format(2/3/4/8 bits).")


def _layer_bits(cfg, default: int) -> int:
    if isinstance(cfg, QuantizationScheme):
        return cfg.bits
    return int(cfg.get("bits", default))


def resolve_format(format: Optional[str], scheme: QuantizationScheme, layer_config: Optional[dict] = None,
                   layers=()) -> ResolvedFormat:
    """formats/resolver.py:111-142 and formats/backends/{autoround,auto_gptq,auto_awq}.py: check `format` against the
    scheme and the shapes of `layers` ((full name, nn.Linear, its resolved scheme) of every layer to be quantised) and
    return what it resolves to.  Pure host logic: it runs before any GPU work, so an unsupported combination costs milliseconds, not a tuning run.
    Raises the reference's errors where it raises; where it only warns and then fails while packing (AWQ shapes), the
    pack-time error is raised here."""
    name = format or "auto_round"
    if name not in SUPPORTED_FORMATS:
        raise ValueError(f"{name} is not supported, we only support {list(SUPPORTED_FORMATS)}")
    layer_config = layer_config or {}
    is_int = scheme.data_type == "int"
    writer, _, backend = name.partition(":")
    if writer == "gptqmodel":
        writer = "auto_gptq"
    backend = {"gptqmodel": "auto_gptq"}.get(backend, backend)

    def check_scheme(fmt_name, presets, ok_bits):
        errors = []
        if scheme.bits not in ok_bits:
            errors.append(f"bits={scheme.bits}")
        if not is_int:
            errors.append(f"data_type={scheme.data_type}")
        if scheme.super_bits:
            errors.append(f"super_bits={scheme.super_bits}")
        if scheme.super_group_size:
            errors.append(f"super_group_size={scheme.super_group_size}")
        if errors:
            raise ValueError(f"{fmt_name} format support quantization scheme with {presets} but got {', '.join(errors)}, "
                             "please have a check.")

    def check_awq():
        check_scheme("auto_awq", "W4A16", (4,))
        for key, cfg in layer_config.items():
            if _layer_bits(cfg, scheme.bits) not in (4,) and _layer_bits(cfg, scheme.bits) <= 8:
                raise ValueError(f"auto_awq format support quantization scheme with W4A16 but got bits="
                                 f"{_layer_bits(cfg, scheme.bits)} for layer {key}")
        for lname, lin, sc in layers:
            g = lin.in_features if sc.group_size == -1 else sc.group_size
            if g <= 0 or lin.in_features % g != 0:
                raise ValueError(f"in_features ({lin.in_features}) shape mismatch: layer {lname}, group_size {g}")
            if lin.out_features % 8 != 0:
                raise ValueError(f"out_features ({lin.out_features}) shape mismatch: layer {lname}")

    def check_gptq():
        check_scheme("auto_gptq", "W4A16,W2A16,W3A16,W8A16,BF16,W2A16G64,W2A16G32,W4A16_MIXED", (2, 3, 4, 8, 16))
        if not scheme.sym:
            logger.warning(GPTQ_ASYM_WARNING)

    if writer == "auto_awq" or backend == "auto_awq":
        check_awq()
        return ResolvedFormat(writer, "awq", "auto_round:auto_awq" if writer == "auto_round" else None)
    if writer == "auto_gptq":
        check_gptq()
        return ResolvedFormat("auto_gptq", "gptq")
    # format == "auto_round" (the explicit auto_round:auto_gptq spelling resolves the same way, except for int4 asym)
    if is_int and not scheme.sym and scheme.bits == 4:
        if backend == "auto_gptq":
            check_gptq()
            return ResolvedFormat("auto_round", "gptq", "auto_round:auto_gptq")
        if all(_layer_bits(c, 4) == 4 or _layer_bits(c, 4) >= 16 for c in layer_config.values()):
            check_awq()
            return ResolvedFormat("auto_round", "awq", "auto_round:auto_awq")
    return ResolvedFormat("auto_round", "auto", packing_format_of(scheme))


@torch.no_grad()
def pack_linear(layer: nn.Linear, scheme: QuantizationScheme, device=None, out_device="cpu",
                fmt: Optional[ResolvedFormat] = None) -> QuantLinear:
    """Pack one tuned nn.Linear (weight = qdq weight, `.scale/.zp/.weight_global_scale` set by the tuner) in the layout
    `fmt` resolved to (default: the auto_round layouts)."""
    if not hasattr(layer, "scale"):
        raise RuntimeError("pack_linear: layer has no `.scale` (was it quantised?)")
    dev = torch.device(device) if device is not None else (layer.weight.device if layer.weight.is_cuda else torch.device("cuda"))
    wq = layer.weight.data.to(dev).to(torch.bfloat16).contiguous()
    n, k = wq.shape
    name = scheme.qdq_name
    layout = fmt.layout if fmt is not None else "auto"
    bias = None if layer.bias is None else layer.bias.detach().to(torch.float16).to(out_device)
    persist_g_idx = False
    if name in ("int_sym", "int_asym"):
        scale = layer.scale.to(dev).to(torch.float16).reshape(n, -1).contiguous()
        zp = None if name == "int_sym" else layer.zp.to(dev).to(torch.float32).reshape(n, -1).contiguous()
        zp_const = int(layer.zp) if name == "int_sym" else 0
        if layout == "awq":
            if scheme.bits != 4:
                raise NotImplementedError("Only 4-bit are supported for now.")        # export_to_awq/utils.py:144-145
            qw, qz, st = ops.pack_awq(wq, scale, zp, scheme.group_size, zp_const=zp_const)
            bufs = {"qweight": qw, "qzeros": qz, "scales": st}
        elif layout == "gptq" or name == "int_sym":
            qw, qz, st, gi = ops.pack_int(wq, scale, zp, scheme.bits, scheme.group_size, zp_minus_one=True, zp_const=zp_const)
            bufs = {"qweight": qw, "qzeros": qz, "scales": st, "g_idx": gi}
            persist_g_idx = fmt is not None and fmt.writer == "auto_gptq"
        else:
            qw, qz, st, _ = ops.pack_int(wq, scale, zp, scheme.bits, scheme.group_size, zp_minus_one=False)
            bufs = {"qweight": qw, "qzeros": qz, "scales": st}
    elif layout != "auto":
        raise ValueError(f"the {layout} layout holds integer weights only, got {name}")
    elif name == "nv_fp4":
        scale = layer.scale.to(dev).to(torch.float32).reshape(n, -1).contiguous()
        gs = layer.weight_global_scale.to(dev).to(torch.float32).reshape(1).contiguous()
        pk, sc = ops.pack_fp4_nv(wq, scale, gs)
        bufs = {"weight_packed": pk, "weight_scale": sc.view(torch.float8_e4m3fn), "weight_global_scale": gs.clone()}
    elif name == "mx_fp4":
        e = layer.scale.to(dev).to(torch.bfloat16).reshape(n, -1).contiguous()
        pk, sc = ops.pack_fp4_mx(wq, e)
        bufs = {"weight_packed": pk, "weight_scale": sc}
    else:
        raise NotImplementedError(name)
    bufs = {k_: v.to(out_device) for k_, v in bufs.items()}
    return QuantLinear(k, n, scheme, bufs, bias, persist_g_idx=persist_g_idx)


def pack_layer(name: str, model: nn.Module, scheme: QuantizationScheme, device=None, out_device="cpu",
               fmt: Optional[ResolvedFormat] = None):
    """Replace `model.<name>` by its packed QuantLinear (immediate_pack, compressors/utils.py:534-554)."""
    layer = model.get_submodule(name)
    if type(layer) is not nn.Linear or not hasattr(layer, "scale"):
        return None
    ql = pack_linear(layer, scheme, device, out_device, fmt)
    set_module(model, name, ql)
    layer.weight = None                     # release the dense weight
    return ql


def extra_config_entry(scheme: QuantizationScheme) -> dict:
    """`extra_config[layer]` of a quantised layer outside the blocks (lm_head): every QuantizationScheme field of the
    resolved per-layer config (export_to_autoround/export.py:303-306).  For the weight-only schemes in scope the reference
    resolves the activation fields to their defaults (16 bit float, dynamic, symmetric, the weight's group size)."""
    return {"act_bits": 16, "act_data_type": "float", "act_dynamic": True, "act_group_size": scheme.group_size, "act_sym": True,
            "bits": scheme.bits, "data_type": scheme.data_type, "group_size": scheme.group_size, "rotation_config": None,
            "super_bits": None, "super_group_size": None, "sym": scheme.sym}


def build_quantization_config(scheme: QuantizationScheme, block_names, extra: Optional[dict] = None, iters=200,
                              nsamples=128, seqlen=2048, batch_size=8, tuning: Optional[dict] = None,
                              packing_format: Optional[str] = None) -> dict:
    """Keys of export_to_autoround/export.py:286-336 after filter_quantization_config (export/utils.py:334-374): a
    hyper-parameter is written only when it differs from the reference's default (`iters` 200, `lr` / `minmax_lr` 1/iters,
    `enable_minmax_tuning` / `enable_quanted_input` True); nsamples / seqlen / batch_size are not part of the serialised
    config in v0.15.0 (pinned by tests/test_export_config.py against configs the reference wrote)."""
    cfg = _common_config(scheme, iters, tuning)
    cfg["block_name_to_quantize"] = block_names
    cfg["quant_method"] = "auto-round"
    cfg["packing_format"] = packing_format or packing_format_of(scheme)
    if extra:
        cfg["extra_config"] = extra
    return cfg


def _common_config(scheme: QuantizationScheme, iters, tuning: Optional[dict]) -> dict:
    """The keys every writer of the reference serialises: the scheme and the non-default hyper-parameters."""
    cfg = {"bits": scheme.bits, "group_size": scheme.group_size, "sym": scheme.sym, "data_type": scheme.data_type}
    tuning = tuning or {}
    if iters == 0:
        cfg["enable_quanted_input"] = False            # RTN route of the reference; the default (True) is filtered out
    else:
        if iters != 200:
            cfg["iters"] = int(iters)
        default_lr = 1.0 / iters
        for key in ("lr", "minmax_lr"):
            if tuning.get(key) is not None and float(tuning[key]) != default_lr:
                cfg[key] = float(tuning[key])
        for key in ("enable_minmax_tuning", "enable_quanted_input"):
            if tuning.get(key) is False:
                cfg[key] = False
    cfg["static_attention_granularity"] = "tensor"
    cfg["static_kv_granularity"] = "tensor"
    cfg["autoround_version"] = AUTOROUND_VERSION
    return cfg


def build_awq_config(scheme: QuantizationScheme, block_names, modules_to_not_convert, iters=200,
                     tuning: Optional[dict] = None) -> dict:
    """`auto_awq` (export_to_awq/export.py:192-212 after filter_quantization_config), key set pinned by
    tests/golden/rtn_export_fmt_*__auto_awq.pt.  The AWQ config has no per-layer overrides: layers left unquantised are
    listed in `modules_to_not_convert` (sorted here; the reference writes them in set order)."""
    cfg = _common_config(scheme, iters, tuning)
    cfg.update(to_quant_block_names=block_names, provider="auto-round", quant_method="awq", zero_point=not scheme.sym,
               version="gemm")
    if modules_to_not_convert:
        cfg["modules_to_not_convert"] = sorted(modules_to_not_convert)
    return cfg


def gptq_dynamic(overrides: dict) -> dict:
    """Per-layer overrides as GPTQ `dynamic` rules (export_to_autogptq/export.py:86-108): `+:regex` with the layer's
    bits / group_size / sym for a quantised layer, `-:regex` for one kept in 16 bit.  `overrides`: full layer name ->
    resolved QuantizationScheme."""
    out = {}
    for name, sc in overrides.items():
        regex = f".*{re.escape(name)}.*"                        # to_standard_regex of a plain layer name
        if sc.bits < 16:
            out[f"+:{regex}"] = {"bits": sc.bits, "group_size": sc.group_size, "sym": sc.sym}
        else:
            out[f"-:{regex}"] = {}
    return out


def build_gptq_config(scheme: QuantizationScheme, overrides: Optional[dict] = None, lm_head: bool = False,
                      modules_in_block_to_quantize=None, iters=200, tuning: Optional[dict] = None) -> dict:
    """`auto_gptq` (export_to_autogptq/export.py:232-310 after filter_quantization_config), key set pinned by
    tests/golden/rtn_export_fmt_*__auto_gptq.pt."""
    cfg = _common_config(scheme, iters, tuning)
    cfg.update(lm_head=bool(lm_head), provider="auto-round", quant_method="gptq", desc_act=False, true_sequential=False,
               damp_percent=0.01)
    if overrides:
        cfg["dynamic"] = gptq_dynamic(overrides)
    if modules_in_block_to_quantize is not None:
        cfg["modules_in_block_to_quantize"] = modules_in_block_to_quantize
    return cfg


def save_quantized(model: nn.Module, output_dir: str, quantization_config: dict, tokenizer=None, fp16: bool = False):
    """Write the checkpoint.  `fp16`: the `auto_gptq` / `auto_awq` writers store every tensor that is not packed in
    fp16 and declare `torch_dtype: float16`, what the kernels that load these formats compute in
    (export_to_awq/export.py:216-225, export_to_autogptq/export.py:314-322)."""
    os.makedirs(output_dir, exist_ok=True)
    if fp16:
        for p_ in model.parameters():
            if p_.is_floating_point():
                p_.data = p_.data.to(torch.float16)
        if hasattr(model, "config"):
            model.config.torch_dtype = torch.float16
    if hasattr(model, "config"):
        model.config.quantization_config = quantization_config
    if tokenizer is not None and hasattr(tokenizer, "save_pretrained"):
        try:
            tokenizer.save_pretrained(output_dir)
        except Exception:  # noqa: BLE001  (dummy tokenizers in tests)
            pass
    if hasattr(model, "save_pretrained"):
        model.save_pretrained(output_dir, safe_serialization=True)
    else:
        from safetensors.torch import save_file
        save_file({k: v.contiguous() for k, v in model.state_dict().items()}, os.path.join(output_dir, "model.safetensors"))
        with open(os.path.join(output_dir, "quantization_config.json"), "w") as f:
            json.dump(quantization_config, f, indent=2)
    return output_dir
