"""Fixtures for the `auto_awq` / `auto_gptq` writers and the AWQ layout of `auto_round`, from the UNMODIFIED reference
(v0.15.0, imported by oracle/ref_shim.py).

TEST INFRASTRUCTURE ONLY.  Writes new files only; none of the fixtures of oracle/gen_golden.py is touched:

    python -m oracle.gen_golden_formats            # pack_awq.pt + every rtn_export_fmt_*.pt
    python -m oracle.gen_golden_formats pack       # pack_awq.pt only
"""
from __future__ import annotations

import json
import os
import sys
import tempfile

import torch

from oracle.gen_golden import GOLDEN, _weights, tiny_llama


def gen_pack_awq():
    """WQLinear_GEMM.from_linear (export_to_awq/utils.py:197-273) called the way export_to_awq/export.py:114-145 calls it:
    scales / zeros transposed to [G, N], a symmetric layer's zero-point as one python int."""
    import torch.nn as nn
    from auto_round.data_type.int import quant_tensor_asym, quant_tensor_sym
    from auto_round.export.export_to_awq.utils import WQLinear_GEMM

    out = {}
    cases = [("asym_g128", False, 128, 64, 256, False), ("asym_g32", False, 32, 24, 96, False),
             ("sym_g128", True, 128, 64, 256, False), ("asym_gm1", False, -1, 40, 160, False),
             ("asym_g64_bias", False, 64, 32, 128, True)]
    for ci, (name, sym, g, n, k, bias) in enumerate(cases):
        w = _weights(n, k, 700 + ci)
        if not sym:
            w[6, : (k if g == -1 else g)] = w[6, : (k if g == -1 else g)].abs() + 0.01     # a group with zero-point 0
        ge = k if g == -1 else g
        v = torch.rand(n * k // ge, ge, generator=torch.Generator().manual_seed(ci)) - 0.5
        wq, scale, zp = (quant_tensor_sym if sym else quant_tensor_asym)(w, bits=4, group_size=g, v=v)
        scale2 = scale.reshape(n, -1)
        zp2 = int(zp.flatten()[0]) if sym and isinstance(zp, torch.Tensor) else (int(zp) if sym else zp.reshape(n, -1))
        m = nn.Linear(k, n, bias=bias)
        m.weight.data = wq.clone()
        if bias:
            m.bias.data = torch.randn(n, generator=torch.Generator().manual_seed(9)).to(torch.bfloat16)
        zeros = zp2 if sym else zp2.t().contiguous().to(torch.float32)
        ql = WQLinear_GEMM.from_linear(m, 4, g, False, scales=scale2.t().contiguous(), zeros=zeros, device="cpu")
        out[name] = dict(wq=wq, scale=scale2, zp=zp2, group_size=g, qweight=ql.qweight, qzeros=ql.qzeros, scales=ql.scales,
                         bias_in=None if not bias else m.bias.data.clone(), bias=None if not bias else ql.bias)
        if not sym:
            assert int((zp2 == 0).sum()) > 0, name
    torch.save(out, os.path.join(GOLDEN, "pack_awq.pt"))
    print("pack_awq.pt:", {k: tuple(v["qweight"].shape) for k, v in out.items()})


def gen_rtn_export_format(tag, scheme_kwargs, fmt, layer_config=None):
    """The recorder of gen_golden.gen_rtn_export with the `format` argument: every tensor of the decoder layers, the
    `quantization_config` (the GPTQ writer also leaves it in quantize_config.json) and the saved dtype of one norm."""
    from auto_round import AutoRound
    from safetensors import safe_open

    from oracle.ref_shim import DummyTokenizer

    model = tiny_llama()
    with torch.no_grad():            # groups whose minimum is positive: asymmetric zero-point 0
        model.model.layers[0].self_attn.q_proj.weight[3, :32].abs_().add_(0.01)
        model.model.layers[1].mlp.down_proj.weight[40:48, 64:96].abs_().add_(0.01)
    init_state = {k: v.clone() for k, v in model.state_dict().items()}
    tokens = torch.randint(0, 128, (8, 16), generator=torch.Generator().manual_seed(1))
    kw = dict(scheme_kwargs)
    if layer_config:
        kw["layer_config"] = {k: dict(v) for k, v in layer_config.items()}
    with tempfile.TemporaryDirectory() as d:
        ar = AutoRound(model, tokenizer=DummyTokenizer(), iters=0, disable_opt_rtn=True, nsamples=8, seqlen=16, batch_size=4,
                       dataset=[tokens[:4], tokens[4:]], device_map="cpu", enable_torch_compile=False, seed=42, **kw)
        _, folders = ar.quantize_and_save(d, format=fmt)
        d = folders[0] if isinstance(folders, (list, tuple)) else folders
        tensors = {}
        for fn in sorted(os.listdir(d)):
            if fn.endswith(".safetensors"):
                with safe_open(os.path.join(d, fn), "pt") as f:
                    for k in f.keys():
                        tensors[k] = f.get_tensor(k)
        cfg = json.load(open(os.path.join(d, "config.json")))
        files = sorted(os.listdir(d))
    keep = {k: v for k, v in tensors.items() if ".layers." in k and "layernorm" not in k}
    rec = {"init_state": init_state, "tokens": tokens, "tensors": keep, "quantization_config": cfg["quantization_config"],
           "scheme_kwargs": scheme_kwargs, "format": fmt, "layer_config": layer_config, "files": files,
           "torch_dtype": cfg.get("torch_dtype", cfg.get("dtype")), "norm_dtype": tensors["model.norm.weight"].dtype,
           "embed_dtype": tensors["model.embed_tokens.weight"].dtype}
    torch.save(rec, os.path.join(GOLDEN, f"rtn_export_fmt_{tag}.pt"))
    print(f"rtn_export_fmt_{tag}.pt: {len(keep)} tensors; norm {rec['norm_dtype']}; config {cfg['quantization_config']}")


W4A = dict(scheme="W4A16", group_size=32, sym=False)
W4S = dict(scheme="W4A16", group_size=32)
CASES = [
    ("w4a16_asym_g32__auto_round", W4A, "auto_round", None),
    ("w4a16_asym_g32__auto_awq", W4A, "auto_awq", None),
    ("w4a16_sym_g32__auto_awq", W4S, "auto_awq", None),
    ("w4a16_sym_g32__auto_gptq", W4S, "auto_gptq", None),
    ("w2a16_asym_g32__auto_gptq", dict(scheme="W2A16", group_size=32, sym=False), "auto_gptq", None),
    ("w4a16_asym_g32_mixed8__auto_round", W4A, "auto_round", {"model.layers.1.mlp.down_proj": {"bits": 8}}),
]


def main(argv):
    from oracle.ref_shim import import_reference

    import_reference()
    what = set(argv) or {"pack", "export"}
    if "pack" in what:
        gen_pack_awq()
    if "export" in what:
        for tag, kw, fmt, lc in CASES:
            gen_rtn_export_format(tag, kw, fmt, lc)


if __name__ == "__main__":
    main(sys.argv[1:])
