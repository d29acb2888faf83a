"""Generate tests/golden/*.pt from the UNMODIFIED reference (/root/reference, v0.15.0).

TEST INFRASTRUCTURE ONLY.  Run here (build container; the reference is absent on the GPU box):

    python -m oracle.gen_golden            # all fixtures
    python -m oracle.gen_golden qdq pack   # a subset

Fixtures are small (<1 MB total) and committed together with this script.
"""
from __future__ import annotations

import os
import random
import sys

import torch

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def _weights(n, k, seed, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(n, k, generator=g) * 0.05).to(dtype)
    # edge cases: an all-zero group, a group whose +max and -min tie, exact .5 rounding ties,
    # a negative-dominant and a positive-dominant group, one huge outlier
    w[0, :16] = 0
    w[1, :32] = 0
    w[1, 0], w[1, 1] = 0.25, -0.25
    w[2, :8] = torch.tensor([0.5, -0.5, 1.5, -1.5, 2.5, -2.5, 0.0, 3.0]).to(dtype) * 0.125
    w[3, :4] = torch.tensor([-1.0, 0.2, 0.1, 0.3]).to(dtype)
    w[4, :4] = torch.tensor([1.0, -0.2, -0.1, -0.3]).to(dtype)
    w[5, 7] = 8.0
    return w


def gen_qdq():
    from auto_round.data_type.int import quant_tensor_asym, quant_tensor_rtn_sym, quant_tensor_sym
    from auto_round.data_type.mxfp import quant_mx
    from auto_round.data_type.nvfp import calculate_gparam, nv_fp4
    from auto_round.data_type.utils import reshape_pad_tensor_by_group_size

    out = {}
    cases = [
        ("int_sym_w4g128", quant_tensor_sym, dict(bits=4, group_size=128), 16, 256),
        ("int_sym_w2g32", quant_tensor_sym, dict(bits=2, group_size=32), 16, 128),
        ("int_sym_w8g64", quant_tensor_sym, dict(bits=8, group_size=64), 8, 128),
        ("int_sym_w3g128", quant_tensor_sym, dict(bits=3, group_size=128), 8, 256),
        ("int_sym_w4g128_pad", quant_tensor_sym, dict(bits=4, group_size=128), 8, 200),
        ("int_asym_w2g32", quant_tensor_asym, dict(bits=2, group_size=32), 16, 128),
        ("int_asym_w4g128", quant_tensor_asym, dict(bits=4, group_size=128), 16, 256),
        ("mx_fp4_g32", quant_mx, dict(bits=4, group_size=32, data_type="mx_fp"), 16, 128),
        ("nv_fp4_g16", nv_fp4, dict(bits=4, group_size=16), 16, 128),
    ]
    for ci, (name, fn, kw, n, k) in enumerate(cases):
        w = _weights(n, k, 100 + ci)
        grp, _, _ = reshape_pad_tensor_by_group_size(w, kw["group_size"])
        gen = torch.Generator().manual_seed(7 + ci)
        v0 = (torch.rand(grp.shape, generator=gen) - 0.5).to(torch.float32)
        mn0 = (0.5 + 0.5 * torch.rand(grp.shape[0], generator=gen)).to(torch.float32)
        mx0 = (0.5 + 0.5 * torch.rand(grp.shape[0], generator=gen)).to(torch.float32)
        gq = torch.randn(n, k, generator=gen).to(torch.float32)
        for tag, (v_, mn_, mx_) in {"init": (torch.zeros_like(v0), torch.ones_like(mn0), torch.ones_like(mx0)),
                                    "tuned": (v0, mn0, mx0)}.items():
            v = v_.clone().requires_grad_(True)
            mn = mn_.clone().requires_grad_(True)
            mx = mx_.clone().requires_grad_(True)
            extra = {}
            if name.startswith("int"):
                wmin = torch.clamp(grp.min(1)[0], max=0)
                wmax = torch.clamp(grp.max(1)[0], min=0)
                extra = dict(tensor_min=wmin, tensor_max=wmax, min_scale=mn, scale_dtype=torch.float16,
                             q_scale_thresh=1e-5)
            if name.startswith("nv"):
                extra = dict(global_scale=calculate_gparam(w, 16))
            wq, scale, zp = fn(w, v=v, max_scale=mx, **kw, **extra)
            (wq.to(torch.float32) * gq).sum().backward()
            rec = dict(w=w, v=v_.clone(), min_scale=mn_.clone(), max_scale=mx_.clone(), gq=gq, wq=wq.detach(),
                       scale=scale.detach(), zp=(zp.detach() if isinstance(zp, torch.Tensor) else zp),
                       dv=v.grad.clone(), dmax=None if mx.grad is None else mx.grad.clone(),
                       dmin=None if mn.grad is None else mn.grad.clone(), kw=kw)
            if name.startswith("nv"):
                rec["global_scale"] = extra["global_scale"]
            out[f"{name}/{tag}"] = rec
    # plain RTN (iters == 0, disable_opt_rtn): data_type/int.py:125-162
    w = _weights(16, 256, 55)
    wq, scale, zp = quant_tensor_rtn_sym(w.clone(), bits=4, group_size=128)
    out["rtn_int_sym_w4g128"] = dict(w=w, wq=wq, scale=scale, zp=zp)
    torch.save(out, os.path.join(GOLDEN, "qdq.pt"))
    print("qdq.pt:", len(out), "cases")


def gen_pack():
    import torch.nn as nn
    from auto_round.data_type.int import quant_tensor_asym, quant_tensor_sym
    from auto_round.data_type.mxfp import quant_mx
    from auto_round.data_type.nvfp import calculate_gparam, nv_fp4
    from auto_round.export.export_to_autoround.qlinear_fp import QuantLinear as FpQL
    from auto_round_extension.torch.qlinear_torch import QuantLinear as PlainQL
    from auto_round_extension.torch.qlinear_torch_zp import QuantLinear as ZpQL

    out = {}

    def lin(wq):
        m = nn.Linear(wq.shape[1], wq.shape[0], bias=False)
        m.weight.data = wq.clone()
        return m

    for bits, g, n, k in [(4, 128, 64, 256), (2, 32, 64, 128), (8, 64, 32, 128), (3, 128, 32, 256)]:
        w = _weights(n, k, 300 + bits)
        v = (torch.rand(n * k // g, g, generator=torch.Generator().manual_seed(bits)) - 0.5)
        wq, scale, zp = quant_tensor_sym(w, bits=bits, group_size=g, v=v)
        scale2 = scale.reshape(n, -1)
        ql = ZpQL(bits, g, k, n, False, g_idx=True)
        ql.pack(lin(wq), scale2.clone(), int(zp), None, "cpu")
        out[f"int_sym_w{bits}g{g}_gptq_zp"] = dict(wq=wq, scale=scale2, zp=int(zp), bits=bits, group_size=g,
                                                    qweight=ql.qweight, qzeros=ql.qzeros, scales=ql.scales,
                                                    g_idx=ql.g_idx)
    for bits, g, n, k in [(2, 32, 64, 128), (8, 64, 32, 128), (3, 128, 32, 256)]:
        w = _weights(n, k, 400 + bits)
        v = (torch.rand(n * k // g, g, generator=torch.Generator().manual_seed(bits)) - 0.5)
        wq, scale, zp = quant_tensor_asym(w, bits=bits, group_size=g, v=v)
        scale2, zp2 = scale.reshape(n, -1), zp.reshape(n, -1)
        ql = PlainQL(bits, g, k, n, False)
        ql.device = "cpu"   # export.py:205 sets this before pack()
        ql.pack(lin(wq), scale2.clone(), zp2.clone(), None, "cpu")
        out[f"int_asym_w{bits}g{g}_plain"] = dict(wq=wq, scale=scale2, zp=zp2, bits=bits, group_size=g,
                                                   qweight=ql.qweight, qzeros=ql.qzeros, scales=ql.scales)
    # FP4
    n, k = 32, 128
    w = _weights(n, k, 501)
    gs = calculate_gparam(w, 16)
    v = (torch.rand(n * k // 16, 16, generator=torch.Generator().manual_seed(1)) - 0.5)
    wq, scale, _ = nv_fp4(w, group_size=16, v=v, global_scale=gs)
    ql = FpQL(4, 16, k, n, False, data_type="nv_fp", act_bits=16)
    ql.pack(lin(wq), scale.reshape(n, -1), global_scale=gs, device="cpu")
    out["nv_fp4"] = dict(wq=wq, scale=scale.reshape(n, -1), global_scale=gs, weight_packed=ql.weight_packed,
                         weight_scale=ql.weight_scale.view(torch.uint8), weight_global_scale=ql.weight_global_scale)
    w = _weights(n, k, 502)
    v = (torch.rand(n * k // 32, 32, generator=torch.Generator().manual_seed(2)) - 0.5)
    wq, e, _ = quant_mx(w, bits=4, group_size=32, v=v, data_type="mx_fp")
    ql = FpQL(4, 32, k, n, False, data_type="mx_fp", act_bits=16)
    ql.pack(lin(wq), e.reshape(n, -1), device="cpu")
    out["mx_fp4"] = dict(wq=wq, scale=e.reshape(n, -1), weight_packed=ql.weight_packed, weight_scale=ql.weight_scale)
    torch.save(out, os.path.join(GOLDEN, "pack.pt"))
    print("pack.pt:", len(out), "cases")


# ---------------------------------------------------------------------------------------------
# whole-path fixtures: run AutoRound(...).quantize() of the reference on tiny random-init models and
# record, per block, the arguments quantize_block received, the sampled batches, every loss and
# the final per-layer qdq weight / scale / zp.
# ---------------------------------------------------------------------------------------------
def tiny_llama(seed=0, layers=2, hidden=64, inter=128, heads=4, kv=2, vocab=128):
    from transformers import LlamaConfig, LlamaForCausalLM

    torch.manual_seed(seed)
    cfg = LlamaConfig(hidden_size=hidden, intermediate_size=inter, num_hidden_layers=layers,
                      num_attention_heads=heads, num_key_value_heads=kv, vocab_size=vocab,
                      max_position_embeddings=64, rms_norm_eps=1e-5, rope_theta=10000.0,
                      tie_word_embeddings=False)
    m = LlamaForCausalLM(cfg).to(torch.bfloat16).eval()
    return m


def tiny_opt(seed=0):
    from transformers import OPTConfig, OPTForCausalLM

    torch.manual_seed(seed)
    cfg = OPTConfig(hidden_size=64, ffn_dim=128, num_hidden_layers=2, num_attention_heads=4, vocab_size=128,
                    max_position_embeddings=64, word_embed_proj_dim=64)
    return OPTForCausalLM(cfg).to(torch.bfloat16).eval()


def tiny_qwen2(seed=0):
    from transformers import Qwen2Config, Qwen2ForCausalLM

    torch.manual_seed(seed)
    cfg = Qwen2Config(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=2, vocab_size=128, max_position_embeddings=64, tie_word_embeddings=False)
    return Qwen2ForCausalLM(cfg).to(torch.bfloat16).eval()


def tiny_mixtral(seed=0):
    from transformers import MixtralConfig, MixtralForCausalLM

    torch.manual_seed(seed)
    cfg = MixtralConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4,
                        num_key_value_heads=2, vocab_size=128, max_position_embeddings=64, num_local_experts=4,
                        num_experts_per_tok=2, tie_word_embeddings=False)
    m = MixtralForCausalLM(cfg).to(torch.bfloat16).eval()
    for p in m.parameters():              # HF leaves the fused 3-D expert parameters uninitialised-small: give them signal
        if p.dim() >= 2:
            p.data.normal_(0, 0.05)
    return m


def gen_block(tag, scheme_kwargs, iters=8, nsamples=8, seqlen=16, batch_size=4, model_factory=None, save=True):
    import auto_round.algorithms.quantization.sign_round.quantizer as qz
    import auto_round.compressors.utils as cu
    from auto_round import AutoRound
    from oracle.ref_shim import DummyTokenizer

    model = (model_factory or tiny_llama)()
    init_state = {k: v.clone() for k, v in model.state_dict().items()}
    tokens = torch.randint(0, 128, (nsamples, seqlen), generator=torch.Generator().manual_seed(1))
    dataset = [tokens[i:i + batch_size] for i in range(0, nsamples, batch_size)]

    rec = {"blocks": [], "tokens": tokens, "init_state": init_state, "iters": iters, "batch_size": batch_size,
           "scheme_kwargs": scheme_kwargs}
    cur = {}

    orig_qb = qz.SignRoundQuantizer.quantize_block
    orig_next = cu.IndexSampler.next_batch
    orig_bwd = qz.SignRoundQuantizer._scale_loss_and_backward

    def detach_tree(x):
        if isinstance(x, torch.Tensor):
            return x.detach().clone()
        if isinstance(x, (list, tuple)):
            return type(x)(detach_tree(i) for i in x)
        if isinstance(x, dict):
            return {k: detach_tree(v) for k, v in x.items()}
        return x

    def qb(self, block, fp_inputs, input_others, fp_outputs, q_inputs, block_ctx, input_ids=None, **kw):
        cur.clear()
        cur.update(inputs=detach_tree(fp_inputs), others=detach_tree(input_others), fp_outputs=detach_tree(fp_outputs),
                   input_ids=detach_tree(input_ids), batches=[], losses=[],
                   block_state={k: v.clone() for k, v in block.state_dict().items()},
                   nv_gs={n: m.weight_global_scale.clone() for n, m in block.named_modules()
                          if hasattr(m, "weight_global_scale")},
                   # enable_alg_ext: the (unnormalised) importance matrix each layer holds when the tuner starts
                   imatrix={n: m.imatrix.detach().float().clone() for n, m in block.named_modules()
                            if isinstance(getattr(m, "imatrix", None), torch.Tensor)})
        r = orig_qb(self, block, fp_inputs, input_others, fp_outputs, q_inputs, block_ctx, input_ids=input_ids, **kw)
        layers = {}
        for n, m in block.named_modules():
            if type(m) is torch.nn.Linear and hasattr(m, "scale"):
                layers[n] = dict(weight=m.weight.data.clone(), scale=detach_tree(m.scale), zp=detach_tree(m.zp),
                                 gs=detach_tree(getattr(m, "weight_global_scale", None)))
        cur["layers"] = layers
        rec["blocks"].append(dict(cur))
        return r

    def nb(self):
        b = orig_next(self)
        cur["batches"].append(list(b))
        return b

    def bwd(self, scaler, loss):
        cur["losses"].append(float(loss.item()))
        return orig_bwd(self, scaler, loss)

    qz.SignRoundQuantizer.quantize_block = qb
    cu.IndexSampler.next_batch = nb
    qz.SignRoundQuantizer._scale_loss_and_backward = bwd
    try:
        ar = AutoRound(model, tokenizer=DummyTokenizer(), iters=iters, nsamples=nsamples, seqlen=seqlen,
                       batch_size=batch_size, dataset=dataset, device_map="cpu", enable_torch_compile=False,
                       seed=42, **scheme_kwargs)
        ar.quantize()
    finally:
        qz.SignRoundQuantizer.quantize_block = orig_qb
        cu.IndexSampler.next_batch = orig_next
        qz.SignRoundQuantizer._scale_loss_and_backward = orig_bwd
    if not save:
        return rec
    torch.save(rec, os.path.join(GOLDEN, f"block_{tag}.pt"))
    print(f"block_{tag}.pt: {len(rec['blocks'])} blocks, losses[0][:3] =", rec["blocks"][0]["losses"][:3])
    return rec


def gen_opt_rtn():
    """Optimized-RTN functions (iters == 0 default route): search_scales / search_nvfp4_scale / search_mx_scale behind
    opt_rtn_int_sym, opt_rtn_nv_fp4, opt_rtn_mx_fp4, with and without an importance matrix."""
    from auto_round.data_type import QUANT_FUNC_WITH_DTYPE as Q
    from auto_round.data_type.int import search_scales
    from auto_round.data_type.mxfp import search_mx_scale
    from auto_round.data_type.nvfp import calculate_gparam, search_nvfp4_scale
    from auto_round.data_type.utils import reshape_pad_tensor_by_group_size

    out = {}
    cases = [
        ("int_sym_w4g128", "opt_rtn_int_sym", dict(bits=4, group_size=128), 16, 256, "im"),
        ("int_sym_w2g32", "opt_rtn_int_sym", dict(bits=2, group_size=32), 16, 128, "im"),
        ("int_sym_w3g128", "opt_rtn_int_sym", dict(bits=3, group_size=128), 8, 256, None),
        ("int_sym_w8g64", "opt_rtn_int_sym", dict(bits=8, group_size=64), 8, 128, "im"),
        ("int_sym_w4g128_pad", "opt_rtn_int_sym", dict(bits=4, group_size=128), 8, 200, "im"),
        ("int_sym_w4g32_imzero", "opt_rtn_int_sym", dict(bits=4, group_size=32), 8, 128, "imzero"),
        ("nv_fp4_g16", "opt_rtn_nv_fp4", dict(bits=4, group_size=16), 16, 128, "im"),
        ("nv_fp4_g16_noim", "opt_rtn_nv_fp4", dict(bits=4, group_size=16), 8, 64, None),
        ("mx_fp4_g32", "opt_rtn_mx_fp4", dict(bits=4, group_size=32, data_type="mx_fp4"), 16, 128, "im"),
    ]
    for ci, (name, fname, kw, n, k, imk) in enumerate(cases):
        w = _weights(n, k, 300 + ci)
        gen = torch.Generator().manual_seed(50 + ci)
        im = None
        if imk:
            im = (torch.rand(k, generator=gen) ** 2 * 40 + 0.01).to(torch.float32)
            if imk == "imzero":
                im[:20] = 0          # group 0: > g/2 zeros -> weight-derived importance
                im[40:44] = 0        # group 1: <= g/2 zeros -> mean fill
        kwargs = dict(kw)
        if im is not None:
            kwargs["imatrix"] = im.clone()
        if "nv" in fname:
            kwargs["global_scale"] = calculate_gparam(w) * 0.9
        qdq, scale, zp = Q[fname](w.clone(), **kwargs)
        grp, _, _ = reshape_pad_tensor_by_group_size(w.clone(), kw["group_size"])
        rec = {"w": w, "imatrix": im, "kw": {k_: v for k_, v in kw.items()}, "fn": fname, "qdq": qdq, "scale": scale,
               "zp": zp if not isinstance(zp, torch.Tensor) else zp.clone(),
               "global_scale": kwargs.get("global_scale")}
        out[name] = rec
        print(name, "qdq", tuple(qdq.shape), "scale", tuple(scale.shape), scale.dtype)
    torch.save(out, os.path.join(GOLDEN, "opt_rtn.pt"))
    print("opt_rtn.pt:", len(out), "cases")


def main(argv):
    from oracle.ref_shim import import_reference

    import_reference()
    os.makedirs(GOLDEN, exist_ok=True)
    what = (set(argv) - {"rtn"}) or ({"qdq", "pack", "block", "opt"} if "rtn" not in argv else set())
    if "opt" in what:
        gen_opt_rtn()
    if "qdq" in what:
        gen_qdq()
    if "pack" in what:
        gen_pack()
    if "block" in what:
        gen_block("w4a16_sym_g32", dict(scheme="W4A16", group_size=32))
        gen_block("w2a16_asym_g32", dict(scheme="W2A16", group_size=32, sym=False))
        gen_block("nvfp4", dict(scheme="NVFP4", act_bits=16, act_data_type="float"))
        gen_block("mxfp4", dict(scheme="MXFP4", act_bits=16))
    if "arch" in what:
        # other architectures of BASELINE.json's configs: OPT (LayerNorm / ReLU / biases / learned positions) and Qwen2 (q/k/v bias)
        gen_block("opt_w4a16_sym_g32", dict(scheme="W4A16", group_size=32), model_factory=tiny_opt)
        gen_block("qwen2_nvfp4", dict(scheme="NVFP4", act_bits=16, act_data_type="float"), model_factory=tiny_qwen2)
        gen_block("mixtral_mxfp4", dict(scheme="MXFP4", act_bits=16), model_factory=tiny_mixtral)
    if "algext" in what:
        # enable_alg_ext (sign_roundv2): searched init_scale, max_scale in [0,2]; outlier-masked loss when bits < 4
        gen_block("algext_w2a16_sym_g32", dict(scheme="W2A16", group_size=32, enable_alg_ext=True))
        gen_block("algext_w4a16_sym_g32", dict(scheme="W4A16", group_size=32, enable_alg_ext=True))
        gen_block("algext_mxfp4", dict(scheme="MXFP4", act_bits=16, enable_alg_ext=True))
        gen_block("algext_nvfp4", dict(scheme="NVFP4", act_bits=16, act_data_type="float", enable_alg_ext=True))


if __name__ == "__main__":
    main(sys.argv[1:])


# ---------------------------------------------------------------------------------------------
# RTN + export fixture: the reference's own `iters=0, disable_opt_rtn=True` path through
# quantize_and_save(format="auto_round") on the tiny Llama -> every packed tensor of the checkpoint.
# Deterministic (no tuning), so the GPU path must reproduce the packed integers bit-for-bit.
# ---------------------------------------------------------------------------------------------
def gen_rtn_export(tag, scheme_kwargs, opt=False):
    import json
    import tempfile

    from auto_round import AutoRound
    from safetensors import safe_open

    from oracle.ref_shim import DummyTokenizer

    model = tiny_llama()
    init_state = {k: v.clone() for k, v in model.state_dict().items()}
    tokens = torch.randint(0, 128, (8, 16), generator=torch.Generator().manual_seed(1))
    imatrices = {}
    if opt:
        # observe (not alter) the reference: record each layer's normalised importance matrix as the optimized-RTN
        # quantizer sees it, so that the oracle / CUDA scale search can be checked layer by layer
        from auto_round.algorithms.quantization.rtn.quantizer import OptimizedRTNQuantizer

        orig_qb = OptimizedRTNQuantizer.quantize_block

        def spy(self, block, *a, **k):
            for _n, m in block.named_modules():
                if hasattr(m, "imatrix") and hasattr(m, "global_name"):
                    imatrices[m.global_name] = (m.imatrix / m.imatrix_cnt).detach().float().cpu().clone()
            return orig_qb(self, block, *a, **k)

        OptimizedRTNQuantizer.quantize_block = spy
    with tempfile.TemporaryDirectory() as d:
        ar = AutoRound(model, tokenizer=DummyTokenizer(), iters=0, disable_opt_rtn=(None if opt else True), nsamples=8, seqlen=16, batch_size=4,
                       dataset=[tokens[:4], tokens[4:]], device_map="cpu", enable_torch_compile=False, seed=42,
                       **scheme_kwargs)
        _, folders = ar.quantize_and_save(d, format="auto_round")
        d = folders[0] if isinstance(folders, (list, tuple)) else folders      # the reference appends e.g. "w4g32/"
        tensors = {}
        for fn in sorted(os.listdir(d)):
            if fn.endswith(".safetensors"):
                with safe_open(os.path.join(d, fn), "pt") as f:
                    for k in f.keys():
                        t = f.get_tensor(k)
                        tensors[k] = t.view(torch.uint8) if t.dtype == torch.float8_e4m3fn else t
        qcfg = json.load(open(os.path.join(d, "config.json")))["quantization_config"]
    if opt:
        OptimizedRTNQuantizer.quantize_block = orig_qb
    keep = {k: v for k, v in tensors.items() if ".layers." in k and "layernorm" not in k}
    rec = {"init_state": init_state, "tokens": tokens, "tensors": keep, "quantization_config": qcfg,
           "scheme_kwargs": scheme_kwargs}
    if opt:
        rec["imatrix"] = imatrices
    torch.save(rec, os.path.join(GOLDEN, f"rtn_export_{tag}.pt"))
    print(f"rtn_export_{tag}.pt: {len(keep)} tensors; config keys {sorted(qcfg)}")


if __name__ == "__main__" and "rtn" in sys.argv[1:]:
    from oracle.ref_shim import import_reference as _imp

    _imp()
    gen_rtn_export("w4a16_sym_g32", dict(scheme="W4A16", group_size=32))
    gen_rtn_export("w2a16_asym_g32", dict(scheme="W2A16", group_size=32, sym=False))
    gen_rtn_export("nvfp4", dict(scheme="NVFP4", act_bits=16, act_data_type="float"))
    gen_rtn_export("mxfp4", dict(scheme="MXFP4", act_bits=16))
    # optimized RTN (the reference's default for iters=0): imatrix from the calibration forward + scale search
    gen_rtn_export("opt_w4a16_sym_g32", dict(scheme="W4A16", group_size=32), opt=True)
    gen_rtn_export("opt_nvfp4", dict(scheme="NVFP4", act_bits=16, act_data_type="float"), opt=True)
    gen_rtn_export("opt_mxfp4", dict(scheme="MXFP4", act_bits=16), opt=True)


# ---------------------------------------------------------------------------------------------
# lm_head fixture: `quant_lm_head=True` sends the output projection through
# SignRoundQuantizer.quantize_layer_outside_block (sign_round/quantizer.py:554-759): micro-batches of one sample,
# gradients accumulated over `batch_size` samples per iteration, MSELoss(reduction="sum"), num_elm fixed before the loop.
# ---------------------------------------------------------------------------------------------
def gen_lm_head(tag, scheme_kwargs, iters=8, nsamples=8, seqlen=16, batch_size=4):
    import auto_round.algorithms.quantization.sign_round.quantizer as qz
    import auto_round.compressors.utils as cu
    from auto_round import AutoRound
    from oracle.ref_shim import DummyTokenizer

    model = tiny_llama()
    init_state = {k: v.clone() for k, v in model.state_dict().items()}
    tokens = torch.randint(0, 128, (nsamples, seqlen), generator=torch.Generator().manual_seed(1))
    dataset = [tokens[i:i + batch_size] for i in range(0, nsamples, batch_size)]
    rec = {"tokens": tokens, "init_state": init_state, "iters": iters, "batch_size": batch_size, "scheme_kwargs": scheme_kwargs,
           "layers": []}
    cur = {"active": False}
    orig_ql = qz.SignRoundQuantizer.quantize_layer_outside_block
    orig_next = cu.IndexSampler.next_batch
    orig_bwd = qz.SignRoundQuantizer._scale_loss_and_backward

    def clone_list(x):
        return None if x is None else [t.detach().clone() for t in x]

    def ql(self, layer, fp_inputs=None, q_inputs=None, disable_opt_rtn=None, input_ids=None):
        cur.update(active=True, name=layer.global_name, fp_inputs=clone_list(fp_inputs), q_inputs=clone_list(q_inputs),
                   input_ids=clone_list(input_ids), weight=layer.weight.detach().clone(),
                   bias=None if layer.bias is None else layer.bias.detach().clone(), batches=[], losses=[])
        r = orig_ql(self, layer, fp_inputs=fp_inputs, q_inputs=q_inputs, disable_opt_rtn=disable_opt_rtn, input_ids=input_ids)
        from auto_round.utils import get_module
        m = get_module(self.model, cur["name"])
        out = {k: v for k, v in cur.items() if k != "active"}
        out.update(out_weight=m.weight.detach().clone(), scale=m.scale.detach().clone() if hasattr(m, "scale") else None,
                   zp=m.zp.detach().clone() if isinstance(getattr(m, "zp", None), torch.Tensor) else getattr(m, "zp", None))
        rec["layers"].append(out)
        cur["active"] = False
        return r

    def nb(self):
        b = orig_next(self)
        if cur["active"]:
            cur["batches"].append(list(b))
        return b

    def bwd(self, scaler, loss):
        if cur["active"]:
            cur["losses"].append(float(loss.item()))
        return orig_bwd(self, scaler, loss)

    qz.SignRoundQuantizer.quantize_layer_outside_block = ql
    cu.IndexSampler.next_batch = nb
    qz.SignRoundQuantizer._scale_loss_and_backward = bwd
    try:
        ar = AutoRound(model, tokenizer=DummyTokenizer(), iters=iters, nsamples=nsamples, seqlen=seqlen, batch_size=batch_size,
                       dataset=dataset, device_map="cpu", enable_torch_compile=False, seed=42, quant_lm_head=True,
                       **scheme_kwargs)
        ar.quantize()
    finally:
        qz.SignRoundQuantizer.quantize_layer_outside_block = orig_ql
        cu.IndexSampler.next_batch = orig_next
        qz.SignRoundQuantizer._scale_loss_and_backward = orig_bwd
    torch.save(rec, os.path.join(GOLDEN, f"lm_head_{tag}.pt"))
    for lay in rec["layers"]:
        print(f"lm_head_{tag}.pt:", lay["name"], "fp_inputs", None if lay["fp_inputs"] is None else len(lay["fp_inputs"]),
              "q_inputs", None if lay["q_inputs"] is None else len(lay["q_inputs"]), "losses", lay["losses"][:3],
              "batches", lay["batches"][:2])


if __name__ == "__main__" and "lm_head" in sys.argv[1:]:
    from oracle.ref_shim import import_reference as _imp2

    _imp2()
    gen_lm_head("w4a16_sym_g32", dict(scheme="W4A16", group_size=32))
