"""Pins the CPU oracle (oracle/) against fixtures produced by the UNMODIFIED reference
(oracle/gen_golden.py -> tests/golden/*.pt).  Everything here is bit-exact: the oracle restates the
reference with the same torch-CPU ops in the same order."""
import os

import numpy as np
import pytest
import torch

from oracle import pack as P
from oracle import qdq as Q
from oracle import signround as S


def _same(a, b):
    """bit-equality that also accepts NaN==NaN (the reference yields NaN d(max_scale) for an all-zero
    NVFP4 group: 0 * inf in its autograd graph)."""
    return a.shape == b.shape and torch.equal(torch.isnan(a), torch.isnan(b)) and \
        torch.equal(torch.nan_to_num(a, nan=0.0), torch.nan_to_num(b, nan=0.0))


def _load(golden_dir, name):
    return torch.load(os.path.join(golden_dir, name), weights_only=False)


def _run_qdq(name, rec):
    kw = rec["kw"]
    w = rec["w"]
    v = rec["v"].clone().requires_grad_(True)
    mn = rec["min_scale"].clone().requires_grad_(True)
    mx = rec["max_scale"].clone().requires_grad_(True)
    if name.startswith("int_sym"):
        wmin, wmax = Q.group_minmax(w, kw["group_size"])
        out = Q.int_sym(w, kw["bits"], kw["group_size"], v, mn, mx, wmin, wmax)
    elif name.startswith("int_asym"):
        wmin, wmax = Q.group_minmax(w, kw["group_size"])
        out = Q.int_asym(w, kw["bits"], kw["group_size"], v, mn, mx, wmin, wmax)
    elif name.startswith("mx"):
        out = Q.mx_fp4(w, kw["group_size"], v, mx)
    else:
        out = Q.nv_fp4(w, kw["group_size"], v, rec["global_scale"], mx)
    wq, scale, zp = out
    (wq.to(torch.float32) * rec["gq"]).sum().backward()
    return wq.detach(), scale.detach(), zp, v.grad, mn.grad, mx.grad


def test_qdq_matches_reference_bit_exact(golden_dir):
    gold = _load(golden_dir, "qdq.pt")
    n = 0
    for key, rec in gold.items():
        if key.startswith("rtn"):
            continue
        name = key.split("/")[0]
        wq, scale, zp, dv, dmn, dmx = _run_qdq(name, rec)
        assert torch.equal(wq, rec["wq"]), key
        assert torch.equal(scale.float(), rec["scale"].float()), key
        if isinstance(rec["zp"], torch.Tensor):
            assert torch.equal(zp.detach(), rec["zp"]), key
        else:
            assert zp == rec["zp"], key
        assert _same(dv, rec["dv"]), key
        if rec["dmax"] is not None:
            assert _same(dmx, rec["dmax"]), key
        if rec["dmin"] is not None:
            assert _same(dmn, rec["dmin"]), key
        else:
            assert dmn is None, key
        n += 1
    assert n >= 18


def test_rtn_matches_reference(golden_dir):
    rec = _load(golden_dir, "qdq.pt")["rtn_int_sym_w4g128"]
    wq, scale, zp = Q.rtn_int_sym(rec["w"].clone(), 4, 128)
    assert torch.equal(wq, rec["wq"]) and torch.equal(scale, rec["scale"]) and zp == rec["zp"]


def test_cast_to_fp4_known_answers():
    # reference table: test/unit/test_cpu/data_type/test_nvfp.py:75-80 and data_type/nvfp.py:440-447
    x = torch.tensor([0.0, 0.24, 0.25, 0.26, 0.75, 1.25, 1.75, 2.5, 3.5, 5.0, 7.0, -0.75, -2.5, -5.0])
    want = torch.tensor([0.0, 0.0, 0.0, 0.5, 1.0, 1.0, 2.0, 2.0, 4.0, 4.0, 6.0, -1.0, -2.0, -4.0])
    assert torch.equal(Q.cast_to_fp4(x), want)


def test_nv_global_scale_formula():
    # calculate_gparam = 448*6/amax (test_nvfp.py:174-179)
    w = torch.tensor([[0.5, -2.0, 1.0]])
    assert float(Q.nv_global_scale(w)) == pytest.approx(448.0 * 6.0 / 2.0)
    assert float(Q.nv_global_scale(0.0)) == 0.0


def test_fp4_nibble_known_answers():
    # test/unit/test_cpu/export/test_qlinear_fp_helpers.py:174-221
    assert P._two_per_byte(P.fp4_nibbles(torch.tensor([[6.0, 6.0]])))[0, 0] == 0x77
    assert P._two_per_byte(P.fp4_nibbles(torch.tensor([[-6.0, -6.0]])))[0, 0] == 0xFF
    assert P._two_per_byte(P.fp4_nibbles(torch.tensor([[0.5, 0.5]])))[0, 0] == 0x11
    assert P._two_per_byte(P.fp4_nibbles(torch.tensor([[0.0, -0.0]])))[0, 0] == 0x80


def test_pack_matches_reference_bit_exact(golden_dir):
    gold = _load(golden_dir, "pack.pt")
    for key, rec in gold.items():
        if key.startswith("int"):
            out = P.pack_int(rec["wq"], rec["scale"], rec["zp"], rec["bits"], rec["group_size"],
                             zp_minus_one=key.endswith("gptq_zp"))
            assert np.array_equal(out["qweight"], rec["qweight"].numpy()), key
            assert np.array_equal(out["qzeros"], rec["qzeros"].numpy()), key
            assert np.array_equal(out["scales"], rec["scales"].numpy()), key
            if "g_idx" in rec:
                assert np.array_equal(out["g_idx"], rec["g_idx"].numpy()), key
        elif key == "nv_fp4":
            out = P.pack_nvfp4(rec["wq"], rec["scale"], rec["global_scale"])
            assert np.array_equal(out["weight_packed"], rec["weight_packed"].numpy())
            assert np.array_equal(out["weight_scale"], rec["weight_scale"].numpy())
            assert np.array_equal(out["weight_global_scale"], rec["weight_global_scale"].numpy())
        else:
            out = P.pack_mxfp4(rec["wq"], rec["scale"])
            assert np.array_equal(out["weight_packed"], rec["weight_packed"].numpy())
            assert np.array_equal(out["weight_scale"], rec["weight_scale"].numpy())


def test_pack_unpack_roundtrip():
    codes = np.random.default_rng(0).integers(0, 16, size=(64, 256)).astype(np.int32)
    assert np.array_equal(P.unpack_int(P._pack_rows_pow2(codes, 4).T.copy(), 4), codes)


SCHEMES = {
    "w4a16_sym_g32": S.LayerScheme(4, 32, True, "int"),
    "w2a16_asym_g32": S.LayerScheme(2, 32, False, "int"),
    "nvfp4": S.LayerScheme(4, 16, True, "nv_fp"),
    "mxfp4": S.LayerScheme(4, 32, True, "mx_fp"),
}


def _tiny_block(state):
    from transformers import LlamaConfig
    from transformers.models.llama.modeling_llama import LlamaDecoderLayer

    cfg = LlamaConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=2, vocab_size=128, max_position_embeddings=64, rms_norm_eps=1e-5,
                      rope_theta=10000.0, tie_word_embeddings=False)
    cfg._attn_implementation = "sdpa"
    blk = LlamaDecoderLayer(cfg, 0).to(torch.bfloat16).eval()
    blk.load_state_dict(state)
    return blk


@pytest.mark.parametrize("tag", list(SCHEMES))
def test_tune_block_matches_reference_bit_exact(golden_dir, tag):
    rec = _load(golden_dir, f"block_{tag}.pt")
    sc = SCHEMES[tag]
    for b in rec["blocks"]:
        blk = _tiny_block(b["block_state"])
        masks = [(ids != -100).to(torch.long) for ids in b["input_ids"]]
        res = S.tune_block(blk, b["inputs"], b["others"], b["fp_outputs"], lambda n, m: sc, iters=rec["iters"],
                           batch_size=rec["batch_size"], token_masks=masks, nv_global_scales=b["nv_gs"] or None,
                           sampler=S.ReplaySampler(b["batches"]))
        # the fixture logs the raw mean loss (before /num_elm); compare via the same normalisation
        assert len(res.losses) == len(b["losses"])
        nvalid = [sum(int(masks[i].sum()) for i in batch) for batch in b["batches"]]
        got = [l * n for l, n in zip(res.losses, nvalid)]
        assert got == pytest.approx(b["losses"], rel=1e-6)
        for name, lay in b["layers"].items():
            mod = blk.get_submodule(name)
            assert torch.equal(mod.weight.data, lay["weight"]), (tag, name)
            assert torch.equal(mod.scale.float().reshape(-1), lay["scale"].float().reshape(-1)), (tag, name)
            if isinstance(lay["zp"], torch.Tensor):
                assert torch.equal(mod.zp.reshape(-1), lay["zp"].reshape(-1)), (tag, name)


ALGEXT = {
    "algext_w2a16_sym_g32": S.LayerScheme(2, 32, True, "int"),      # init scale + outlier-masked loss
    "algext_w4a16_sym_g32": S.LayerScheme(4, 32, True, "int"),      # init scale only
    "algext_mxfp4": S.LayerScheme(4, 32, True, "mx_fp"),
    "algext_nvfp4": S.LayerScheme(4, 16, True, "nv_fp"),
    # int asym keeps the plain wrapper; the only effect of enable_alg_ext is the loss over ALL tokens (BASELINE config 3)
    "algext_w2a16_asym_g32": S.LayerScheme(2, 32, False, "int"),
}


@pytest.mark.parametrize("tag", list(ALGEXT))
def test_tune_block_alg_ext_matches_reference_bit_exact(golden_dir, tag):
    """enable_alg_ext=True (sign_roundv2): searched init_scale, max_scale in [0,2], outlier-masked loss for bits < 4."""
    rec = _load(golden_dir, f"block_{tag}.pt")
    sc = ALGEXT[tag]
    for b in rec["blocks"]:
        assert len(b["imatrix"]) == 7
        blk = _tiny_block(b["block_state"])
        masks = [(ids != -100).to(torch.long) for ids in b["input_ids"]]
        res = S.tune_block(blk, b["inputs"], b["others"], b["fp_outputs"], lambda n, m: sc, iters=rec["iters"],
                           batch_size=rec["batch_size"], token_masks=masks, nv_global_scales=b["nv_gs"] or None,
                           sampler=S.ReplaySampler(b["batches"]), alg_ext=True, imatrices=b["imatrix"])
        nvalid = [sum(int(masks[i].sum()) for i in batch) for batch in b["batches"]]
        got = [l * n for l, n in zip(res.losses, nvalid)]
        assert got == pytest.approx(b["losses"], rel=1e-6)
        for name, lay in b["layers"].items():
            mod = blk.get_submodule(name)
            assert torch.equal(mod.weight.data, lay["weight"]), (tag, name)
            assert torch.equal(mod.scale.float().reshape(-1), lay["scale"].float().reshape(-1)), (tag, name)


def test_index_sampler_is_python_random():
    import random

    random.seed(42)
    s = S.IndexSampler(8, 4)
    got = [s.next_batch() for _ in range(4)]
    random.seed(42)
    idx = list(range(8))
    random.shuffle(idx)
    assert got[0] == idx[:4] and got[1] == idx[4:]
    random.shuffle(idx)
    assert got[2] == idx[:4]


def test_tune_layer_lm_head_matches_reference_bit_exact(golden_dir):
    """quant_lm_head=True -> quantize_layer_outside_block (sign_round/quantizer.py:554-759): every micro-batch loss of the
    8 iterations and the final lm_head weight / scale."""
    rec = _load(golden_dir, "lm_head_w4a16_sym_g32.pt")
    assert len(rec["layers"]) == 1
    lay = rec["layers"][0]
    n, k = lay["weight"].shape
    lin = torch.nn.Linear(k, n, bias=lay["bias"] is not None).to(torch.bfloat16)
    lin.weight.data.copy_(lay["weight"])
    masks = [(ids != -100).to(torch.long) for ids in lay["input_ids"]]
    res = S.tune_layer(lin, lay["fp_inputs"], lay["q_inputs"], S.LayerScheme(4, 32, True, "int"), iters=rec["iters"],
                       batch_size=rec["batch_size"], token_masks=masks, sampler=S.ReplaySampler(lay["batches"]))
    assert res.micro_losses == pytest.approx(lay["losses"], rel=1e-6)
    assert torch.equal(lin.weight.data, lay["out_weight"])
    assert torch.equal(lin.scale.float().reshape(-1), lay["scale"].float().reshape(-1))


def test_iters1000_low_bit_lr_rule_matches_reference(golden_dir):
    """BASELINE.json config 3 hyper-parameters on the tiny Llama: W2A16 asym g32, enable_alg_ext, iters=1000 -> lr = 2/iters
    (bits <= 3 and iters >= 1000, sign_round/config.py:107-136), LinearLR over 1000 steps in the lr tensor's fp32, loss over
    every token.  All 1000 losses and the final weights of block 0, bit for bit."""
    rec = _load(golden_dir, "block_w2a16_asym_g32_iters1000.pt")
    assert rec["iters"] == 1000
    sc = S.LayerScheme(2, 32, False, "int")
    b = rec["blocks"][0]
    blk = _tiny_block(b["block_state"])
    masks = [(ids != -100).to(torch.long) for ids in b["input_ids"]]
    res = S.tune_block(blk, b["inputs"], b["others"], b["fp_outputs"], lambda n, m: sc, iters=1000, batch_size=rec["batch_size"],
                       token_masks=masks, sampler=S.ReplaySampler(b["batches"]), alg_ext=True, imatrices=b["imatrix"])
    nvalid = [sum(int(masks[i].sum()) for i in batch) for batch in b["batches"]]
    got = [l * n for l, n in zip(res.losses, nvalid)]
    assert got == pytest.approx(b["losses"], rel=1e-6)
    for name, lay in b["layers"].items():
        assert torch.equal(blk.get_submodule(name).weight.data, lay["weight"]), name


def _arch_block(arch, state):
    """Decoder layer of the tiny OPT / Qwen2 the fixtures were generated on (oracle/gen_golden.py tiny_opt / tiny_qwen2)."""
    if arch == "opt":
        from transformers import OPTConfig
        from transformers.models.opt.modeling_opt import OPTDecoderLayer

        cfg = OPTConfig(hidden_size=64, ffn_dim=128, num_hidden_layers=2, num_attention_heads=4, vocab_size=128,
                        max_position_embeddings=64, word_embed_proj_dim=64)
        cfg._attn_implementation = "sdpa"
        blk = OPTDecoderLayer(cfg, layer_idx=0)
    else:
        from transformers import Qwen2Config
        from transformers.models.qwen2.modeling_qwen2 import Qwen2DecoderLayer

        cfg = Qwen2Config(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4,
                          num_key_value_heads=2, vocab_size=128, max_position_embeddings=64, tie_word_embeddings=False)
        cfg._attn_implementation = "sdpa"
        blk = Qwen2DecoderLayer(cfg, 0)
    blk = blk.to(torch.bfloat16).eval()
    blk.load_state_dict(state)
    return blk


@pytest.mark.parametrize("arch,tag,sc", [("opt", "opt_w4a16_sym_g32", S.LayerScheme(4, 32, True, "int")),
                                          ("qwen2", "qwen2_nvfp4", S.LayerScheme(4, 16, True, "nv_fp"))])
def test_tune_block_other_architectures_match_reference_bit_exact(golden_dir, arch, tag, sc):
    """BASELINE.json configs 0 and 3: OPT (LayerNorm, ReLU, biases, attention-mask-only kwargs) and Qwen2 (q/k/v bias, NVFP4
    with the fused q/k/v and gate/up global scales) through the same oracle loop."""
    rec = _load(golden_dir, f"block_{tag}.pt")
    for b in rec["blocks"]:
        blk = _arch_block(arch, b["block_state"])
        masks = [(ids != -100).to(torch.long) for ids in b["input_ids"]]
        res = S.tune_block(blk, b["inputs"], b["others"], b["fp_outputs"], lambda n, m: sc, iters=rec["iters"],
                           batch_size=rec["batch_size"], token_masks=masks, nv_global_scales=b["nv_gs"] or None,
                           sampler=S.ReplaySampler(b["batches"]))
        nvalid = [sum(int(masks[i].sum()) for i in batch) for batch in b["batches"]]
        got = [l * n for l, n in zip(res.losses, nvalid)]
        assert got == pytest.approx(b["losses"], rel=1e-6)
        for name, lay in b["layers"].items():
            mod = blk.get_submodule(name)
            assert torch.equal(mod.weight.data, lay["weight"]), (tag, name)
            assert torch.equal(mod.scale.float().reshape(-1), lay["scale"].float().reshape(-1)), (tag, name)


def test_tune_block_mixtral_moe_matches_reference_bit_exact(golden_dir):
    """BASELINE.json config 5 (Mixtral, MXFP4 weight-only) on a tiny 4-expert block: the reference un-fuses the fused 3-D
    expert parameters into per-expert linears (modeling/fused_moe/moe_experts_interface.py:173-260).  The block here is built
    with the oracle's restatement of that un-fusing and expert loop (oracle/moe_loop.py), so a bit-exact replay of the
    reference's 8 iterations pins it and the oracle loop on ragged expert batches (experts that see no token get no update);
    the product's grouped wgmma path (auto_round_b200/moe.py) is checked against it on the GPU (tests/test_gpu_moe.py)."""
    from transformers import MixtralConfig
    from transformers.models.mixtral.modeling_mixtral import MixtralDecoderLayer

    from oracle.moe_loop import unfuse_experts_cpu as unfuse_experts

    rec = _load(golden_dir, "block_mixtral_mxfp4.pt")
    sc = S.LayerScheme(4, 32, True, "mx_fp")
    cfg = MixtralConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4,
                        num_key_value_heads=2, vocab_size=128, max_position_embeddings=64, num_local_experts=4,
                        num_experts_per_tok=2, tie_word_embeddings=False)
    cfg._attn_implementation = "sdpa"
    for b in rec["blocks"]:
        blk = MixtralDecoderLayer(cfg, 0).to(torch.bfloat16).eval()
        assert unfuse_experts(blk) == 1
        blk.load_state_dict(b["block_state"])
        masks = [(ids != -100).to(torch.long) for ids in b["input_ids"]]
        res = S.tune_block(blk, b["inputs"], b["others"], b["fp_outputs"], lambda n, m: sc, iters=rec["iters"],
                           batch_size=rec["batch_size"], token_masks=masks, sampler=S.ReplaySampler(b["batches"]))
        assert len(b["layers"]) == 16
        nvalid = [sum(int(masks[i].sum()) for i in batch) for batch in b["batches"]]
        got = [l * n for l, n in zip(res.losses, nvalid)]
        assert got == pytest.approx(b["losses"], rel=1e-6)
        for name, lay in b["layers"].items():
            mod = blk.get_submodule(name)
            assert torch.equal(mod.weight.data, lay["weight"]), name
            assert torch.equal(mod.scale.float().reshape(-1), lay["scale"].float().reshape(-1)), name


def test_reference_ste_and_reshape_unit_tests_on_the_oracle():
    """The assertions of the reference's own test/unit/test_cuda/data_type/test_ste.py (grad flow through the straight-through
    helpers, pad / revert of the group reshape for group sizes 4, 0, -1 and 3-D inputs), restated against oracle/qdq.py."""
    x = torch.randn(4, 8, requires_grad=True)
    for fn in (Q.round_ste, Q.floor_ste, Q.e4m3_ste):
        fn(x).sum().backward()
        assert torch.all(x.grad == 1.0)
        x.grad = None
    v = torch.tensor([1.2, 2.7, -0.5], requires_grad=True)
    y = Q.round_ste(v)
    assert torch.equal(y, v.round())
    y.sum().backward()
    assert torch.equal(v.grad, torch.ones_like(v))
    t = torch.arange(0, 30, dtype=torch.float32).reshape(3, 10)
    out, shape, pad = Q.to_groups(t, 4)
    assert pad == 2 and tuple(out.shape) == (9, 4) and torch.equal(Q.from_groups(out, shape, pad), t)
    t3 = torch.randn(3, 4, 8)
    out, shape, pad = Q.to_groups(t3, 0)
    assert pad == 0 and tuple(out.shape) == (1, t3.numel()) and torch.equal(Q.from_groups(out, shape, pad), t3)
    t2 = torch.randn(3, 8)
    out, shape, pad = Q.to_groups(t2, -1)
    assert pad == 0 and out is t2
    t4 = torch.randn(2, 3, 10)
    out, shape, pad = Q.to_groups(t4, 4)
    assert pad == 2 and torch.equal(Q.from_groups(out, shape, pad), t4)
