"""Checkpoints in the AWQ / GPTQ layouts on the GPU: for every tests/golden/rtn_export_fmt_*.pt (written by the
unmodified reference, oracle/gen_golden_formats.py) `quantize_and_save(format=...)` writes the same tensor names, dtypes,
shapes and bytes and the same quantization_config; a tuned int4-asymmetric run saves and unpacks to the tuner's weights."""
import json
import os

import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("CUDA device required", allow_module_level=True)

from auto_round_b200 import AutoRound, ops  # noqa: E402

DEV = torch.device("cuda", 0)
FIXTURES = ["w4a16_asym_g32__auto_round", "w4a16_asym_g32__auto_awq", "w4a16_sym_g32__auto_awq", "w4a16_sym_g32__auto_gptq",
            "w2a16_asym_g32__auto_gptq", "w4a16_asym_g32_mixed8__auto_round"]


class _Tok:
    pad_token_id = None
    pad_token = None

    def save_pretrained(self, *a, **k):
        return None


def _tiny_llama(state):
    from transformers import LlamaConfig, LlamaForCausalLM

    cfg = LlamaConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=2, vocab_size=128, max_position_embeddings=64, rms_norm_eps=1e-5,
                      rope_theta=10000.0, tie_word_embeddings=False)
    model = LlamaForCausalLM(cfg).to(torch.bfloat16).eval()
    model.load_state_dict(state)
    return model


def _read(out):
    from safetensors import safe_open

    got = {}
    with safe_open(os.path.join(out, "model.safetensors"), "pt") as f:
        for k in f.keys():
            got[k] = f.get_tensor(k)
    return got, json.load(open(os.path.join(out, "config.json")))


@pytest.mark.parametrize("tag", FIXTURES)
def test_rtn_checkpoint_bit_exact(golden_dir, tag, tmp_path):
    rec = torch.load(os.path.join(golden_dir, f"rtn_export_fmt_{tag}.pt"), weights_only=False)
    model = _tiny_llama(rec["init_state"])
    ar = AutoRound(model, tokenizer=_Tok(), iters=0, disable_opt_rtn=True, nsamples=8, seqlen=16, batch_size=4, dataset=None,
                   device_map=0, seed=42, layer_config=rec["layer_config"], **rec["scheme_kwargs"])
    out = str(tmp_path / "ckpt")
    ar.quantize_and_save(out, format=rec["format"])
    got, cfg = _read(out)
    for k, ref in rec["tensors"].items():
        assert k in got, k
        assert got[k].dtype == ref.dtype and tuple(got[k].shape) == tuple(ref.shape), k
        assert torch.equal(got[k], ref), k
    extra = {k for k in got if ".layers." in k and "layernorm" not in k} - set(rec["tensors"])
    assert not extra, extra
    assert cfg["quantization_config"] == rec["quantization_config"]
    if rec["format"] in ("auto_awq", "auto_gptq"):
        # these writers declare float16 and store the tensors that are not packed in it
        assert rec["torch_dtype"] == "float16" and cfg.get("torch_dtype", cfg.get("dtype")) == "float16"
        assert got["model.norm.weight"].dtype == torch.float16 and got["model.embed_tokens.weight"].dtype == torch.float16
    else:
        assert got["model.norm.weight"].dtype == torch.bfloat16


def _tuned_w4_asym(golden_dir, **kw):
    rec = torch.load(os.path.join(golden_dir, "rtn_export_fmt_w4a16_asym_g32__auto_round.pt"), weights_only=False)
    model = _tiny_llama(rec["init_state"])
    tokens = rec["tokens"]
    return AutoRound(model, tokenizer=_Tok(), iters=4, nsamples=8, seqlen=16, batch_size=4, dataset=[tokens[:4], tokens[4:]],
                     device_map=0, seed=42, scheme="W4A16", group_size=32, sym=False, **kw)


def test_tuned_int4_asym_saves_and_unpacks_to_the_tuned_weights(golden_dir, tmp_path):
    ar = _tuned_w4_asym(golden_dir)
    model, _ = ar.quantize()
    tuned = {n: m.weight.data.detach().to(torch.bfloat16).cpu() for n, m in model.named_modules()
             if type(m) is nn.Linear and hasattr(m, "scale")}
    assert len(tuned) == 14
    with pytest.raises(ValueError, match="is not supported"):          # a rejected format packs nothing
        ar.save_quantized(str(tmp_path / "bad"), format="gguf:q4_0")
    assert type(model.model.layers[0].self_attn.q_proj) is nn.Linear and not os.path.exists(tmp_path / "bad")
    out = str(tmp_path / "ckpt")
    ar.save_quantized(out, format="auto_round")
    got, cfg = _read(out)
    assert cfg["quantization_config"]["packing_format"] == "auto_round:auto_awq"
    assert cfg["quantization_config"]["iters"] == 4 and cfg["quantization_config"]["sym"] is False
    for name, w in tuned.items():
        n, k = w.shape
        qw, qz, st = (got[f"{name}.{key}"].to(DEV) for key in ("qweight", "qzeros", "scales"))
        assert tuple(qw.shape) == (k, n // 8) and tuple(qz.shape) == (k // 32, n // 8) and f"{name}.g_idx" not in got
        back, _ = ops.unpack_awq(qw, qz, st, n, k, 32)
        assert torch.equal(back.cpu(), w), name
    # the words are packed: another layout is refused, the same one (under its own config) is not
    with pytest.raises(RuntimeError, match="already packed"):
        ar.save_quantized(str(tmp_path / "gptq"), format="auto_gptq")
    ar.save_quantized(str(tmp_path / "awq"), format="auto_awq")
    got2, cfg2 = _read(str(tmp_path / "awq"))
    assert cfg2["quantization_config"]["quant_method"] == "awq" and cfg2["quantization_config"]["zero_point"] is True
    assert all(torch.equal(got2[k], got[k]) for k in got if k.endswith(("qweight", "qzeros")))


def test_quant_lm_head_is_packed_in_the_awq_layout(golden_dir, tmp_path):
    ar = _tuned_w4_asym(golden_dir, quant_lm_head=True)
    out = str(tmp_path / "ckpt")
    ar.quantize_and_save(out, format="auto_awq")
    got, cfg = _read(out)
    assert tuple(got["lm_head.qweight"].shape) == (64, 128 // 8) and got["lm_head.qweight"].dtype == torch.int32
    assert tuple(got["lm_head.qzeros"].shape) == (2, 16) and tuple(got["lm_head.scales"].shape) == (2, 128)
    assert "lm_head.weight" not in got and "lm_head.g_idx" not in got
    assert "modules_to_not_convert" not in cfg["quantization_config"]
    codes = ops.unpack_awq(got["lm_head.qweight"].to(DEV), got["lm_head.qzeros"].to(DEV), got["lm_head.scales"].to(DEV),
                           128, 64, 32, want_codes=True)[1]
    assert int(codes.min()) >= 0 and int(codes.max()) <= 15 and codes.unique().numel() > 4
