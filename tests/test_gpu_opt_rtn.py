"""Optimized RTN on the GPU (SURVEY.md 8 row a18): the importance-weighted scale searches (ar_search_scale_int / _nv / _mx),
the importance-matrix accumulator, and `AutoRound(iters=0)` end to end against checkpoints written by the unmodified
reference (tests/golden/opt_rtn.pt, rtn_export_opt_*.pt).

Tolerance: the searches pick argmin over candidates with `loss < best`; the fp32 loss is a sum over the group whose order
differs between torch-CPU (fixtures), torch-CUDA and these kernels, so a group whose two best candidates tie to ~1 ulp may
resolve differently.  Expected: bit-exact; accepted: a differing group must have an oracle loss within 1e-5 relative of the
reference's choice, and at most 2 % of the groups may differ."""
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("CUDA device required", allow_module_level=True)

from auto_round_b200 import AutoRound, ops  # noqa: E402
from auto_round_b200.wrapper import importance_weights  # noqa: E402
from oracle import qdq as Q  # noqa: E402

DEV = torch.device("cuda", 0)


def _group_loss(w, qdq, imatrix, bits, g):
    grp, _, _ = Q.to_groups(w.float(), g)
    qg, _, _ = Q.to_groups(qdq.float(), g)
    qw = Q.imatrix_weights(imatrix, Q.to_groups(w, g)[0], bits, g) if imatrix is not None else 1.0
    return (((qg - grp) ** 2) * qw).sum(-1)


@pytest.mark.parametrize("case", ["int_sym_w4g128", "int_sym_w2g32", "int_sym_w3g128", "int_sym_w8g64", "int_sym_w4g128_pad",
                                  "int_sym_w4g32_imzero", "nv_fp4_g16", "nv_fp4_g16_noim", "mx_fp4_g32"])
def test_search_kernels_match_reference(golden_dir, case):
    r = torch.load(os.path.join(golden_dir, "opt_rtn.pt"), weights_only=False)[case]
    w = r["w"].to(DEV)
    im = None if r["imatrix"] is None else r["imatrix"].to(DEV)
    bits, g = r["kw"]["bits"], r["kw"]["group_size"]
    n, k = w.shape
    if r["fn"] == "opt_rtn_int_sym":
        spec = ops.make_spec("int_sym", bits, g, n, k)
        scale, wq = ops.search_scale_int(spec, w, importance_weights(im, w, bits, g))
        got_scale = scale.cpu()
    else:
        name = "nv_fp4" if "nv" in r["fn"] else "mx_fp4"
        spec = ops.make_spec(name, 4, g, n, k)
        wsrc = w if name == "nv_fp4" else w.float()
        qw = importance_weights(im, wsrc, 4, g)
        coeff = ops.search_scale_nv(spec, w, qw) if name == "nv_fp4" else ops.search_scale_mx(spec, w, qw)
        gs = None if r["global_scale"] is None else r["global_scale"].to(DEV).reshape(1).float()
        wq, sc, _ = ops.qdq_fwd(spec, w, None, None, coeff, None, None, gs, want_scale=True)
        got_scale = sc.float().cpu()
    torch.cuda.synchronize()
    ref_q, ref_s = r["qdq"], r["scale"].reshape(-1).float()
    wq = wq.cpu()
    if torch.equal(wq, ref_q) and torch.equal(got_scale.reshape(-1), ref_s):
        return
    # near-tie resolution: every differing group must be as good as the reference's choice
    bad = (got_scale.reshape(-1) != ref_s)
    assert bad.float().mean() <= 0.02, (case, int(bad.sum()), bad.numel())
    l_got = _group_loss(r["w"], wq, r["imatrix"], bits, g)
    l_ref = _group_loss(r["w"], ref_q, r["imatrix"], bits, g)
    assert torch.all((l_got - l_ref).abs()[bad] <= 1e-5 * l_ref[bad].abs() + 1e-12), case
    same = ~bad
    gq, _, _ = Q.to_groups(wq.float(), g)
    gr, _, _ = Q.to_groups(ref_q.float(), g)
    assert torch.equal(gq[same], gr[same]), case


def test_search_int_without_wq_and_bad_args():
    w = (torch.randn(8, 256, device=DEV) * 0.05).bfloat16()
    spec = ops.make_spec("int_sym", 4, 128, 8, 256)
    s1, wq = ops.search_scale_int(spec, w, None)
    s2, none = ops.search_scale_int(spec, w, None, want_wq=False)
    assert none is None and torch.equal(s1, s2)
    # the search must never be worse than plain RTN's scale on its own objective
    plain, _, _ = ops.qdq_fwd(ops.make_spec("int_sym", 4, 128, 8, 256), w, want_scale=False)
    e_opt = ((wq.float() - w.float()) ** 2).reshape(-1, 128).sum(-1)
    e_rtn = ((plain.float() - w.float()) ** 2).reshape(-1, 128).sum(-1)
    assert e_opt.sum() <= e_rtn.sum() * 1.02
    with pytest.raises(ValueError):
        ops.search_scale_int(spec, w, torch.ones(255, device=DEV))
    with pytest.raises(RuntimeError):
        ops.search_scale_mx(ops.make_spec("mx_fp4", 4, 64, 8, 256), w, None)      # MX groups are 32 wide


@pytest.mark.parametrize("rows,k", [(1, 64), (37, 200), (4096, 4096), (5, 14336)])
def test_imatrix_accum(rows, k):
    torch.manual_seed(rows + k)
    x = (torch.randn(rows, k, device=DEV) * 0.7).bfloat16()
    im = torch.full((k,), 0.25, dtype=torch.float32, device=DEV)
    ops.imatrix_accum(x, im)
    ref = 0.25 + x.float().pow(2).sum(0)
    assert torch.allclose(im, ref, rtol=2e-5, atol=1e-6)
    ops.imatrix_accum(x, im)                                   # accumulates
    assert torch.allclose(im, 0.25 + 2 * x.float().pow(2).sum(0), rtol=2e-5, atol=1e-6)


class _Tok:
    pad_token_id = None
    pad_token = None

    def save_pretrained(self, *a, **k):
        return None


KW = {"opt_w4a16_sym_g32": dict(scheme="W4A16", group_size=32), "opt_nvfp4": dict(scheme="NVFP4", act_bits=16, act_data_type="float"),
      "opt_mxfp4": dict(scheme="MXFP4", act_bits=16)}


def _tiny_llama(state):
    from transformers import LlamaConfig, LlamaForCausalLM

    cfg = LlamaConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=2, vocab_size=128, max_position_embeddings=64, rms_norm_eps=1e-5,
                      rope_theta=10000.0, tie_word_embeddings=False)
    model = LlamaForCausalLM(cfg).to(torch.bfloat16).eval()
    model.load_state_dict(state)
    return model


@pytest.mark.parametrize("tag", list(KW))
def test_opt_rtn_layers_bit_exact_given_reference_imatrix(golden_dir, tag):
    """Layer by layer, with the importance matrix the REFERENCE collected (recorded in the fixture; None for MXFP4):
    search -> qdq -> pack must reproduce every packed tensor of the reference's checkpoint bit for bit."""
    from auto_round_b200 import export
    from auto_round_b200.quantizer import SignRoundQuantizer
    from auto_round_b200.schemes import parse_scheme

    rec = torch.load(os.path.join(golden_dir, f"rtn_export_{tag}.pt"), weights_only=False)
    model = _tiny_llama(rec["init_state"])
    kw = dict(KW[tag])
    scheme = parse_scheme(kw.pop("scheme"), kw)
    quantizer = SignRoundQuantizer(scheme, iters=0, batch_size=4)
    for li, block in enumerate(model.model.layers):
        block.to(DEV)
        names = [n for n, m in block.named_modules() if quantizer.layer_filter(n, m)]
        assert len(names) == 7
        nv_gs = AutoRound._fuse_nv_global_scales(block, names) if scheme.qdq_name == "nv_fp4" else None
        imx = {n: (rec["imatrix"][f"model.layers.{li}.{n}"].to(DEV) if rec["imatrix"] else None) for n in names}
        done = quantizer.rtn_block(block, None, nv_gs, imatrices=imx)
        for n in done:
            ql = export.pack_linear(block.get_submodule(n), scheme, DEV)
            for key, ref in rec["tensors"].items():
                base, leaf = key.rsplit(".", 1)
                if base != f"model.layers.{li}.{n}":
                    continue
                got = getattr(ql, leaf)
                got = got.view(torch.uint8) if got.dtype == torch.float8_e4m3fn else got
                assert got.dtype == ref.dtype and tuple(got.shape) == tuple(ref.shape), key
                assert torch.equal(got.cpu(), ref), key
        block.to("cpu")


@pytest.mark.parametrize("tag", list(KW))
def test_default_rtn_checkpoint_matches_reference(golden_dir, tag, tmp_path):
    """`AutoRound(iters=0)` end to end with the reference's default routing (calibrated imatrix search for int sym and
    NVFP4, zero-shot search for MXFP4): tensor names, dtypes, shapes and quantization_config exactly.  Values: MXFP4 (no
    calibration) bit-exact.  For the calibrated routes the importance matrix comes from OUR bf16 block forward on the GPU,
    the fixture's from the reference's CPU forward; activations differ in the last bf16 bit, the imatrix by ~1e-3, and the
    argmin over 200 near-flat candidates then moves for a few percent of the groups (the reference's own CPU and CUDA runs
    differ the same way).  `reference_mask_cast=True` reproduces the reference's bf16 cast of the boolean attention mask
    (autoround.py:199-203).  Checked: imatrix within 5 % of the recorded one, and < 2 % of any tensor's bytes differ (measured 0.2 %); the
    bit-exact statement is test_opt_rtn_layers_bit_exact_given_reference_imatrix above."""
    from safetensors import safe_open

    rec = torch.load(os.path.join(golden_dir, f"rtn_export_{tag}.pt"), weights_only=False)
    model = _tiny_llama(rec["init_state"])
    tokens = rec["tokens"]
    ar = AutoRound(model, tokenizer=_Tok(), iters=0, nsamples=8, seqlen=16, batch_size=4, dataset=[tokens[:4], tokens[4:]],
                   device_map=0, seed=42, reference_mask_cast=True, **KW[tag])
    ar.keep_imatrix = True
    assert ar._rtn_mode() == ("zero_shot_opt" if tag == "opt_mxfp4" else "calibrated_opt")
    out = str(tmp_path / "ckpt")
    ar.quantize_and_save(out, format="auto_round")
    got = {}
    with safe_open(os.path.join(out, "model.safetensors"), "pt") as f:
        for k in f.keys():
            t = f.get_tensor(k)
            got[k] = t.view(torch.uint8) if t.dtype == torch.float8_e4m3fn else t
    worst = 0.0
    for k, ref in rec["tensors"].items():
        assert k in got, k
        assert got[k].dtype == ref.dtype and tuple(got[k].shape) == tuple(ref.shape), k
        a, b = got[k].contiguous().view(torch.uint8).reshape(-1), ref.contiguous().view(torch.uint8).reshape(-1)
        frac = (a != b).float().mean().item()
        worst = max(worst, frac)
        assert frac <= (0.0 if tag == "opt_mxfp4" else 0.02), (k, frac)
    print(f"{tag}: worst mismatching byte fraction {worst:.5f}")
    extra = {k for k in got if ".layers." in k and "layernorm" not in k} - set(rec["tensors"])
    assert not extra, extra
    qc = json.load(open(os.path.join(out, "config.json")))["quantization_config"]
    assert qc == rec["quantization_config"]
    if tag != "opt_mxfp4":
        seen = 0
        for res in ar.block_results:
            for n, t in res["imatrix"].items():
                ref = rec["imatrix"][f"{res['block']}.{n}"]
                assert torch.allclose(t, ref, rtol=5e-2, atol=1e-6), (res["block"], n, (t - ref).abs().max().item())
                seen += 1
        assert seen == 14


def test_rtn_routing_mirrors_reference():
    from transformers import LlamaConfig, LlamaForCausalLM

    cfg = LlamaConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=1, num_attention_heads=4,
                      num_key_value_heads=2, vocab_size=128, max_position_embeddings=64)
    model = LlamaForCausalLM(cfg).to(torch.bfloat16).eval()

    def mode(**kw):
        return AutoRound(model, tokenizer=_Tok(), iters=0, device_map=0, **kw)._rtn_mode()

    assert mode(scheme="W4A16") == "calibrated_opt"
    assert mode(scheme="W4A16", disable_opt_rtn=True) == "plain"
    assert mode(scheme="W2A16", sym=False) == "plain"
    assert mode(scheme="W8A16") == "plain"
    assert mode(scheme="W8A16", disable_opt_rtn=False) == "calibrated_opt"
    assert mode(scheme="MXFP4", act_bits=16) == "zero_shot_opt"
    assert mode(scheme="NVFP4", act_bits=16, act_data_type="float") == "calibrated_opt"
