"""Format resolution and the `auto_awq` / `auto_gptq` configs (host logic, CPU).  The expected layouts and
`quantization_config` dictionaries are the ones the unmodified reference wrote for tests/golden/rtn_export_fmt_*.pt
(oracle/gen_golden_formats.py); the oracle reproduces every packed tensor of those checkpoints from the initial weights."""
import logging
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

from auto_round_b200 import export
from auto_round_b200.export import ResolvedFormat, resolve_format
from auto_round_b200.schemes import parse_scheme
from oracle import pack as P
from oracle import pack_awq as A
from oracle import qdq as Q

W4S = parse_scheme("W4A16", {"group_size": 32})
W4A = parse_scheme("W4A16", {"group_size": 32, "sym": False})
W2A = parse_scheme("W2A16", {"group_size": 32, "sym": False})
NVFP4 = parse_scheme("NVFP4", {"act_bits": 16, "act_data_type": "float"})
MXFP4 = parse_scheme("MXFP4", {"act_bits": 16})
FIXTURES = ["w4a16_asym_g32__auto_round", "w4a16_asym_g32__auto_awq", "w4a16_sym_g32__auto_awq", "w4a16_sym_g32__auto_gptq",
            "w2a16_asym_g32__auto_gptq", "w4a16_asym_g32_mixed8__auto_round"]


def _load(golden_dir, tag):
    return torch.load(os.path.join(golden_dir, f"rtn_export_fmt_{tag}.pt"), weights_only=False)


# ------------------------------------------------------------------------------------------------ the resolver table
@pytest.mark.parametrize("fmt,scheme,layer_config,want", [
    ("auto_round", W4S, None, ResolvedFormat("auto_round", "auto", "auto_round:auto_gptq")),
    (None, W4S, None, ResolvedFormat("auto_round", "auto", "auto_round:auto_gptq")),
    ("auto_round:auto_gptq", W4S, None, ResolvedFormat("auto_round", "auto", "auto_round:auto_gptq")),
    ("auto_round:gptqmodel", W4S, None, ResolvedFormat("auto_round", "auto", "auto_round:auto_gptq")),
    ("auto_round", W4A, None, ResolvedFormat("auto_round", "awq", "auto_round:auto_awq")),
    ("auto_round", W4A, {"lm_head": {"bits": 16}}, ResolvedFormat("auto_round", "awq", "auto_round:auto_awq")),
    ("auto_round", W4A, {"model.layers.1.mlp.down_proj": {"bits": 8}}, ResolvedFormat("auto_round", "auto", "auto_round")),
    ("auto_round", W2A, None, ResolvedFormat("auto_round", "auto", "auto_round")),
    ("auto_round", NVFP4, None, ResolvedFormat("auto_round", "auto", "auto_round:llm_compressor")),
    ("auto_round", MXFP4, None, ResolvedFormat("auto_round", "auto", "auto_round:llm_compressor")),
    ("auto_gptq", W4S, None, ResolvedFormat("auto_gptq", "gptq", None)),
    ("gptqmodel", W4S, None, ResolvedFormat("auto_gptq", "gptq", None)),
    ("auto_gptq", W2A, None, ResolvedFormat("auto_gptq", "gptq", None)),
    ("auto_awq", W4S, None, ResolvedFormat("auto_awq", "awq", None)),
    ("auto_awq", W4A, None, ResolvedFormat("auto_awq", "awq", None)),
    ("auto_round:auto_awq", W4S, None, ResolvedFormat("auto_round", "awq", "auto_round:auto_awq")),
])
def test_resolver_table(fmt, scheme, layer_config, want):
    assert resolve_format(fmt, scheme, layer_config) == want


def test_only_the_new_layouts_enter_the_resume_signature():
    assert not resolve_format("auto_round", W4S).is_new_layout
    assert not resolve_format("auto_round", W2A).is_new_layout
    assert not resolve_format("auto_round", NVFP4).is_new_layout
    assert resolve_format("auto_round", W4A).is_new_layout
    assert resolve_format("auto_gptq", W4S).is_new_layout and resolve_format("auto_awq", W4S).is_new_layout


def test_rejections():
    with pytest.raises(ValueError, match="gguf:q4_k_m is not supported"):
        resolve_format("gguf:q4_k_m", W4S)
    with pytest.raises(ValueError, match=r"auto_awq format support quantization scheme with W4A16 but got bits=2"):
        resolve_format("auto_awq", W2A)
    with pytest.raises(ValueError, match=r"auto_awq format support .* data_type=nv_fp"):
        resolve_format("auto_awq", NVFP4)
    with pytest.raises(ValueError, match=r"auto_gptq format support .* data_type=mx_fp"):
        resolve_format("auto_gptq", MXFP4)
    with pytest.raises(ValueError, match="bits=8 for layer"):
        resolve_format("auto_awq", W4S, {"model.layers.0.mlp.down_proj": {"bits": 8}})
    odd_n, odd_k = nn.Linear(64, 12), nn.Linear(48, 64)
    with pytest.raises(ValueError, match=r"out_features \(12\) shape mismatch"):
        resolve_format("auto_awq", W4S, None, [("a.b", odd_n, W4S)])
    with pytest.raises(ValueError, match=r"in_features \(48\) shape mismatch"):
        resolve_format("auto_round", W4A, None, [("a.b", odd_k, W4A)])
    # the same shapes are no obstacle for the layouts that pack along K in 32-bit words
    assert resolve_format("auto_round", W4S, None, [("a.b", odd_n, W4S)]).layout == "auto"


def test_gptq_asym_warns_like_the_reference(caplog):
    with caplog.at_level(logging.WARNING, logger=export.logger.name):
        resolve_format("auto_gptq", W2A)
    assert "asymmetrical kernel of the GPTQ format" in caplog.text
    caplog.clear()
    with caplog.at_level(logging.WARNING, logger=export.logger.name):
        resolve_format("auto_gptq", W4S)
    assert caplog.text == ""


class _Untouchable(nn.Module):
    """A model whose forward raises: a rejected format must never get as far as running it."""

    def __init__(self):
        super().__init__()
        blk = nn.Module()
        blk.proj = nn.Linear(64, 12)
        self.layers = nn.ModuleList([blk])
        self.calls = 0

    def forward(self, *a, **k):
        self.calls += 1
        raise AssertionError("the model was run")


@pytest.mark.parametrize("fmt,kw,err", [
    ("gguf:q4_0", dict(scheme="W4A16"), "is not supported"),
    ("auto_awq", dict(scheme="W2A16"), "bits=2"),
    ("auto_awq", dict(scheme="MXFP4", act_bits=16), "data_type=mx_fp"),
    ("auto_gptq", dict(scheme="NVFP4", act_bits=16, act_data_type="float"), "data_type=nv_fp"),
    ("auto_awq", dict(scheme="W4A16", group_size=32), r"out_features \(12\) shape mismatch"),
    ("auto_round", dict(scheme="W4A16", group_size=32, sym=False), r"out_features \(12\) shape mismatch"),
])
def test_quantize_and_save_rejects_before_touching_the_model(fmt, kw, err, tmp_path, monkeypatch):
    from auto_round_b200 import AutoRound
    from auto_round_b200 import autoround as ar_mod

    monkeypatch.setattr(ar_mod.AutoRound, "_resolve_device", staticmethod(lambda device_map: torch.device("cuda", 0)))
    model = _Untouchable()
    before = {k: v.clone() for k, v in model.state_dict().items()}
    ar = AutoRound(model, tokenizer=object(), iters=2, nsamples=2, seqlen=8, dataset=[torch.zeros(2, 8, dtype=torch.long)], **kw)
    with pytest.raises(ValueError, match=err):
        ar.quantize_and_save(str(tmp_path / "out"), format=fmt)
    with pytest.raises(ValueError, match=err):
        ar.save_quantized(str(tmp_path / "out"), format=fmt)
    assert model.calls == 0 and not os.path.exists(tmp_path / "out")
    assert all(torch.equal(v, before[k]) for k, v in model.state_dict().items())
    assert type(model.layers[0].proj) is nn.Linear


# -------------------------------------------------------------------------------- configs the reference wrote
def test_configs_equal_the_recorded_ones(golden_dir):
    """Built from the recorded scheme alone (iters=0), each writer's config equals what the reference serialised."""
    for tag in FIXTURES:
        rec = _load(golden_dir, tag)
        kw = dict(rec["scheme_kwargs"])
        sc = parse_scheme(kw.pop("scheme"), kw)
        fmt = resolve_format(rec["format"], sc, rec["layer_config"])
        if fmt.writer == "auto_round":
            got = export.build_quantization_config(sc, "model.layers", rec["layer_config"], 0, packing_format=fmt.packing_format)
        elif fmt.writer == "auto_awq":
            got = export.build_awq_config(sc, "model.layers", ["lm_head"], 0)
        else:
            got = export.build_gptq_config(sc, None, False, None, 0)
        assert got == rec["quantization_config"], tag


def test_gptq_dynamic_rules():
    eight = parse_scheme("W8A16", {"group_size": 32})
    sixteen = parse_scheme("W4A16", {"bits": 16})
    cfg = export.build_gptq_config(W4S, {"model.layers.1.mlp.down_proj": eight, "model.layers.0.mlp.up_proj": sixteen}, True,
                                   [["mlp.down_proj", "self_attn.q_proj"]], 2, {})
    assert cfg["dynamic"] == {r"+:.*model\.layers\.1\.mlp\.down_proj.*": {"bits": 8, "group_size": 32, "sym": True},
                              r"-:.*model\.layers\.0\.mlp\.up_proj.*": {}}
    assert cfg["lm_head"] is True and cfg["iters"] == 2
    assert cfg["modules_in_block_to_quantize"] == [["mlp.down_proj", "self_attn.q_proj"]]


# ------------------------------------------------------------- the recorded checkpoints, rebuilt by the oracle
def _oracle_layer(rec, name, layout, sc):
    w = rec["init_state"][name + ".weight"]
    n = w.shape[0]
    if sc.sym:
        wq, s, zp = Q.rtn_int_sym(w.clone(), sc.bits, sc.group_size)
    else:
        wq, s, zp = Q.int_asym(w, sc.bits, sc.group_size)
        zp = zp.reshape(n, -1)
    s = s.reshape(n, -1)
    if layout == "awq":
        return A.pack_awq(wq, s, zp if not sc.sym else int(zp), sc.group_size), zp
    return P.pack_int(wq, s, zp, sc.bits, sc.group_size, layout == "gptq"), zp


@pytest.mark.parametrize("tag", FIXTURES)
def test_oracle_reproduces_reference_checkpoint(golden_dir, tag):
    rec = _load(golden_dir, tag)
    kw = dict(rec["scheme_kwargs"])
    base = parse_scheme(kw.pop("scheme"), kw)
    fmt = resolve_format(rec["format"], base, rec["layer_config"])
    tensors = rec["tensors"]
    layers = sorted({k.rsplit(".", 1)[0] for k in tensors})
    assert len(layers) == 14
    zero_groups = 0
    for name in layers:
        sc = parse_scheme(base, (rec["layer_config"] or {}).get(name))
        layout = fmt.layout if fmt.layout != "auto" else ("gptq" if sc.sym else "plain")
        out, zp = _oracle_layer(rec, name, layout, sc)
        keys = sorted(k.rsplit(".", 1)[1] for k in tensors if k.rsplit(".", 1)[0] == name)
        # g_idx: absent from auto_round checkpoints, present in auto_gptq ones
        assert keys == (["g_idx", "qweight", "qzeros", "scales"] if fmt.writer == "auto_gptq" else ["qweight", "qzeros", "scales"])
        for key in keys:
            assert np.array_equal(np.asarray(out[key]), tensors[f"{name}.{key}"].numpy()), (tag, name, key)
        if isinstance(zp, torch.Tensor):
            zero_groups += int((zp == 0).sum())
    if not base.sym:
        # zero-point 0 under the zp-1 layout is the field value -1: the shifted lanes are summed, so it borrows from the
        # fields above it exactly as the reference's sum does
        assert zero_groups > 0, "the fixture must contain groups with zero-point 0"


def test_awq_entry_points_validate_arguments_without_a_gpu():
    from auto_round_b200 import _lib

    lib = _lib.load()
    assert lib.ar_pack_awq(None, None, None, 0, 64, 64, 32, None, None, None, None) == -1
    assert lib.ar_unpack_awq(None, None, None, 64, 64, 32, None, None, None) == -1
    assert b"null pointer" in lib.ar_last_error()
