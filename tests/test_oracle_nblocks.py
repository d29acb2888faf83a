"""nblocks > 1 (consecutive decoder blocks tuned as one group) without a GPU: the CPU oracle against fixtures of the
unmodified reference's group path (tools/gen_golden_nblocks.py -> tests/golden/block_nblocks2_*.pt, a 3-layer tiny Llama
tuned as the groups [0, 1] and [2]), and the host logic of AutoRound's group loop."""
import logging
import os

import pytest
import torch
import torch.nn as nn

from auto_round_b200.autoround import AutoRound, BlockGroup, block_groups
from oracle import signround as S

SCHEMES = {
    "w4a16_sym_g32": S.LayerScheme(4, 32, True, "int"),
    "w2a16_asym_g32": S.LayerScheme(2, 32, False, "int"),
}


def _load(golden_dir, tag):
    return torch.load(os.path.join(golden_dir, f"block_nblocks2_{tag}.pt"), weights_only=False)


def _llama_cfg():
    from transformers import LlamaConfig

    cfg = LlamaConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=3, num_attention_heads=4,
                      num_key_value_heads=2, vocab_size=128, max_position_embeddings=64, rms_norm_eps=1e-5,
                      rope_theta=10000.0, tie_word_embeddings=False)
    cfg._attn_implementation = "sdpa"
    return cfg


def tiny_group(state, first: int = 0) -> BlockGroup:
    """The BlockGroup of a fixture record: its state dict holds `layers.<j>.…` for every member."""
    from transformers.models.llama.modeling_llama import LlamaDecoderLayer

    n = 1 + max(int(k.split(".")[1]) for k in state)
    cfg = _llama_cfg()
    members = [LlamaDecoderLayer(cfg, first + j).to(torch.bfloat16).eval() for j in range(n)]
    g = BlockGroup(members, [f"model.layers.{first + j}" for j in range(n)])
    g.load_state_dict(state)
    return g


@pytest.mark.parametrize("tag", list(SCHEMES))
def test_tune_group_matches_reference_bit_exact(golden_dir, tag):
    """Both groups ([0, 1] and the short [2]): every iteration's loss, the best iteration, and each layer's final qdq
    weight, scale and zero-point of the reference's WrapperMultiblock run, reproduced by the oracle tuning a BlockGroup."""
    rec = _load(golden_dir, tag)
    assert rec["nblocks"] == 2 and len(rec["blocks"]) == 2
    sc = SCHEMES[tag]
    for gi, (b, size) in enumerate(zip(rec["blocks"], (2, 1))):
        grp = tiny_group(b["block_state"], first=2 * gi)
        assert len(grp.layers) == size and len(b["layers"]) == 7 * size
        masks = [(ids != -100).to(torch.long) for ids in b["input_ids"]]
        res = S.tune_block(grp, b["inputs"], b["others"], b["fp_outputs"], lambda n, m: sc, iters=rec["iters"],
                           batch_size=rec["batch_size"], token_masks=masks, sampler=S.ReplaySampler(b["batches"]))
        nvalid = [sum(int(masks[i].sum()) for i in batch) for batch in b["batches"]]
        got = [l * n for l, n in zip(res.losses, nvalid)]
        assert got == pytest.approx(b["losses"], rel=1e-6), (tag, gi)
        assert res.best_iter == b["best_iter"], (tag, gi)
        for name, lay in b["layers"].items():
            mod = grp.get_submodule(name)
            assert torch.equal(mod.weight.data, lay["weight"]), (tag, gi, name)
            assert torch.equal(mod.scale.float().reshape(-1), lay["scale"].float().reshape(-1)), (tag, gi, name)
            if isinstance(lay["zp"], torch.Tensor):
                assert torch.equal(mod.zp.reshape(-1), lay["zp"].reshape(-1)), (tag, gi, name)


def test_group_forward_chains_members(golden_dir):
    """The group's output on the fixture inputs is the reference's FP output of the whole group (first group, untuned)."""
    b = _load(golden_dir, "w4a16_sym_g32")["blocks"][0]
    grp = tiny_group(b["block_state"])
    masks = [(ids != -100).to(torch.long) for ids in b["input_ids"]]
    with torch.no_grad():
        for i in range(len(b["inputs"])):
            x, sel = S.select_batch(b["inputs"], b["others"], [i])
            assert torch.equal(S.block_forward(grp, x, sel), b["fp_outputs"][i]), i
    assert len(masks) == len(b["fp_outputs"])


@pytest.mark.parametrize("nblk", [1, 3, 4])
@pytest.mark.parametrize("nblocks", [1, 2, 3, 5])
def test_block_groups_partition(nblk, nblocks):
    want = {
        (1, 1): [[0]], (1, 2): [[0]], (1, 3): [[0]], (1, 5): [[0]],
        (3, 1): [[0], [1], [2]], (3, 2): [[0, 1], [2]], (3, 3): [[0, 1, 2]], (3, 5): [[0, 1, 2]],
        (4, 1): [[0], [1], [2], [3]], (4, 2): [[0, 1], [2, 3]], (4, 3): [[0, 1, 2], [3]], (4, 5): [[0, 1, 2, 3]],
    }[(nblk, nblocks)]
    assert block_groups(nblk, nblocks) == want


def test_layer_config_full_names_reach_the_layer_inside_a_group():
    from auto_round_b200.quantizer import SignRoundQuantizer
    from auto_round_b200.schemes import parse_scheme

    q = SignRoundQuantizer(parse_scheme("W4A16"), iters=1,
                           layer_config={"model.layers.2.mlp.down_proj": {"bits": 8}, "self_attn.o_proj": {"group_size": 32},
                                         "model.layers.1.mlp.up_proj": {"bits": 16}})
    lin = nn.Linear(8, 8)
    grp = BlockGroup([nn.Module(), nn.Module()], ["model.layers.1", "model.layers.2"])
    q.block_prefix = grp.prefix_map()
    assert q.layer_names("layers.1.mlp.down_proj") == ("model.layers.2.mlp.down_proj", "mlp.down_proj")
    assert q.scheme_for("layers.1.mlp.down_proj", lin).bits == 8
    assert q.scheme_for("layers.0.mlp.down_proj", lin).bits == 4
    assert q.scheme_for("layers.0.mlp.up_proj", lin).bits == 16
    assert q.scheme_for("layers.1.mlp.up_proj", lin).bits == 4
    for j in (0, 1):                                                   # a bare block-relative key: every member
        assert q.scheme_for(f"layers.{j}.self_attn.o_proj", lin).group_size == 32
    q.block_prefix = "model.layers.2"                                  # one block at a time: unchanged
    assert q.layer_names("mlp.down_proj") == ("model.layers.2.mlp.down_proj", "mlp.down_proj")
    assert q.scheme_for("mlp.down_proj", lin).bits == 8


class _Tok:
    pad_token_id = None
    pad_token = None


class _Untouchable(nn.Module):
    def __init__(self):
        super().__init__()
        self.lin = nn.Linear(4, 4)

    def forward(self, *a, **k):
        raise AssertionError("the model must not run")

    def eval(self):
        raise AssertionError("the model must not be touched")


@pytest.mark.parametrize("bad", [0, -1, 1.5, 2.0, "2", True, [2]])
def test_invalid_nblocks_raises_before_model_work(bad):
    with pytest.raises(ValueError, match="nblocks"):
        AutoRound(_Untouchable(), tokenizer=_Tok(), nblocks=bad, device_map=0)


def _tiny_model():
    from transformers import LlamaForCausalLM

    torch.manual_seed(0)
    return LlamaForCausalLM(_llama_cfg()).to(torch.bfloat16).eval()


def test_resume_dir_with_nblocks_warns_and_skips_nothing(tmp_path, monkeypatch, caplog):
    """AR_RESUME_DIR with nblocks=2: a warning, tuning from block 0, and the resume directory is neither read nor written.
    The same directory still resumes an nblocks=1 run."""
    from auto_round_b200.autoround import find_blocks

    monkeypatch.setenv("AR_RESUME_DIR", str(tmp_path))
    model = _tiny_model()
    prefix, blocks = find_blocks(model)
    one = AutoRound(model, tokenizer=_Tok(), iters=4, nsamples=2, seqlen=8, batch_size=2, device_map=0)
    st, start = one._open_resume(prefix, blocks)
    assert start == 0
    st.mark_block_done(f"{prefix}.0", {}, None, [torch.zeros(1, 8, 64)])
    before = sorted((p.name, p.stat().st_mtime_ns) for p in tmp_path.rglob("*"))

    two = AutoRound(model, tokenizer=_Tok(), iters=4, nsamples=2, seqlen=8, batch_size=2, device_map=0, nblocks=2)
    with caplog.at_level(logging.WARNING, logger="auto_round_b200.autoround"):
        assert two._open_resume(prefix, blocks) == (None, 0)
    assert any("nblocks" in r.getMessage() and "AR_RESUME_DIR" in r.getMessage() for r in caplog.records)
    assert sorted((p.name, p.stat().st_mtime_ns) for p in tmp_path.rglob("*")) == before
    assert one._open_resume(prefix, blocks)[1] == 1


def test_fused_block_ops_patch_the_rotary_helper_of_a_group():
    """The group module is defined outside the model file, so the rotary helper is found through its members."""
    from transformers.models.llama import modeling_llama
    from transformers.models.llama.modeling_llama import LlamaDecoderLayer

    from auto_round_b200.fused import fused_block_ops

    cfg = _llama_cfg()
    grp = BlockGroup([LlamaDecoderLayer(cfg, j) for j in range(2)], ["model.layers.0", "model.layers.1"])
    orig = modeling_llama.apply_rotary_pos_emb
    with fused_block_ops(grp):
        assert getattr(modeling_llama.apply_rotary_pos_emb, "_ar_fused", False)
    assert modeling_llama.apply_rotary_pos_emb is orig
