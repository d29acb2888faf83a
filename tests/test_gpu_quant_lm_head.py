"""`AutoRound(..., quant_lm_head=True).quantize_and_save()` end to end on the GPU: after the blocks, lm_head is tuned on the
final norm of the block chain, packed like the block linears and listed in `extra_config`.  The tuning loop itself is
compared with the oracle in tests/test_gpu_lm_head.py."""
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("CUDA device required", allow_module_level=True)

from auto_round_b200 import AutoRound, export  # noqa: E402
from test_gpu_resume import _model, _tensors, _Tok  # noqa: E402  (tests/ is on sys.path)


def test_quant_lm_head_packs_and_exports_lm_head(golden_dir, tmp_path, monkeypatch):
    rec = torch.load(os.path.join(golden_dir, "rtn_export_w4a16_sym_g32.pt"), weights_only=False)
    tokens, iters = rec["tokens"], 12
    monkeypatch.delenv("AR_RESUME_DIR", raising=False)
    model = _model(rec["init_state"])
    ar = AutoRound(model, tokenizer=_Tok(), scheme="W4A16", group_size=32, iters=iters, nsamples=8, seqlen=16, batch_size=4,
                   dataset=[tokens[:4], tokens[4:]], device_map=0, seed=42, quant_lm_head=True)
    out = str(tmp_path / "ckpt")
    ar.quantize_and_save(out, format="auto_round")

    assert [r["block"] for r in ar.block_results] == ["model.layers.0", "model.layers.1", "lm_head"]
    head = ar.block_results[-1]
    assert len(head["losses"]) == iters and head["best_loss"] <= head["init_loss"] * (1 + 1e-6)
    assert isinstance(model.lm_head, export.QuantLinear)

    got = _tensors(out)
    assert "lm_head.weight" not in got
    # lm_head [vocab 128, hidden 64] has the shape of gate_proj [intermediate 128, hidden 64]: same packed layout
    for leaf in ("qweight", "qzeros", "scales"):
        ref = got[f"model.layers.0.mlp.gate_proj.{leaf}"]
        assert got[f"lm_head.{leaf}"].dtype == ref.dtype and got[f"lm_head.{leaf}"].shape == ref.shape, leaf

    qc = json.load(open(os.path.join(out, "config.json")))["quantization_config"]
    assert qc["extra_config"] == {"lm_head": export.extra_config_entry(ar.scheme)}
    assert qc["extra_config"]["lm_head"]["bits"] == 4 and qc["extra_config"]["lm_head"]["group_size"] == 32
