"""nblocks > 1 on the GPU: consecutive decoder blocks tuned as one BlockGroup by the captured SignRound iteration.

Against the CPU oracle (pinned bit-exact to the reference's group path by tests/test_oracle_nblocks.py) with the bars of
tests/test_gpu_engine.py: iteration-0 loss within 2e-2, best loss <= iteration-0 loss, final group-output MSE within
+-25 % of the oracle's, the reference's scale / zp shapes.  Then the public API end to end, grouped MoE experts, the loop
options, and data parallelism (2 ranks must reproduce 1 rank, the bars of tests/test_gpu_dp.py)."""
import json
import os
import random
import socket

import pytest
import torch
import torch.multiprocessing as mp
import torch.nn as nn

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("CUDA device required", allow_module_level=True)

from auto_round_b200 import AutoRound, ops  # noqa: E402
from auto_round_b200.autoround import BlockGroup  # noqa: E402
from auto_round_b200.export import QuantLinear  # noqa: E402
from auto_round_b200.quantizer import DataParallel, SignRoundQuantizer  # noqa: E402
from auto_round_b200.schemes import parse_scheme  # noqa: E402
from oracle import signround as S  # noqa: E402
from oracle.tests_support import tiny_block  # noqa: E402

DEV = torch.device("cuda", 0)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

SCHEMES = {
    "w4a16_sym_g32": (dict(scheme="W4A16", group_size=32), S.LayerScheme(4, 32, True, "int")),
    "w2a16_asym_g32": (dict(scheme="W2A16", group_size=32, sym=False), S.LayerScheme(2, 32, False, "int")),
}


class _Tok:
    pad_token_id = None
    pad_token = None

    def save_pretrained(self, *a, **k):
        return None


def _load(tag):
    return torch.load(os.path.join(GOLDEN, f"block_nblocks2_{tag}.pt"), weights_only=False)


def _scheme(kw):
    return parse_scheme(kw["scheme"], {k: v for k, v in kw.items() if k != "scheme"})


def _member(state, j):
    p = f"layers.{j}."
    return tiny_block({k[len(p):]: v for k, v in state.items() if k.startswith(p)})


def _group(state, device="cpu"):
    n = 1 + max(int(k.split(".")[1]) for k in state)
    g = BlockGroup([_member(state, j) for j in range(n)], [f"model.layers.{j}" for j in range(n)]).to(device)
    for p in g.parameters():
        p.requires_grad_(False)
    return g


def _dev(o):
    if isinstance(o, torch.Tensor):
        return o.to(DEV)
    return type(o)(_dev(x) for x in o) if isinstance(o, (list, tuple)) else o


def _mse(block, inputs, others, fp_outputs, masks, device):
    from test_gpu_engine import _block_mse
    return _block_mse(block, inputs, others, fp_outputs, masks, device)


def _tune(block, b, scheme, iters, batches, **kw):
    q = SignRoundQuantizer(scheme, iters=iters, batch_size=len(batches[0]) // kw.get("gradient_accumulate_steps", 1),
                           **{k: v for k, v in kw.items() if k != "keep_arena"})
    q.quantize_block(block, [t.to(DEV) for t in b["inputs"]], b["others"], [t.to(DEV) for t in b["fp_outputs"]], None, None,
                     input_ids=b["input_ids"], sampler=S.ReplaySampler(batches), keep_arena=kw.get("keep_arena", False))
    return q


def _launches_per_iteration(make, b, scheme, batches):
    """ops.LAUNCHES per replayed iteration: the difference of two runs of different length (captured graph in both)."""
    counts = []
    for iters in (6, 10):
        before = ops.LAUNCHES[0]
        q = _tune(make(), b, scheme, iters, batches[:iters])
        assert q.last_result.used_cuda_graph
        counts.append(ops.LAUNCHES[0] - before)
    return (counts[1] - counts[0]) / 4


@pytest.mark.parametrize("tag", list(SCHEMES))
def test_group_vs_oracle(tag):
    rec = _load(tag)
    kw, osc = SCHEMES[tag]
    b = rec["blocks"][0]                                              # the group [0, 1]
    masks = [(ids != -100).to(torch.long) for ids in b["input_ids"]]
    iters = 40
    random.seed(1234)
    ogrp = _group(b["block_state"])
    ores = S.tune_block(ogrp, b["inputs"], b["others"], b["fp_outputs"], lambda n, m: osc, iters=iters,
                        batch_size=rec["batch_size"], token_masks=masks)
    o_mse = _mse(ogrp, b["inputs"], b["others"], b["fp_outputs"], masks, "cpu")

    grp = _group(b["block_state"], DEV)
    q = _tune(grp, b, _scheme(kw), iters, ores.batches)
    res = q.last_result
    assert res.used_cuda_graph, "the whole group's iteration must be one captured graph"
    assert len(res.losses) == iters and res.batches == ores.batches
    assert sorted(res.quantized_layers) == sorted(b["layers"])
    assert res.losses[0] == pytest.approx(ores.losses[0], rel=2e-2)
    assert res.best_loss <= res.losses[0] + 1e-12
    g_mse = _mse(grp, b["inputs"], b["others"], b["fp_outputs"], masks, DEV)
    assert g_mse == pytest.approx(o_mse, rel=0.25), (g_mse, o_mse)
    for name, lay in b["layers"].items():
        mod = grp.get_submodule(name)
        assert type(mod) is nn.Linear and tuple(mod.scale.shape) == tuple(lay["scale"].shape), name
        if isinstance(lay["zp"], torch.Tensor):
            assert tuple(mod.zp.shape) == tuple(lay["zp"].shape), name
        else:
            assert mod.zp == lay["zp"], name

    # kernel launches per iteration: the group against its two members tuned alone on the same batches
    st, sc = b["block_state"], _scheme(kw)
    n_group = _launches_per_iteration(lambda: _group(st, DEV), b, sc, ores.batches)
    n_alone = [_launches_per_iteration(lambda j=j: _member(st, j).to(DEV).requires_grad_(False), b, sc, ores.batches)
               for j in (0, 1)]
    print(f"\n[{tag}] launches per iteration: group {n_group:g}, blocks alone {n_alone[0]:g} + {n_alone[1]:g} = "
          f"{sum(n_alone):g}, difference {n_group - sum(n_alone):+g}")


def test_gradient_accumulation_group_vs_oracle():
    """gradient_accumulate_steps=2 across a group: micro-batches of 2, one sign-SGD step per iteration for all 14 layers."""
    rec = _load("w4a16_sym_g32")
    b = rec["blocks"][0]
    osc = S.LayerScheme(4, 32, True, "int")
    masks = [(ids != -100).to(torch.long) for ids in b["input_ids"]]
    iters = 30
    random.seed(77)
    ogrp = _group(b["block_state"])
    ores = S.tune_block(ogrp, b["inputs"], b["others"], b["fp_outputs"], lambda n, m: osc, iters=iters, batch_size=2,
                        token_masks=masks, gradient_accumulate_steps=2)
    o_mse = _mse(ogrp, b["inputs"], b["others"], b["fp_outputs"], masks, "cpu")
    grp = _group(b["block_state"], DEV)
    q = _tune(grp, b, parse_scheme("W4A16", {"group_size": 32}), iters, ores.batches, gradient_accumulate_steps=2)
    res = q.last_result
    assert res.used_cuda_graph and len(res.quantized_layers) == 14
    assert res.losses[0] == pytest.approx(ores.losses[0], rel=2e-2)
    assert res.best_loss <= res.losses[0] + 1e-12
    g_mse = _mse(grp, b["inputs"], b["others"], b["fp_outputs"], masks, DEV)
    assert g_mse == pytest.approx(o_mse, rel=0.25), (g_mse, o_mse)


def test_mixtral_group_tunes_the_experts_of_both_members():
    """Two tiny 4-expert Mixtral blocks as one group on the grouped expert path: captured, all 32 layers tuned, and every
    expert projection of both members moved off V = 0 (each expert receives tokens in these batches)."""
    from test_gpu_moe import _mixtral_block

    rec = torch.load(os.path.join(GOLDEN, "block_mixtral_mxfp4.pt"), weights_only=False)
    members = [_mixtral_block(blk["block_state"], True, DEV) for blk in rec["blocks"]]
    grp = BlockGroup(members, ["model.layers.0", "model.layers.1"])
    for p in grp.parameters():
        p.requires_grad_(False)
    b0 = rec["blocks"][0]
    others = {k: _dev(v) for k, v in b0["others"].items()}
    with torch.no_grad():
        fp_out = [S.block_forward(grp, *S.select_batch([t.to(DEV) for t in b0["inputs"]], others, [i]))
                  for i in range(len(b0["inputs"]))]
    b = dict(b0, fp_outputs=fp_out)
    iters = 24
    batches = [[(4 * i + j) % len(b0["inputs"]) for j in range(rec["batch_size"])] for i in range(iters)]
    q = _tune(grp, b, parse_scheme("MXFP4", {"act_bits": 16}), iters, batches, keep_arena=True)
    res = q.last_result
    assert res.used_cuda_graph and len(res.quantized_layers) == 32
    assert res.best_loss <= res.losses[0] + 1e-12
    experts = [n for n in res.quantized_layers if ".experts." in n]
    assert len(experts) == 24 and {n.split(".")[1] for n in experts} == {"0", "1"}
    for n in experts:
        assert float(q.last_arena.layer_views(n)["value"].abs().sum()) > 0, n


def _llama3(state):
    from transformers import LlamaConfig, LlamaForCausalLM

    cfg = LlamaConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=3, num_attention_heads=4,
                      num_key_value_heads=2, vocab_size=128, max_position_embeddings=64, rms_norm_eps=1e-5,
                      rope_theta=10000.0, tie_word_embeddings=False)
    m = LlamaForCausalLM(cfg).to(torch.bfloat16).eval()
    m.load_state_dict(state)
    return m


def _autoround(rec, nblocks, **kw):
    tokens = rec["tokens"]
    bs = rec["batch_size"]
    return AutoRound(_llama3(rec["init_state"]), tokenizer=_Tok(), iters=rec["iters"], nsamples=tokens.shape[0],
                     seqlen=tokens.shape[1], batch_size=bs, dataset=[tokens[i:i + bs] for i in range(0, tokens.shape[0], bs)],
                     device_map=0, seed=42, nblocks=nblocks, **kw)


def _read(out):
    from safetensors import safe_open

    got = {}
    with safe_open(os.path.join(out, "model.safetensors"), "pt") as f:
        for k in f.keys():
            got[k] = f.get_tensor(k)
    return got, json.load(open(os.path.join(out, "config.json")))["quantization_config"]


def test_autoround_nblocks2_quantize_and_save(tmp_path):
    """Public API on the 3-layer tiny Llama: groups [0, 1] and [2], every linear of every block packed, the checkpoint's
    quantization_config equal to the nblocks=1 run's, and the saved model loads and runs a forward."""
    rec = _load("w4a16_sym_g32")
    kw = SCHEMES["w4a16_sym_g32"][0]
    ar = _autoround(rec, 2, **kw)
    model, _ = ar.quantize_and_save(str(tmp_path / "g2"), format="auto_round")
    assert [r["block"] for r in ar.block_results] == ["model.layers.0", "model.layers.2"]
    assert [r["blocks"] for r in ar.block_results] == [["model.layers.0", "model.layers.1"], ["model.layers.2"]]
    for r in ar.block_results:
        assert r["cuda_graph"] and r["best_loss"] <= r["init_loss"] * (1 + 1e-6)
        assert set(r["phases_ms"]) == {"ref_forward_ms", "tune_ms", "q_forward_ms", "pack_ms"}
    # the tuned group's output MSE needs its quantised-chain forward, which only a group followed by another one runs
    assert ar.block_results[0]["block_mse"] > 0 and ar.block_results[1]["block_mse"] is None
    packed = {n for n, m in model.named_modules() if isinstance(m, QuantLinear)}
    assert len(packed) == 21 and not any(type(m) is nn.Linear for n, m in model.model.layers.named_modules())
    got, cfg = _read(str(tmp_path / "g2"))
    for n in packed:
        assert f"{n}.qweight" in got and f"{n}.scales" in got, n

    one = _autoround(rec, 1, **kw)
    one.quantize_and_save(str(tmp_path / "g1"), format="auto_round")
    assert all("blocks" not in r for r in one.block_results) and len(one.block_results) == 3
    got1, cfg1 = _read(str(tmp_path / "g1"))
    assert cfg == cfg1
    assert set(got) == set(got1) and all(got[k].dtype == got1[k].dtype and got[k].shape == got1[k].shape for k in got)

    # load: a fresh model takes the unpacked weights and the checkpoint's other tensors, then runs a forward
    fresh = _llama3(rec["init_state"])
    for n, m in list(fresh.named_modules()):
        if f"{n}.qweight" in got:
            nn_, k = m.weight.shape
            w, _ = ops.unpack_int(got[f"{n}.qweight"].to(DEV), got[f"{n}.qzeros"].to(DEV), got[f"{n}.scales"].to(DEV),
                                  nn_, k, 4, 32, True)
            m.weight.data.copy_(w.cpu())
    fresh.load_state_dict({k: v for k, v in got.items() if k in fresh.state_dict()}, strict=False)
    fresh = fresh.to(DEV)
    with torch.no_grad():
        logits = fresh(rec["tokens"][:2].to(DEV)).logits
    ref = _llama3(rec["init_state"]).to(DEV)
    with torch.no_grad():
        ref_logits = ref(rec["tokens"][:2].to(DEV)).logits
    assert torch.isfinite(logits).all()
    assert float((logits.float() - ref_logits.float()).pow(2).mean()) < float(ref_logits.float().pow(2).mean())


def test_autoround_nblocks2_alg_ext_w2_sym(tmp_path):
    """enable_alg_ext with W2A16 sym: imatrix hooks on the group's FP forward, searched init scales and the outlier-suppressed
    loss at the group's output."""
    rec = _load("w4a16_sym_g32")
    ar = _autoround(rec, 2, scheme="W2A16", group_size=32, enable_alg_ext=True)
    ar.quantize()
    assert len(ar.block_results) == 2
    for r in ar.block_results:
        assert r["cuda_graph"] and r["best_loss"] <= r["init_loss"] * (1 + 1e-6)
        assert all(l == l and l > 0 for l in r["losses"])
    q = sum(1 for m in ar.model.model.layers.modules() if type(m) is nn.Linear and hasattr(m, "scale"))
    assert q == 21


# ------------------------------------------------------------------------------------------------------ data parallel
ITERS = 24


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _dp_tune(rank, world, dev, graph):
    rec = _load("w4a16_sym_g32")
    b = rec["blocks"][0]
    grp = _group(b["block_state"], dev)
    q = SignRoundQuantizer(parse_scheme("W4A16", {"group_size": 32}), iters=ITERS, batch_size=rec["batch_size"],
                           dp=DataParallel(rank, world, None), use_cuda_graph=graph)
    batches = [[(4 * i + j) % len(b["inputs"]) for j in range(rec["batch_size"])] for i in range(ITERS)]
    q.quantize_block(grp, [t.to(dev) for t in b["inputs"]], b["others"], [t.to(dev) for t in b["fp_outputs"]], None, None,
                     input_ids=b["input_ids"], sampler=S.ReplaySampler(batches))
    res = q.last_result
    masks = [(ids != -100).to(torch.long) for ids in b["input_ids"]]
    return {"losses": res.losses, "best_iter": res.best_iter, "graph": res.used_cuda_graph,
            "weights": {n: grp.get_submodule(n).weight.detach().cpu() for n in res.quantized_layers},
            "scales": {n: grp.get_submodule(n).scale.detach().float().cpu() for n in res.quantized_layers},
            "mse": _mse(grp, b["inputs"], b["others"], b["fp_outputs"], masks, dev)}


def _dp_worker(rank, world, port, backend, out_dir):
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    try:
        if backend == "nccl":
            dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
        else:
            dist.init_process_group("gloo", rank=rank, world_size=world)
        torch.save(("ok", _dp_tune(rank, world, dev, graph=(backend == "nccl"))), os.path.join(out_dir, f"rank{rank}.pt"))
    except Exception as e:  # noqa: BLE001
        import traceback
        torch.save(("error: " + repr(e) + "\n" + traceback.format_exc(), None), os.path.join(out_dir, f"rank{rank}.pt"))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def _dp_check(backend, tmp_path, world=2):
    ctx = mp.get_context("spawn")
    port = _free_port()
    procs = [ctx.Process(target=_dp_worker, args=(r, world, port, backend, str(tmp_path))) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=600)
        assert not p.is_alive(), "data-parallel worker hung"
    got = {}
    for rank in range(world):
        f = os.path.join(str(tmp_path), f"rank{rank}.pt")
        assert os.path.exists(f), f"rank {rank} died without a result (exit code {procs[rank].exitcode})"
        status, r = torch.load(f, weights_only=False)
        assert status == "ok", f"rank {rank}: {status}"
        got[rank] = r
    one = _dp_tune(0, 1, DEV, graph=(backend == "nccl"))
    r0 = got[0]
    for r in range(1, world):
        assert got[r]["losses"] == r0["losses"] and got[r]["best_iter"] == r0["best_iter"]
        for n in r0["weights"]:
            assert torch.equal(got[r]["weights"][n], r0["weights"][n]), n
            assert torch.equal(got[r]["scales"][n], r0["scales"][n]), n
    if backend == "nccl":
        assert r0["graph"]
    assert len(r0["weights"]) == 14
    assert r0["losses"][0] == pytest.approx(one["losses"][0], rel=1e-4)
    assert r0["mse"] == pytest.approx(one["mse"], rel=0.25), (r0["mse"], one["mse"])
    assert min(r0["losses"]) <= r0["losses"][0]


def test_group_two_ranks_one_gpu_gloo_equals_one_rank(tmp_path):
    _dp_check("gloo", tmp_path)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="one rank per GPU over NCCL needs >= 2 GPUs")
def test_group_two_ranks_nccl_graph_equals_one_rank(tmp_path):
    _dp_check("nccl", tmp_path)
