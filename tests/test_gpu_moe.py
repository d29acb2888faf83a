"""GPU parity of the MoE path (SURVEY.md 8 f2): device-side routing, grouped wgmma GEMMs and the combine kernels of
auto_round_b200/moe.py against the reference's expert loop restated in oracle/moe_loop.py (auto_round/modeling/fused_moe/
moe_experts_interface.py:173-260), and a whole Mixtral block tuned against the oracle on the reference's own fixture."""
import copy
import os
import random

import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("CUDA device required", allow_module_level=True)

from auto_round_b200 import ops  # noqa: E402
from auto_round_b200.moe import PROJS, GroupedExperts, unfuse_experts  # noqa: E402
from auto_round_b200.quantizer import SignRoundQuantizer  # noqa: E402
from auto_round_b200.schemes import parse_scheme  # noqa: E402
from oracle import signround as S  # noqa: E402
from oracle.moe_loop import LoopExperts, unfuse_experts_cpu  # noqa: E402

DEV = torch.device("cuda", 0)


class _Fused(torch.nn.Module):
    def __init__(self, e, h, inter, seed=0):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.gate_up_proj = torch.nn.Parameter((torch.randn(e, 2 * inter, h, generator=g) * 0.05).bfloat16())
        self.down_proj = torch.nn.Parameter((torch.randn(e, h, inter, generator=g) * 0.05).bfloat16())
        self.act_fn = torch.nn.SiLU()


def _routing(tokens, e, k, seed, skip_expert=None):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(tokens, e, generator=g)
    if skip_expert is not None:
        logits[:, skip_expert] = -1e9                  # an expert no token is routed to
    w, idx = torch.topk(torch.softmax(logits, -1), k, dim=-1)
    return idx, (w / w.sum(-1, keepdim=True)).bfloat16()


@pytest.mark.parametrize("tokens,e,k,e_begin,e_local", [(300, 4, 2, 0, 4), (1000, 8, 2, 0, 8), (1000, 8, 2, 4, 4), (257, 3, 1, 1, 2),
                                                        (16384, 8, 2, 0, 8),       # Mixtral at a production token count
                                                        (4096, 128, 8, 64, 32),    # EP rank at the 32-local-expert limit
                                                        (2048, 64, 8, 32, 32),
                                                        (5, 32, 1, 0, 32)])        # fewer pairs than threads
def test_route_tables(tokens, e, k, e_begin, e_local):
    idx, _ = _routing(tokens, e, k, seed=tokens)
    ids = idx.reshape(-1).to(DEV)
    route = ops.moe_route(ops.MoeRoute(tokens * k, e_local, DEV), ids, e_begin)
    torch.cuda.synchronize()
    ids_c = ids.cpu()
    counts = torch.bincount(ids_c, minlength=e)[e_begin:e_begin + e_local]
    assert route.counts.cpu().tolist() == counts.tolist()
    padded = (counts + 255) // 256 * 256
    offs = [0] + torch.cumsum(padded, 0).tolist()
    assert route.offsets.cpu().tolist() == offs
    rop, por = route.row_of_pair.cpu(), route.pair_of_row.cpu()
    local = (ids_c >= e_begin) & (ids_c < e_begin + e_local)
    assert bool((rop[~local] == -1).all()) and bool((rop[local] >= 0).all())
    for j in range(e_local):                            # rows of expert j: a permutation of its pairs, in pair order (stable)
        pairs = torch.nonzero(ids_c == e_begin + j).reshape(-1)
        assert rop[pairs].tolist() == list(range(offs[j], offs[j] + len(pairs)))
        assert por[offs[j]:offs[j] + len(pairs)].tolist() == pairs.tolist()
        assert bool((por[offs[j] + len(pairs):offs[j + 1]] == -1).all())
    assert bool((por[offs[-1]:] == -1).all())
    nmt = int(route.num_mt)
    mt = route.mtab.cpu()[:2 * nmt].reshape(-1, 2).tolist()
    want = [[m0, j] for j in range(e_local) for m0 in range(offs[j], offs[j + 1], 256)]
    assert mt == want
    kt = route.ktab.cpu()[:3 * int(route.num_active)].reshape(-1, 3).tolist()
    assert kt == [[j, offs[j], int(padded[j])] for j in range(e_local) if counts[j] > 0]


@pytest.mark.parametrize("tokens,e,k,h,inter,skip", [(300, 4, 2, 64, 128, None), (1000, 8, 2, 256, 512, 5), (64, 4, 2, 64, 128, 0)])
def test_grouped_forward_matches_expert_loop(tokens, e, k, h, inter, skip):
    fused = _Fused(e, h, inter, seed=tokens)
    ref = LoopExperts(fused).to(DEV)
    mod = GroupedExperts(copy.deepcopy(fused).to(DEV))
    x = (torch.randn(tokens, h, generator=torch.Generator().manual_seed(1)) * 0.5).bfloat16().to(DEV)
    idx, w = _routing(tokens, e, k, seed=7, skip_expert=skip)
    with torch.no_grad():
        want = ref(x, idx.to(DEV), w.to(DEV))
        got = mod(x, idx.to(DEV), w.to(DEV))
    scale = want.float().abs().max()
    assert float((got.float() - want.float()).abs().max() / scale) < 2e-2          # bf16 GEMM outputs, different sum order


def test_grouped_backward_matches_autograd_of_the_loop():
    """Tuning mode: the grouped backward's input gradient, routing-weight gradient and the bf16 weight gradients dWq of every
    expert against torch autograd through the reference loop run on the SAME fake-quant weights."""
    tokens, e, k, h, inter = 500, 4, 2, 64, 256
    fused = _Fused(e, h, inter, seed=3)
    blk = torch.nn.Module()
    blk.experts = GroupedExperts(copy.deepcopy(fused).to(DEV))
    q = SignRoundQuantizer(parse_scheme("MXFP4", {"act_bits": 16}), iters=1)
    wrapped, arena = q.wrapper_block(blk)
    mod = blk.experts
    mod.bind_wrapped(None)
    for wl in wrapped.values():
        wl.refresh_wq()
        wl.on_grad = None
    ref = LoopExperts(fused).to(DEV)
    for i in range(e):
        for p in PROJS:
            getattr(getattr(ref, str(i)), p).weight.data.copy_(mod.layer(i, p).wq)
            getattr(getattr(ref, str(i)), p).weight.requires_grad_(True)
    idx, w = _routing(tokens, e, k, seed=11, skip_expert=2)
    x = (torch.randn(tokens, h, generator=torch.Generator().manual_seed(5)) * 0.5).bfloat16().to(DEV)
    gout = (torch.randn(tokens, h, generator=torch.Generator().manual_seed(6)) * 0.1).bfloat16().to(DEV)
    xr, wr = x.clone().requires_grad_(True), w.to(DEV).clone().requires_grad_(True)
    ref(xr, idx.to(DEV), wr).backward(gout)
    xg, wg = x.clone().requires_grad_(True), w.to(DEV).clone().requires_grad_(True)
    mod(xg, idx.to(DEV), wg).backward(gout)

    def close(a, b, tol):
        return float((a.float() - b.float()).abs().max() / b.float().abs().max().clamp_min(1e-12)) < tol

    assert close(xg.grad, xr.grad, 3e-2)
    assert close(wg.grad, wr.grad, 3e-2)
    for i in range(e):
        for p in PROJS:
            want = getattr(getattr(ref, str(i)), p).weight.grad
            got = mod.layer(i, p).gq
            if i == 2:
                assert want is None or float(want.abs().max()) == 0.0            # no token -> no gradient ...
                assert float(got.abs().max()) == 0.0                              # ... and the buffer is left untouched
            else:
                assert close(got, want, 3e-2), (i, p)
    assert mod.route_for(tokens * k, e, DEV).counts.cpu().tolist()[2] == 0


def _mixtral_block(state, grouped: bool, device):
    from transformers import MixtralConfig
    from transformers.models.mixtral.modeling_mixtral import MixtralDecoderLayer

    cfg = MixtralConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4,
                        num_key_value_heads=2, vocab_size=128, max_position_embeddings=64, num_local_experts=4,
                        num_experts_per_tok=2, tie_word_embeddings=False)
    cfg._attn_implementation = "sdpa"
    blk = MixtralDecoderLayer(cfg, 0).to(torch.bfloat16).eval()
    if grouped:
        blk = blk.to(device)
        assert unfuse_experts(blk) == 1
    else:
        assert unfuse_experts_cpu(blk) == 1
    blk.load_state_dict(state)
    return blk.to(device)


def test_mixtral_block_vs_oracle(golden_dir):
    """BASELINE.json config 5's scheme (MXFP4 weight-only) on the reference's tiny 4-expert Mixtral fixture: grouped wgmma
    path + CUDA graph vs the oracle loop, same batches (bars of tests/test_gpu_engine.py).  The oracle (plain torch) runs on
    the GPU here: top-2 routing is discontinuous, and the router's bf16 GEMM on the CPU sends 1 of the fixture's 64 tokens to
    another expert than the same GEMM on the GPU, which alone moves the loss by 7 % (tools/diag_moe.py: oracle-CPU 3.12e-6,
    oracle-GPU 3.346e-6, this engine 3.349e-6).  The CPU oracle itself is pinned bit-exact to the reference
    (tests/test_oracle_golden.py::test_tune_block_mixtral_moe_matches_reference_bit_exact)."""
    from test_gpu_engine import _block_mse

    rec = torch.load(os.path.join(golden_dir, "block_mixtral_mxfp4.pt"), weights_only=False)
    b = rec["blocks"][0]
    osc = S.LayerScheme(4, 32, True, "mx_fp")
    masks = [(ids != -100).to(torch.long) for ids in b["input_ids"]]
    iters = 40
    random.seed(4321)
    oblk = _mixtral_block(b["block_state"], False, DEV)

    def dev(o):
        if isinstance(o, torch.Tensor):
            return o.to(DEV)
        return type(o)(dev(x) for x in o) if isinstance(o, (list, tuple)) else o

    ores = S.tune_block(oblk, [t.to(DEV) for t in b["inputs"]], {k: dev(v) for k, v in b["others"].items()},
                        [t.to(DEV) for t in b["fp_outputs"]], lambda n, m: osc, iters=iters, batch_size=rec["batch_size"],
                        token_masks=[m.to(DEV) for m in masks])
    o_mse = _block_mse(oblk, b["inputs"], b["others"], b["fp_outputs"], masks, DEV)
    blk = _mixtral_block(b["block_state"], True, DEV)
    for p in blk.parameters():
        p.requires_grad_(False)
    q = SignRoundQuantizer(parse_scheme("MXFP4", {"act_bits": 16}), iters=iters, batch_size=rec["batch_size"])
    q.quantize_block(blk, [t.to(DEV) for t in b["inputs"]], b["others"], [t.to(DEV) for t in b["fp_outputs"]], None, None,
                     input_ids=b["input_ids"], sampler=S.ReplaySampler(ores.batches))
    res = q.last_result
    assert res.used_cuda_graph, "a MoE block's iteration must be graph-captured (static shapes, device-side routing)"
    assert len(res.quantized_layers) == 16
    assert res.losses[0] == pytest.approx(ores.losses[0], rel=2e-2)
    g_mse = _block_mse(blk, b["inputs"], b["others"], b["fp_outputs"], masks, DEV)
    assert res.best_loss <= res.losses[0] + 1e-12
    # 40 sign-SGD iterations on 64-token batches with discontinuous top-2 routing: the two trajectories separate further than
    # for a dense block (tests/test_gpu_engine.py uses +-25 %); both must improve clearly on the RTN start
    assert g_mse == pytest.approx(o_mse, rel=0.4), (g_mse, o_mse)
    assert min(res.losses) < 0.9 * res.losses[0] and min(ores.losses) < 0.9 * ores.losses[0]
    for name, lay in b["layers"].items():
        mod = blk.get_submodule(name)
        assert type(mod) is torch.nn.Linear and tuple(mod.scale.shape) == tuple(lay["scale"].shape), name
