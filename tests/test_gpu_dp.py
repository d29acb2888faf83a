"""Data-parallel tuning on the GPU (SURVEY.md 8e): N ranks must reproduce the 1-rank result.

Two transports for the same code path (quantizer.quantize_block with DataParallel(rank, world)):
  * `gloo`, both ranks on cuda:0 -- runs on the single-GPU box of the round-end test tier: sample sharding, per-layer
    reduce-scatter of the bf16 dWq (emulated), row-sharded fused update (ar_fq_update rows [r0, r1)), all-gather of the
    new fake-quant weight and of the best-parameter shards, global loss for the best-iteration choice;
  * `nccl`, one rank per GPU, iteration captured as a CUDA graph with the collectives inside -- needs >= 2 GPUs
    (skipped on a single-GPU machine).
What is compared (the sum over ranks of bf16-rounded partial gradients is not the bf16 rounding of the total, so sign flips on
~zero gradients make the trajectories differ; SURVEY.md 8d bars):
  * both ranks end with bit-identical weights / scales (no broadcast is needed);
  * iteration-0 loss equals the 1-rank loss to 1e-4 (same parameters, the loss is a sum over the same samples);
  * after the first update >= 99 % of the rounding offsets V took the same step as on one rank;
  * final block MSE within +-25 % of the 1-rank run (the tolerance tests/test_gpu_engine.py uses against the oracle)."""
import os
import socket

import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("CUDA device required", allow_module_level=True)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ITERS = 24


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _tune(rank, world, dev, tag, scheme_kw, iters, graph, alg_ext=False):
    from auto_round_b200.quantizer import DataParallel, SignRoundQuantizer
    from auto_round_b200.schemes import parse_scheme
    from oracle import signround as S
    from oracle.tests_support import tiny_block

    rec = torch.load(os.path.join(GOLDEN, f"block_{tag}.pt"), weights_only=False)
    b = rec["blocks"][0]
    if "mixtral" in tag:
        from test_gpu_moe import _mixtral_block
        blk = _mixtral_block(b["block_state"], True, dev)
    else:
        blk = tiny_block(b["block_state"]).to(dev)
    for p in blk.parameters():
        p.requires_grad_(False)
    scheme = parse_scheme(scheme_kw["scheme"], {k: v for k, v in scheme_kw.items() if k != "scheme"})
    q = SignRoundQuantizer(scheme, iters=iters, batch_size=rec["batch_size"], dp=DataParallel(rank, world, None),
                           use_cuda_graph=graph, enable_alg_ext=alg_ext)
    batches = [[(4 * i + j) % len(b["inputs"]) for j in range(rec["batch_size"])] for i in range(iters)]
    nv = {n: g.to(dev).reshape(1) for n, g in b["nv_gs"].items()} if b.get("nv_gs") else None
    im = {n: t.to(dev) for n, t in b["imatrix"].items()} if alg_ext and b.get("imatrix") else None
    q.quantize_block(blk, [t.to(dev) for t in b["inputs"]], b["others"], [t.to(dev) for t in b["fp_outputs"]], None, None,
                     input_ids=b["input_ids"], nv_global_scales=nv, sampler=S.ReplaySampler(batches), keep_arena=True,
                     imatrices=im)
    res = q.last_result
    out = {"losses": res.losses, "best_iter": res.best_iter, "graph": res.used_cuda_graph,
           "weights": {n: blk.get_submodule(n).weight.detach().cpu() for n in res.quantized_layers},
           "scales": {n: blk.get_submodule(n).scale.detach().float().cpu() for n in res.quantized_layers}}
    # block MSE over all samples
    from test_gpu_engine import _block_mse
    masks = [(ids != -100).to(torch.long) for ids in b["input_ids"]]
    out["mse"] = _block_mse(blk, b["inputs"], b["others"], b["fp_outputs"], masks, dev)
    return out


def _first_step(rank, world, dev, tag, scheme_kw):
    """V after ONE iteration with lr = 1 (= -sign(dV)), full arena."""
    from auto_round_b200.quantizer import DataParallel, SignRoundQuantizer
    from auto_round_b200.schemes import parse_scheme
    from oracle import signround as S
    from oracle.tests_support import tiny_block

    rec = torch.load(os.path.join(GOLDEN, f"block_{tag}.pt"), weights_only=False)
    b = rec["blocks"][0]
    blk = tiny_block(b["block_state"]).to(dev)
    for p in blk.parameters():
        p.requires_grad_(False)
    scheme = parse_scheme(scheme_kw["scheme"], {k: v for k, v in scheme_kw.items() if k != "scheme"})
    q = SignRoundQuantizer(scheme, iters=1, batch_size=rec["batch_size"], dp=DataParallel(rank, world, None), lr=1.0,
                           use_cuda_graph=False)
    q.quantize_block(blk, [t.to(dev) for t in b["inputs"]], b["others"], [t.to(dev) for t in b["fp_outputs"]], None, None,
                     input_ids=b["input_ids"], sampler=S.ReplaySampler([list(range(rec["batch_size"]))]), keep_arena=True)
    a = q.last_arena
    return a.params[:a.clamp_begin].detach().cpu(), a


def _worker(rank, world, port, backend, tag, scheme_kw, alg_ext, out_dir):
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
        r = _tune(rank, world, dev, tag, scheme_kw, ITERS, graph=(backend == "nccl"), alg_ext=alg_ext)
        if "mixtral" not in tag:
            v1, arena = _first_step(rank, world, dev, tag, scheme_kw)
            # the parameter arena is sharded by rows under DP: gather the rows this rank owns from every rank
            full = torch.zeros_like(v1)
            for name, views in arena.views.items():
                o, n, shape = views["value"]
                per = shape[0] // world
                lo, hi = o + rank * per * shape[1], o + (rank + 1) * per * shape[1]
                full[lo:hi] = v1[lo:hi]
            full = full.to(dev)
            dist.all_reduce(full)
            r["v1"] = full.cpu()
        torch.save(("ok", r), os.path.join(out_dir, f"rank{rank}.pt"))
    except Exception as e:  # noqa: BLE001
        import traceback
        torch.save(("error: " + repr(e) + "\n" + traceback.format_exc(), None), os.path.join(out_dir, f"rank{rank}.pt"))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


CASES = {"mixtral_mxfp4": (dict(scheme="MXFP4", act_bits=16), False),      # expert parallelism: rank r owns experts [2r, 2r + 2)
         "w4a16_sym_g32": (dict(scheme="W4A16", group_size=32), False),
         "w2a16_asym_g32": (dict(scheme="W2A16", group_size=32, sym=False), False),
         "algext_w2a16_sym_g32": (dict(scheme="W2A16", group_size=32), True)}


def _check(tag, backend, tmp_path, world=2):
    scheme_kw, alg_ext = CASES[tag]
    ctx = mp.get_context("spawn")
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, backend, tag, scheme_kw, alg_ext, str(tmp_path)))
             for r in range(world)]
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
    dev = torch.device("cuda", 0)
    one = _tune(0, 1, dev, tag, scheme_kw, ITERS, graph=(backend == "nccl"), alg_ext=alg_ext)
    v1_one = None if "mixtral" in tag else _first_step(0, 1, dev, tag, scheme_kw)[0]
    r0 = got[0]
    for r in range(1, world):                      # identical results on every rank, no broadcast needed
        assert got[r]["losses"] == r0["losses"] and got[r]["best_iter"] == r0["best_iter"]
        for n in r0["weights"]:
            assert torch.equal(got[r]["weights"][n], r0["weights"][n]), n
            assert torch.equal(got[r]["scales"][n], r0["scales"][n]), n
    if backend == "nccl":
        assert r0["graph"], "the data-parallel iteration must be captured as a CUDA graph (collectives inside)"
    assert r0["losses"][0] == pytest.approx(one["losses"][0], rel=1e-4)
    if not alg_ext and v1_one is not None:
        agree = float((r0["v1"] == v1_one).float().mean())
        assert agree >= 0.99, agree
    # MoE: top-2 routing is discontinuous -- the sharded attention layers move a few tokens to other experts, so the two
    # trajectories differ more than for a dense block (tests/test_gpu_moe.py explains the 7 % a single token makes)
    assert r0["mse"] == pytest.approx(one["mse"], rel=0.4 if "mixtral" in tag else 0.25), (r0["mse"], one["mse"])
    assert min(r0["losses"]) <= r0["losses"][0]


@pytest.mark.parametrize("tag", list(CASES))
def test_two_ranks_one_gpu_gloo_equals_one_rank(tag, tmp_path):
    _check(tag, "gloo", tmp_path)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="one rank per GPU over NCCL needs >= 2 GPUs")
@pytest.mark.parametrize("tag", ["w4a16_sym_g32", "algext_w2a16_sym_g32", "mixtral_mxfp4"])
def test_two_ranks_nccl_graph_equals_one_rank(tag, tmp_path):
    _check(tag, "nccl", tmp_path)
