"""bench.py -- block-wise SignRound calibration on H100; headline: Llama-3-8B W4A16 (sym, g128), BASELINE.json configs[1].

    python bench.py --gpus N --steps K --warmup W [--config NAME]      # our arm  (torchrun for N > 1)
    python bench.py --impl reference --gpus N --steps K --warmup W     # the reference's CPU path (oracle port)
    python bench.py ... --dump-outputs DIR                              # + the last timed block's packed tensors as .npy

A STEP is one transformer block taken through the whole hot path exactly as the reference's `quantization tuning time`
span counts it (compressors/orchestrator.py:631 -> 792): FP reference forward over all 128 calibration samples, `iters`
sign-SGD iterations (batch 8 x 2048 tokens), forward of the tuned block (next block's inputs), unwrap, low-bit pack.  All
blocks of a model have the same shapes, so `value` (seconds for the whole model) is ms_per_step * n_blocks; with --steps
n_blocks it is measured outright.  Weights are random-init (HF default init, seed 0), calibration tokens are synthetic
(seed 1): there is no network.

Both numbers come from ONE pass through the public API `AutoRound(model_on_host, ...).quantize()`:
  e2e    device time of the whole per-block span: H2D of the block's bf16 weights from pinned host memory ->
         compute -> D2H of the packed tensors (CUDA events, max over ranks)
  value  the same span minus the H2D / D2H segments (inputs already resident in HBM)
Beside them (N = 1), each outside the timed region:
  roofline              the GEMM launch mix of one iteration replayed alone (vs the BURST cuBLAS peak) and, under CUPTI, inside
                        a running iteration (vs the SUSTAINED peak)
  per_block_mse_vs_ref  block 0 tuned by the reference's algorithm (oracle/, torch eager on the same GPU, same batches):
                        final output MSE of both against the FP block -- the second half of BASELINE.json's metric
  gpu_eager_baseline    the reference's own GPU path (eager ATen + cuBLAS + autograd through the fake-quant graph, i.e. the
                        oracle on `cuda`) per iteration at the full shape -- what a user has today on this GPU
  cpu_baseline          the reference's CPU path on the host cores, bounded sample (see cpu_steps)
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

NSAMPLES, SEQLEN, BATCH = 128, 2048, 8

# BASELINE.json configs (SURVEY.md 8d / A.4).  `linears`: (name, N, K, input needs a gradient) of one block.
_LLAMA_LIN = [("q", 4096, 4096, False), ("k", 1024, 4096, False), ("v", 1024, 4096, False), ("o", 4096, 4096, True),
              ("gate", 14336, 4096, True), ("up", 14336, 4096, True), ("down", 4096, 14336, True)]
_QWEN_LIN = [("q", 3584, 3584, False), ("k", 512, 3584, False), ("v", 512, 3584, False), ("o", 3584, 3584, True),
             ("gate", 18944, 3584, True), ("up", 18944, 3584, True), ("down", 3584, 18944, True)]
CONFIGS = {
    "llama3_8b_w4a16": dict(
        metric="Llama-3-8B W4A16 calib wall-clock (s) @200 iters", model="llama3_8b", n_blocks=32, iters=200,
        scheme=dict(scheme="W4A16"), spec=("int_sym", 4, 128), linears=_LLAMA_LIN,
        workload="Llama-3-8B W4A16 sym g128 iters=%d nsamples=128 seqlen=2048 batch=8 on %dxH100"),
    "w2asym_algext": dict(
        metric="Llama-3-8B W2A16 asym g32 enable_alg_ext calib wall-clock (s) @1000 iters", model="llama3_8b", n_blocks=32,
        iters=1000, scheme=dict(scheme="W2A16", group_size=32, sym=False, enable_alg_ext=True), spec=("int_asym", 2, 32),
        linears=_LLAMA_LIN, workload="Llama-3-8B W2A16 asym g32 enable_alg_ext iters=%d nsamples=128 seqlen=2048 batch=8 on %dxH100"),
    "qwen2_nvfp4": dict(
        metric="Qwen2-7B NVFP4 (weight-only) calib wall-clock (s) @200 iters", model="qwen2_7b", n_blocks=28, iters=200,
        scheme=dict(scheme="NVFP4", act_bits=16, act_data_type="float"), spec=("nv_fp4", 4, 16), linears=_QWEN_LIN,
        workload="Qwen2-7B NVFP4 weight-only g16 iters=%d nsamples=128 seqlen=2048 batch=8 on %dxH100"),
}
_MIXTRAL_LIN = [("q", 4096, 4096, False), ("k", 1024, 4096, False), ("v", 1024, 4096, False), ("o", 4096, 4096, True),
                # top-2 of 8 experts: per token two gate / up / down projections are active (the FLOP count of a step)
                ("e0.gate", 14336, 4096, True), ("e0.up", 14336, 4096, True), ("e0.down", 4096, 14336, True),
                ("e1.gate", 14336, 4096, True), ("e1.up", 14336, 4096, True), ("e1.down", 4096, 14336, True)]
CONFIGS["mixtral_mxfp4"] = dict(
    metric="Mixtral-8x7B MXFP4 (weight-only) calib wall-clock (s) @200 iters", model="mixtral_8x7b", n_blocks=32, iters=200,
    scheme=dict(scheme="MXFP4", act_bits=16), spec=("mx_fp4", 4, 32), linears=_MIXTRAL_LIN,
    p_block=4096 * 4096 * 2 + 1024 * 4096 * 2 + 8 * 3 * 14336 * 4096,
    workload="Mixtral-8x7B MXFP4 weight-only g32 iters=%d nsamples=128 seqlen=2048 batch=8 on %dxH100")
MODELS = {
    "mixtral_8x7b": ("MixtralConfig", "MixtralForCausalLM", dict(hidden_size=4096, intermediate_size=14336, num_attention_heads=32,
                                                              num_key_value_heads=8, vocab_size=32000, rope_theta=1000000.0,
                                                              rms_norm_eps=1e-5, max_position_embeddings=32768,
                                                              num_local_experts=8, num_experts_per_tok=2)),
    "llama3_8b": ("LlamaConfig", "LlamaForCausalLM", dict(hidden_size=4096, intermediate_size=14336, num_attention_heads=32,
                                                         num_key_value_heads=8, vocab_size=128256, rope_theta=500000.0,
                                                         rms_norm_eps=1e-5, max_position_embeddings=8192)),
    "qwen2_7b": ("Qwen2Config", "Qwen2ForCausalLM", dict(hidden_size=3584, intermediate_size=18944, num_attention_heads=28,
                                                        num_key_value_heads=4, vocab_size=152064, rope_theta=1000000.0,
                                                        rms_norm_eps=1e-6, max_position_embeddings=32768)),
}


def flops_per_step(cfg, iters):
    """SURVEY.md 8(d): linear-layer FLOPs of one step (one block): `iters` iterations (3 GEMMs per linear, q/k/v need no
    grad-in) + 2 full-set forwards."""
    p_block = sum(n * k for _, n, k, _ in cfg["linears"])
    p_nodx = sum(n * k for _, n, k, dx in cfg["linears"] if not dx)
    return iters * (BATCH * SEQLEN) * (6 * p_block - 2 * p_nodx) + 2 * 2 * (NSAMPLES * SEQLEN) * p_block


def peaks():
    """MEASURED_PEAKS.json (driver-written): `bf16_tflops` = burst (a kernel timed alone), `bf16_tflops_sustained` = inside
    a long step; fallback = NVIDIA's H100 SXM data sheet (dense bf16 / HBM3 at 700 W), a ceiling rather than a measured rate."""
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return {"burst": d.get("bf16_tflops"), "sustained": d.get("bf16_tflops_sustained", d.get("bf16_tflops")),
                "hbm_gbs": d.get("hbm_gbs"), "source": "MEASURED_PEAKS.json"}
    return {"burst": 989.0, "sustained": 989.0, "hbm_gbs": 3350.0, "source": "fallback (H100 SXM data sheet, 700 W)"}


class ClockSampler(threading.Thread):
    """SM clock / throttle reasons during the timed region, through NVML in-process (pynvml).  Spawning `nvidia-smi` twice
    a second takes driver-wide locks and slowed the measured run by ~10 % on one GPU and several-fold on eight, so the
    CLI is only the fallback, at a 5 s period."""

    def __init__(self, index=0):
        super().__init__(daemon=True)
        self.index, self.rows, self.stop_flag = index, [], False
        self.nvml = None
        try:
            import pynvml
            pynvml.nvmlInit()
            self.nvml = pynvml
            self.handle = pynvml.nvmlDeviceGetHandleByIndex(index)
            self.max_sm = pynvml.nvmlDeviceGetMaxClockInfo(self.handle, pynvml.NVML_CLOCK_SM)
        except Exception:  # noqa: BLE001
            self.nvml = None

    def run(self):
        if self.nvml is not None:
            n = self.nvml
            bits = {"hw_slowdown": 0x8, "hw_thermal_slowdown": 0x40, "sw_thermal_slowdown": 0x20, "sw_power_cap": 0x4}
            while not self.stop_flag:
                try:
                    sm = n.nvmlDeviceGetClockInfo(self.handle, n.NVML_CLOCK_SM)
                    try:
                        r = n.nvmlDeviceGetCurrentClocksEventReasons(self.handle)
                    except Exception:  # noqa: BLE001
                        r = n.nvmlDeviceGetCurrentClocksThrottleReasons(self.handle)
                    self.rows.append([str(sm), str(self.max_sm)] + ["Active" if (r & b) else "Not Active" for b in bits.values()])
                except Exception:  # noqa: BLE001
                    pass
                time.sleep(0.5)
            return
        q = "clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown," \
            "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"
        while not self.stop_flag:
            try:
                out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", str(self.index)],
                                     capture_output=True, text=True, timeout=10).stdout.strip()
                if out:
                    self.rows.append([c.strip() for c in out.split(",")])
            except Exception:  # noqa: BLE001
                pass
            time.sleep(5.0)

    def summary(self):
        if not self.rows:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["no clock samples"]}
        sm = sorted(int(r[0]) for r in self.rows if r[0].isdigit())
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = [n for i, n in enumerate(names) if any(r[2 + i].lower().startswith("active") for r in self.rows if len(r) > 2 + i)]
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": int(self.rows[0][1]) if self.rows[0][1].isdigit() else None,
                "reasons": reasons, "samples": len(self.rows), "source": "nvml" if self.nvml is not None else "nvidia-smi"}


class _Tok:
    pad_token_id = None
    pad_token = None

    def save_pretrained(self, *a, **k):
        return None


def build_model(name: str, n_layers: int, device, seed: int = 0):
    """Random-init model of the named architecture with `n_layers` blocks, bf16, in PINNED host memory.  Initialised on
    the GPU (fast) with HF's default init, then moved to the host: the public API receives a host model."""
    import transformers

    cfg_cls, model_cls, kw = MODELS[name]
    cfg = getattr(transformers, cfg_cls)(num_hidden_layers=n_layers, tie_word_embeddings=False, **kw)
    cfg._attn_implementation = "sdpa"
    torch.manual_seed(seed)
    with torch.device("meta"):
        model = getattr(transformers, model_cls)(cfg)
    model = model.to_empty(device=device).to(torch.bfloat16)
    g = torch.Generator(device=device).manual_seed(seed)
    for pname, p in model.named_parameters():
        if p.dim() >= 2:
            p.data.normal_(0.0, cfg.initializer_range, generator=g)
        elif pname.endswith("bias"):
            p.data.zero_()
        else:
            p.data.fill_(1.0)
    # rotary inv_freq is a non-persistent buffer lost by to_empty(): rebuild it
    rot = model.model.rotary_emb
    inv, _ = rot.rope_init_fn(cfg, device) if hasattr(rot, "rope_init_fn") else (None, None)
    if inv is not None:
        rot.inv_freq = inv
        rot.original_inv_freq = inv.clone()
    model = model.cpu()
    for p in model.parameters():
        p.data = p.data.pin_memory()
    return model.eval()


def build_llama(n_layers: int, device, seed: int = 0):
    return build_model("llama3_8b", n_layers, device, seed)


def line_config(cfg, iters, world, n_measured):
    """The `config` object: identical for our arm and the reference arm (same workload)."""
    return {"workload": cfg["workload"] % (iters, world),
            "step": "one decoder block through the tuning span (ref fwd, %d sign-SGD iters, q fwd, unwrap, pack)" % iters,
            "value_is": "ms_per_step x %d blocks (identical shapes)%s" % (cfg["n_blocks"], "" if n_measured != cfg["n_blocks"] else "; measured over all"),
            "parallelism": "dp%d (calibration samples sharded; per layer: reduce-scatter of the bf16 dWq, row-sharded fused update, "
                           "all-gather of the next fake-quant weight, overlapped with the backward%s)"
                           % (world, "; MoE experts: expert-parallel ownership, all-gather of tokens + reduce-scatter of outputs" if "mixtral" in cfg["model"] else ""),
            "l2": "inputs larger than L2 (per-iteration working set 3.4 GB >> 50 MB)"}


def run_ours(args):
    import torch.distributed as dist

    cfg = CONFIGS[args.config]
    iters = args.iters if args.iters else cfg["iters"]
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    from auto_round_b200 import AutoRound, ops

    W, K = args.warmup, args.steps
    model = build_model(cfg["model"], W + K, dev)
    orig_block0 = copy.deepcopy(model.model.layers[0]) if (world == 1 and not args.no_mse_check) else None
    vocab = MODELS[cfg["model"]][2]["vocab_size"]
    tokens = torch.randint(0, vocab, (NSAMPLES, SEQLEN), generator=torch.Generator().manual_seed(1))
    dataset = [tokens[i:i + BATCH] for i in range(0, NSAMPLES, BATCH)]
    ar = AutoRound(model, tokenizer=_Tok(), iters=iters, nsamples=NSAMPLES, seqlen=SEQLEN, batch_size=BATCH, dataset=dataset,
                   device_map=local, seed=42, **cfg["scheme"])
    ar._pack_on_the_fly = True

    ev = {"segs": []}
    clocks = ClockSampler(local)
    launches0 = [0]

    def hook(bi, phase):
        # phases per block: "h2d0" -> "compute0" -> "d2h0" -> "done"
        if bi < W:
            return
        e = torch.cuda.Event(enable_timing=True)
        if bi == W and phase == "h2d0":
            torch.cuda.synchronize()
            if world > 1:
                dist.barrier()
            launches0[0] = ops.LAUNCHES[0]
            if rank == 0:
                clocks.start()
        e.record()
        ev["segs"].append((bi, phase, e))

    ar.block_hook = hook
    ar.quantize()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    clocks.stop_flag = True
    launches = ops.LAUNCHES[0] - launches0[0]

    by = {}
    for bi, phase, e in ev["segs"]:
        by.setdefault(bi, {})[phase] = e
    e2e_ms = by[W]["h2d0"].elapsed_time(by[W + K - 1]["done"])
    copy_ms = sum(b["h2d0"].elapsed_time(b["compute0"]) + b["d2h0"].elapsed_time(b["done"]) for b in by.values())
    comp_ms = e2e_ms - copy_ms
    t = torch.tensor([e2e_ms, comp_ms], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    e2e_ms, comp_ms = t.tolist()

    dp_probe = collective_probe(dev, world, cfg) if world > 1 else None
    dp_timeline = None
    if world > 1 and "mixtral" not in cfg["model"]:
        try:                                   # every rank runs the extra block (collectives inside); rank 0 reports it
            dp_timeline = iteration_timeline(dev, peaks(), cfg, args.config, dp=ar.dp)
        except Exception as e:  # noqa: BLE001
            dp_timeline = {"error": repr(e)[:200]}
    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return
    pk = peaks()
    nb = cfg["n_blocks"]
    ms_per_step = comp_ms / K
    value_s = ms_per_step * nb / 1e3
    e2e_s = (e2e_ms / K) * nb / 1e3
    flops_step = flops_per_step(cfg, iters)
    p_block = cfg.get("p_block") or sum(n * k for _, n, k, _ in cfg["linears"])
    hidden = MODELS[cfg["model"]][2]["hidden_size"]
    h2d = (p_block + 2 * hidden) * 2                                # bf16 linears + the two RMSNorm weights
    bits, g = cfg["spec"][1], cfg["spec"][2]
    d2h = int(p_block * bits / 8 + (p_block // g) * (2 + bits / 8) + hidden * 4 * 7)
    tune_ms = sum(r["phases_ms"]["tune_ms"] for r in ar.block_results[W:]) / K
    conf = line_config(cfg, iters, world, K)
    conf["step_tflops_per_gpu"] = round(flops_step / (ms_per_step / 1e3) / 1e12 / world, 1)
    mses = [r.get("block_mse") for r in ar.block_results[W:] if r.get("block_mse") is not None]
    line = {
        "metric": cfg["metric"], "value": round(value_s, 3), "unit": "s",
        "n_gpus": world, "steps": K, "warmup": W, "ms_per_step": round(ms_per_step, 2), "higher_is_better": False,
        "scaling": "strong", "vs_baseline": None, "dtype": "bf16", "data": "synthetic", "config": conf,
        "e2e": {"value": round(e2e_s, 3), "unit": "s", "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": int(d2h)},
        "gpu_launches": int(launches),
        "clocks": clocks.summary(),
        "step_fraction_of_gemm_roofline": round((flops_step / world / (pk["sustained"] * 1e12)) / (ms_per_step / 1e3), 4),
        "phases_ms_per_step": {k: round(sum(r["phases_ms"][k] for r in ar.block_results[W:]) / K, 1)
                               for k in ar.block_results[W]["phases_ms"]},
        "ms_per_iteration": round(tune_ms / iters, 3),
        "cuda_graph": bool(ar.block_results[W].get("cuda_graph")),
        "losses": {"block0_iter0": ar.block_results[0]["init_loss"], "block0_best": ar.block_results[0]["best_loss"],
                   "block0_best_iter": ar.block_results[0]["best_iter"]},
        "block_output_mse": {"timed_blocks": mses, "what": "mean over valid tokens of (tuned block - FP block)^2 on all 128 samples"},
    }
    if dp_probe is not None:
        line["dp_probe"] = dp_probe
    if dp_timeline is not None:
        line["dp_iteration_timeline"] = dp_timeline
    if world == 1:
        roof = gemm_roofline(dev, pk, cfg)
        if "mixtral" in cfg["model"]:
            roof["note"] = "dense replay of the ACTIVE launch mix (top-2 experts at T tokens each); the run itself uses the grouped kernels"
        else:
            try:
                roof["in_context"] = iteration_timeline(dev, pk, cfg, args.config)
            except Exception as e:  # noqa: BLE001 -- a diagnostic, never the value
                roof["in_context"] = {"error": repr(e)[:200]}
        line["roofline"] = roof
        if orig_block0 is not None:
            try:
                line["per_block_mse_vs_ref"] = mse_vs_reference(ar, model, orig_block0, cfg, iters, dev, line)
            except Exception as e:  # noqa: BLE001
                line["per_block_mse_vs_ref"] = {"error": repr(e)[:300]}
        if not args.no_cpu_baseline:
            line["cpu_baseline"] = cpu_baseline(cfg, steps=8, warmup=1, budget_s=args.cpu_budget)
    else:
        line["roofline"] = {"bound": "tensor", "note": "measured at N=1 (same kernels); see the N=1 line"}
    if args.dump_outputs:
        line["dumped_outputs"] = {"block": W + K - 1, **dump_outputs(model.model.layers[W + K - 1], args.dump_outputs)}
    print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


DUMP_BUDGET_BYTES = 60 << 20          # below 64 MB with the .npy headers


def dump_outputs(block, out_dir):
    """The packed tensors of the last timed block (what `quantize()` hands the caller for it: qweight / qzeros / scales /
    g_idx of every quantized linear) as DIR/<layer>.<buffer>.npy -- integers as float64 (exact), floats as float32.  A
    tensor larger than its share of the budget is replaced by a fixed sample (seed 0, sorted flat indices), so two builds
    run with the same arguments can be compared element for element."""
    import numpy as np

    os.makedirs(out_dir, exist_ok=True)
    bufs = [(n, b) for n, b in block.named_buffers() if b.numel() > 0]
    share = DUMP_BUDGET_BYTES // max(len(bufs), 1)
    written = {}
    for name, b in bufs:
        flat = b.detach().cpu().reshape(-1)
        as64 = not flat.is_floating_point()
        cap = share // (8 if as64 else 4)
        sampled = flat.numel() > cap
        if sampled:
            idx = torch.randperm(flat.numel(), generator=torch.Generator().manual_seed(0))[:cap].sort().values
            flat = flat[idx]
        arr = flat.to(torch.float64 if as64 else torch.float32).numpy()
        np.save(os.path.join(out_dir, name + ".npy"), arr if sampled else arr.reshape(tuple(b.shape)))
        written[name] = {"shape": list(b.shape), "sampled": cap if sampled else None}
    return {"dir": out_dir, "tensors": written}


def collective_probe(dev, world, cfg):
    """The data-path collectives of the DP run timed alone (CUDA events, after the timed region): per iteration one
    reduce-scatter of the bf16 dWq and one all-gather of the bf16 Wq per layer (summed over the block's layers here), and
    per block the all-gather that rebuilds the 128 x 2048 x hidden bf16 block outputs.  Diagnostic only."""
    import torch.distributed as dist

    hidden = MODELS[cfg["model"]][2]["hidden_size"]
    lay = [(n, k) for _, n, k, _ in cfg["linears"] if n % world == 0]
    full = [torch.zeros(n, k, dtype=torch.bfloat16, device=dev) for n, k in lay]
    shard = [torch.zeros(n // world, k, dtype=torch.bfloat16, device=dev) for n, k in lay]
    per = NSAMPLES // world
    loc = torch.zeros(per, SEQLEN, hidden, dtype=torch.bfloat16, device=dev)
    outs = torch.empty(per * world, SEQLEN, hidden, dtype=torch.bfloat16, device=dev)
    nbytes = sum(t.numel() * 2 for t in full)

    def rs():
        for f, s in zip(full, shard):
            dist.reduce_scatter_tensor(s, f)

    def ag():
        for f, s in zip(full, shard):
            dist.all_gather_into_tensor(f, s)

    out = {}
    for name, fn, n, nb in (("reduce_scatter_dwq_all_layers", rs, 10, nbytes), ("all_gather_wq_all_layers", ag, 10, nbytes),
                            ("allgather_outputs", lambda: dist.all_gather_into_tensor(outs, loc), 4, outs.numel() * 2)):
        fn()
        torch.cuda.synchronize()
        dist.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / n
        out[name] = {"ms": round(ms, 3), "bytes": int(nb), "GBps_algo": round(nb / ms / 1e6, 1)}
    return out


def _gemm_mix(dev, cfg):
    from auto_round_b200 import ops

    T = BATCH * SEQLEN
    bufs, flops, nlaunch = {}, 0, 0
    for name, n, k, dx in cfg["linears"]:
        w = (torch.randn(n, k, device=dev) * 0.02).bfloat16()
        bufs[name] = dict(w=w, x=torch.randn(T, k, device=dev).bfloat16(), dy=torch.randn(T, n, device=dev).bfloat16(),
                          gq=torch.empty(n, k, device=dev, dtype=torch.bfloat16), y=torch.empty(T, n, device=dev, dtype=torch.bfloat16),
                          dxo=torch.empty(T, k, device=dev, dtype=torch.bfloat16), dx=dx)
        flops += 2 * T * n * k * (3 if dx else 2)
        nlaunch += 3 if dx else 2

    def one_iter():
        for b in bufs.values():
            ops.gemm(b["x"], b["w"], out=b["y"])                                         # forward  Y = X Wq^T
            if b["dx"]:
                ops.gemm(b["dy"], b["w"], False, True, out=b["dxo"])                     # grad-in  dX = dY Wq
            ops.gemm(b["dy"], b["x"], True, True, out=b["gq"])                           # grad-w   dWq = dY^T X (bf16)
    return one_iter, flops, nlaunch


def gemm_roofline(dev, pk, cfg):
    """Replay the GEMM launch mix of ONE sign-SGD iteration (7 forward, 4 grad-input, 7 grad-weight launches at
    T = 16384 tokens) back to back and time it with CUDA events on the launch stream.  The replay is ~0.2 s of isolated
    launches, so the roofline denominator is the BURST cuBLAS peak; the in-context figure uses the sustained one."""
    one_iter, flops, nlaunch = _gemm_mix(dev, cfg)
    for _ in range(3):
        one_iter()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 10
    s.record()
    for _ in range(reps):
        one_iter()
    e.record()
    torch.cuda.synchronize()
    ms = s.elapsed_time(e) / reps
    achieved = flops / (ms / 1e3) / 1e12
    return {"bound": "tensor", "kernel": "ar::gemm_kernel (wgmma, 128x128x64 tiles, dynamic tile scheduler; fwd / grad-in / grad-w)",
            "achieved": round(achieved, 1), "peak": pk["burst"], "unit": "TFLOP/s", "frac": round(achieved / pk["burst"], 4),
            "peak_source": pk["source"] + " bf16_tflops (burst: the replay is an isolated ~0.2 s run)",
            "flops_per_launch": flops // nlaunch,
            "algorithmic_bytes_per_launch": int(sum(2 * (BATCH * SEQLEN * (n + k) + n * k) * (3 if dx else 2)
                                                    for _, n, k, dx in cfg["linears"]) / nlaunch),
            "avg_launch_ms": round(ms / nlaunch, 4), "launches_per_iteration": nlaunch,
            "how": "%d GEMM launches of one iteration replayed x10 after 3 warm-ups; operands 3.4 GB >> L2" % nlaunch}


def iteration_timeline(dev, pk, cfg, cfg_name, dp=None):
    """Kernel timeline of ONE steady-state iteration inside the CUDA-graph replay of a real block (CUPTI through
    torch.profiler; 14 iterations, the 6th is read): where the iteration's time goes and what the GEMMs achieve IN CONTEXT
    (back to back with everything else, at the sustained clock).  A diagnostic taken under the profiler -- never a value."""
    from torch.profiler import ProfilerActivity, profile

    from auto_round_b200.quantizer import SignRoundQuantizer
    from auto_round_b200.schemes import parse_scheme

    model = build_model(cfg["model"], 1, dev)
    blk = model.model.layers[0].to(dev)
    for p in blk.parameters():
        p.requires_grad_(False)
    hidden = MODELS[cfg["model"]][2]["hidden_size"]
    ns = 16
    torch.manual_seed(0)
    xs = [torch.randn(1, SEQLEN, hidden, device=dev).bfloat16() * 0.05 for _ in range(ns)]
    pos = torch.arange(SEQLEN, device=dev).unsqueeze(0)
    cos, sin = model.model.rotary_emb.to(dev)(xs[0], pos)
    others = {"position_embeddings": [(cos.bfloat16(), sin.bfloat16())], "position_ids": [pos], "attention_mask": None}
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        refs = [blk(x, position_embeddings=others["position_embeddings"][0]) for x in xs]
    refs = [(r[0] if isinstance(r, (tuple, list)) else r).reshape(1, SEQLEN, hidden) for r in refs]
    sk = dict(cfg["scheme"])
    alg_ext = bool(sk.pop("enable_alg_ext", False))
    scheme = parse_scheme(sk.pop("scheme"), sk)
    q = SignRoundQuantizer(scheme, iters=14, batch_size=BATCH, enable_alg_ext=alg_ext, dp=dp)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        q.quantize_block(blk, xs, others, refs, None, None, input_ids=None)
        torch.cuda.synchronize()
    evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    evs.sort(key=lambda e: e.time_range.start)
    idx = [i for i, e in enumerate(evs) if "iter_advance" in e.name]
    if len(idx) < 8:
        return {"error": "timeline too short"}
    it = evs[idx[5] + 1:idx[6] + 1]
    span = (it[-1].time_range.end - it[0].time_range.start) / 1e3
    agg = {}
    for e in it:
        name = e.name
        key = ("nccl" if "nccl" in name.lower() else
               "ar::gemm_kernel" if "gemm_kernel" in name else "cudnn sdpa" if ("sdpa" in name or "cudnn" in name or "fmha" in name)
               else "ar::fq_update_kernel" if "fq_update" in name else "ar::swiglu" if "swiglu" in name
               else "aten elementwise" if "at::native" in name else "ar:: other" if name.startswith(("ar::", "void ar::")) else "other")
        c, t_ = agg.get(key, (0, 0.0))
        agg[key] = (c + 1, t_ + (e.time_range.end - e.time_range.start) / 1e3)
    world = dp.world if dp is not None else 1
    flops_iter = (BATCH * SEQLEN) * (6 * sum(n * k for _, n, k, _ in cfg["linears"]) - 2 * sum(n * k for _, n, k, dx in cfg["linears"] if not dx)) / world
    gemm_ms = agg.get("ar::gemm_kernel", (0, 0.0))[1]
    # time covered by at least one non-NCCL kernel (streams overlap under data parallelism): what is left is exposed communication / idle
    ivs = sorted((e.time_range.start, e.time_range.end) for e in it if "nccl" not in e.name.lower())
    covered, cur_s, cur_e = 0.0, None, None
    for a, b in ivs:
        if cur_e is None or a > cur_e:
            if cur_e is not None:
                covered += cur_e - cur_s
            cur_s, cur_e = a, b
        else:
            cur_e = max(cur_e, b)
    if cur_e is not None:
        covered += cur_e - cur_s
    return {"iteration_ms": round(span, 3), "kernels": len(it), "gemm_ms": round(gemm_ms, 3),
            "compute_covered_ms": round(covered / 1e3, 3), "not_covered_by_compute_ms": round(span - covered / 1e3, 3),
            "gemm_tflops_in_context": round(flops_iter / (gemm_ms / 1e3) / 1e12, 1) if gemm_ms else None,
            "frac_of_sustained_peak": round(flops_iter / (gemm_ms / 1e3) / 1e12 / pk["sustained"], 4) if gemm_ms else None,
            "by_kernel_ms": {k: [c, round(t_, 3)] for k, (c, t_) in sorted(agg.items(), key=lambda kv: -kv[1][1])},
            "how": "torch.profiler (CUPTI) over a 14-iteration quantize_block of one real block, 6th graph-replayed iteration"}


def _block_inputs_for_check(ar, model, dev):
    """Inputs of block 0 exactly as the tuned run cached them (embedding of the synthetic tokens)."""
    hidden, others, ids = ar.cache_block_inputs(model.model.layers[0])
    return hidden, others, ids


def mse_vs_reference(ar, model, orig_block0, cfg, iters, dev, line):
    """BASELINE.json's "per-block MSE vs ref": block 0 (FP inputs = embeddings, so both runs see identical inputs) tuned
    (a) by this engine inside the timed run, (b) by the reference's algorithm -- oracle/signround.py BlockTuner, torch eager
    with autograd on the same GPU, the SAME batch sequence -- and the final output MSE of each against the FP block over
    all 128 samples (valid tokens).  Also yields the reference's eager per-iteration time on this GPU."""
    from oracle import signround as S

    blocks = ar._blocks
    hidden, others, ids = ar.cache_block_inputs(blocks[0])
    blocks[0].to("cpu")
    masks = [(i != -100).to(torch.long).to(dev) for i in ids]
    fp = copy.deepcopy(orig_block0).to(dev)
    okw = {k: v for k, v in others.items()}

    def fwd_all(blk):
        outs = []
        with torch.no_grad():
            for i in range(0, len(hidden), BATCH):
                x, sel = S.select_batch(hidden, okw, list(range(i, min(i + BATCH, len(hidden)))))
                outs.extend(torch.split(S.block_forward(blk, x, sel), 1, dim=0))
        return outs

    def mse(outs, refs):
        tot = torch.zeros((), dtype=torch.float64, device=dev)
        cnt = 0
        for o, r, m in zip(outs, refs, masks):
            d = (o.float() - r.float()) * m.reshape(1, -1, 1)
            tot += (d.double() ** 2).sum()
            cnt += int(m.sum()) * o.shape[-1]
        return float(tot) / cnt

    refs = fwd_all(fp)
    sk = dict(cfg["scheme"])
    alg_ext = bool(sk.pop("enable_alg_ext", False))
    name, bits, g = cfg["spec"]
    osc = S.LayerScheme(bits, g, name != "int_asym", {"int_sym": "int", "int_asym": "int", "mx_fp4": "mx_fp", "nv_fp4": "nv_fp"}[name])
    # RTN (iteration-0 parameters): the floor both tuners start from
    rtn = copy.deepcopy(orig_block0).to(dev)
    from oracle.moe_loop import unfuse_experts_cpu as _unfuse
    _unfuse(rtn)
    wr = S.wrap_block(rtn, lambda n, m: osc)
    S.unwrap_block(rtn, wr, {})
    mse_rtn = mse(fwd_all(rtn), refs)
    del rtn, wr
    # the reference's algorithm, eager on this GPU, same batches as block 0 of the timed run
    oblk = copy.deepcopy(orig_block0).to(dev)
    from oracle.moe_loop import unfuse_experts_cpu
    unfuse_experts_cpu(oblk)                         # MoE: the reference's per-expert loop (no-op for dense blocks)
    batches = ar.block_results[0]["batches"]
    nv = None
    if name == "nv_fp4":
        from oracle import qdq as Q
        nv = {n: Q.nv_global_scale(m.weight.data) for n, m in oblk.named_modules() if type(m) is torch.nn.Linear}
        for grp in (("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj"), ("mlp.gate_proj", "mlp.up_proj")):
            shared = torch.stack([nv[n] for n in grp]).min()
            for n in grp:
                nv[n] = shared
    tuner = S.BlockTuner(oblk, hidden, okw, refs, lambda n, m: osc, iters=iters, batch_size=BATCH, token_masks=masks,
                         sampler=S.ReplaySampler(batches), nv_global_scales=nv, alg_ext=alg_ext)
    times = []
    for it in range(iters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        tuner.step(it)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    ores = tuner.finish()
    mse_ref = mse(fwd_all(oblk), refs)
    ours = ar.block_results[0].get("block_mse")
    steady = sorted(times[3:])
    eager_ms = 1e3 * steady[len(steady) // 2]
    line["gpu_eager_baseline"] = {
        "what": "the reference's algorithm as torch eager + autograd on the same GPU (oracle/signround.py on cuda: ATen fake-quant "
                "graph, cuBLAS GEMMs, SDPA) -- the reference's GPU path without torch.compile",
        "ms_per_iteration": round(eager_ms, 2), "ours_ms_per_iteration": line["ms_per_iteration"],
        "speedup_per_iteration": round(eager_ms / line["ms_per_iteration"], 2),
        "loop_only_extrapolation_s": round(eager_ms * iters * cfg["n_blocks"] / 1e3, 1), "iterations_timed": len(steady)}
    return {"block": 0, "ours": ours, "reference_algorithm": mse_ref, "ratio": (ours / mse_ref) if (ours and mse_ref) else None,
            "rtn": mse_rtn, "ours_init_loss_x_tokens": ar.block_results[0]["init_loss"], "ref_iter0_loss": ores.losses[0],
            "ours_iter0_loss": ar.block_results[0]["losses"][0], "ref_best_iter": ores.best_iter,
            "ours_best_iter": ar.block_results[0]["best_iter"],
            "what": "final output MSE vs the FP block over all 128 samples (valid tokens); same inputs, same batch sequence"}


# ----------------------------------------------------------------------------------------------- reference arm (CPU)
def _cpu_block(cfg):
    import importlib

    import transformers

    cfg_cls, _, kw = MODELS[cfg["model"]]
    c = getattr(transformers, cfg_cls)(num_hidden_layers=1, **kw)
    c._attn_implementation = "sdpa"
    torch.manual_seed(0)
    fam, cls = {"llama3_8b": ("llama", "Llama"), "qwen2_7b": ("qwen2", "Qwen2"), "mixtral_8x7b": ("mixtral", "Mixtral")}[cfg["model"]]
    mod = importlib.import_module(f"transformers.models.{fam}.modeling_{fam}")
    blk = getattr(mod, cls + "DecoderLayer")(c, 0).to(torch.bfloat16).eval()
    from oracle.moe_loop import unfuse_experts_cpu
    unfuse_experts_cpu(blk)                          # MoE: the reference's per-expert linears + loop (no-op otherwise)
    return c, blk, getattr(mod, cls + "RotaryEmbedding")(c)


def cpu_steps(cfg, steps, warmup, budget_s, threads=None):
    """The reference's algorithm on the host cores: oracle/signround.py BlockTuner (CPU restatement pinned bit-exact to the
    reference) on ONE full-shape block.  A whole sign-SGD iteration of that block costs ~40 s of weight-sized work on 128
    cores before a single token is processed, so a STEP is a bounded sample of it: one sign-SGD iteration (forward of the whole
    block, loss, autograd backward, sign-SGD update) in which ONE of the block's linears is tuned (the steps rotate over the
    seven), on T_small = 128 or T_large = 512 tokens (alternating).  Fit: t(layer l, T) = a_l + b T, a_l = weight-sized cost of layer l
    (fake-quant forward/backward + update of its weights), b = per-token cost (GEMMs, attention).  One full iteration is then
    sum_l a_l + b * 16384 tokens and the metric extrapolates it: blocks x iters x that.  Wrappers are built before the timed
    region.  Full-set forwards and pack are not included."""
    from oracle import signround as S

    if threads is None:
        # all the host cores this process may use -- torchrun exports OMP_NUM_THREADS=1 to every rank, which would
        # otherwise turn the reference arm into a single-threaded run at N > 1
        try:
            threads = len(os.sched_getaffinity(0))
        except AttributeError:
            threads = os.cpu_count() or 1
    torch.set_num_threads(max(1, int(threads)))
    cores = torch.get_num_threads()
    c, blk, rot = _cpu_block(cfg)
    name, bits, g = cfg["spec"]
    osc = S.LayerScheme(bits, g, name != "int_asym", {"int_sym": "int", "int_asym": "int", "mx_fp4": "mx_fp", "nv_fp4": "nv_fp"}[name])
    lin_names = [n for n, m in blk.named_modules() if type(m) is torch.nn.Linear]
    weights = {n: blk.get_submodule(n).weight.numel() for n in lin_names}
    order = sorted(lin_names, key=lambda n: weights[n])                      # cheap layers first: the fit needs every layer once
    t_small = 128
    sizes = [t_small, 4 * t_small]
    n_total = steps + warmup
    tuners = {}

    def tuner_for(layer):                                                    # built outside the timed steps
        if layer not in tuners:
            b2 = copy.deepcopy(blk)
            tuners[layer] = S.BlockTuner(b2, [], {"attention_mask": None}, [], lambda n, m, L=layer: osc if n == L else None,
                                         iters=max(cfg["iters"], n_total + 1), batch_size=1, lr=1.0 / cfg["iters"],
                                         sampler=S.ReplaySampler([[0]] * (n_total + 1)))
        return tuners[layer]

    data = {}
    for T in sizes:
        x = torch.randn(1, T, c.hidden_size).to(torch.bfloat16) * 0.02
        pos = torch.arange(T).unsqueeze(0)
        cos, sin = rot(x, pos)
        pe = (cos.to(torch.bfloat16), sin.to(torch.bfloat16))
        with torch.no_grad():
            ref = S.block_forward(blk, x, {"position_embeddings": pe, "position_ids": pos})
        data[T] = (x, ref, {"attention_mask": None, "position_embeddings": [pe], "position_ids": [pos]})
    plan = [(order[i % len(order)], sizes[i % 2]) for i in range(n_total)]     # 7 layers x 2 sizes: all 14 pairs in 14 steps
    for layer in {p[0] for p in plan}:
        tuner_for(layer)
    rows, t_begin = [], time.time()
    for i, (layer, T) in enumerate(plan):
        tn = tuner_for(layer)
        x, ref, others = data[T]
        tn.inputs, tn.fp_outputs, tn.others = [x], [ref], others
        t0 = time.perf_counter()
        tn.step(len(tn.res.losses))
        dt = time.perf_counter() - t0
        if i >= warmup:
            rows.append((layer, T, dt))
        if i >= warmup and (time.time() - t_begin) > budget_s and len(rows) >= 2:
            break
    # least squares for a_l (one per layer seen) and b
    seen = sorted({r[0] for r in rows}, key=lambda n: weights[n])
    import numpy as np
    A = np.zeros((len(rows), len(seen) + 1))
    y = np.zeros(len(rows))
    for j, (layer, T, dt) in enumerate(rows):
        A[j, seen.index(layer)] = 1.0
        A[j, -1] = T
        y[j] = dt
    sol, *_ = np.linalg.lstsq(A, y, rcond=None)
    a = {n: max(float(sol[k]), 0.0) for k, n in enumerate(seen)}
    b = max(float(sol[-1]), 0.0) if len({r[1] for r in rows}) > 1 else 0.0
    # layers never timed (run cut short by the budget): scale the measured weight-sized cost by the weight count
    per_weight = sum(a.values()) / max(sum(weights[n] for n in seen), 1)
    a_total = sum(a.get(n, per_weight * weights[n]) for n in lin_names)
    per_iter = a_total + b * (BATCH * SEQLEN)
    total_s = per_iter * cfg["iters"] * cfg["n_blocks"]
    step_ms = 1e3 * sum(r[2] for r in rows) / max(len(rows), 1)
    return {"value": round(total_s, 1), "unit": "s", "cores": cores, "kind": "port", "ms_per_step": round(step_ms, 1), "steps_timed": len(rows),
            "fit": {"weight_sized_s_per_iter": round(a_total, 3), "s_per_token_per_iter": round(b, 6), "s_per_full_iteration": round(per_iter, 2),
                    "layers_timed": len(seen), "layers": len(lin_names)},
            "sample": "oracle/signround.py BlockTuner (CPU restatement pinned bit-exact to the reference; wrappers built before the timed steps) on "
                      "ONE full-shape block; each step = one sign-SGD iteration with ONE linear tuned (rotating over the block's %d) on %d or %d "
                      "tokens; fit t = a_layer + b T; one iteration = sum a_layer + b x 16384 tokens; x %d iters x %d blocks; EXTRAPOLATED, "
                      "full-set forwards and pack not included; nproc=%d" % (len(lin_names), sizes[0], sizes[1], cfg["iters"], cfg["n_blocks"], cores)}


def cpu_baseline(cfg, steps=8, warmup=1, budget_s=40.0):
    return cpu_steps(cfg, steps, warmup, budget_s)


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    cfg = CONFIGS[args.config]
    iters = args.iters if args.iters else cfg["iters"]
    cb = cpu_steps(cfg, max(args.steps, 2), max(args.warmup, 0), budget_s=180.0)
    line = {"impl": "reference", "metric": cfg["metric"], "value": cb["value"], "unit": "s",
            "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup, "ms_per_step": cb["ms_per_step"],
            "higher_is_better": False, "scaling": "strong", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
            "config": line_config(cfg, iters, args.gpus, args.steps),
            "reference_note": "the reference has no C/C++ on this path; its Python is restated in oracle/ (pinned bit-exact) and timed on the "
                              "host cores; ms_per_step is one bounded sample step, `value` the extrapolation described in cpu_baseline.sample",
            "cpu_baseline": cb,
            "e2e": {"value": cb["value"], "unit": "s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--config", default="llama3_8b_w4a16", choices=sorted(CONFIGS))
    ap.add_argument("--iters", type=int, default=0, help="sign-SGD iterations per block (0: the config's own, metric: 200)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-mse-check", action="store_true")
    ap.add_argument("--cpu-budget", type=float, default=60.0)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the last timed block's packed tensors as DIR/<name>.npy (float32/float64, <= 64 MB)")
    args = ap.parse_args()
    if args.impl == "reference":
        run_reference(args)
    else:
        run_ours(args)


if __name__ == "__main__":
    main()
