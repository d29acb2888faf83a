"""Time of one replayed SignRound iteration for two Llama-3-8B-shaped blocks tuned one at a time (nblocks=1) and together
(nblocks=2).  A development probe, not the bench.

    python tools/nblocks_rate.py [--iters 40] [--skip 5] [--out DIR]

Builds bench.py's Llama-3-8B decoder blocks (random init, seed 0), 8 synthetic calibration samples of 2048 positions
(hidden states drawn from a seeded normal), batch_size 8, so every iteration runs T = 16 384 tokens, W4A16 g128.  Three
tuning calls, each from the same initial weights: block 0 alone, block 1 alone (on block 0's FP outputs), and the group
[0, 1] (a `BlockGroup`, on the FP inputs, against block 1's FP outputs).  Every `CUDAGraph.replay` of the captured iteration
is bracketed by CUDA events; the first `--skip` replays are warm-up and the median of the rest is the time per iteration.
Also reports the peak allocated memory of each call.  Prints one JSON line with the card
name and power limit read in the same run and writes it to DIR/nblocks_rate.json.  Needs a CUDA device.
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys

ap = argparse.ArgumentParser()
ap.add_argument("--iters", type=int, default=40)
ap.add_argument("--skip", type=int, default=5)
ap.add_argument("--out", default="nblocks_rate_out")
args = ap.parse_args()
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import bench  # noqa: E402
from auto_round_b200.autoround import BlockGroup  # noqa: E402
from auto_round_b200.quantizer import SignRoundQuantizer  # noqa: E402
from auto_round_b200.schemes import parse_scheme  # noqa: E402

SAMPLES, SEQ, HIDDEN, BATCH = 8, 2048, 4096, 8


def card_info():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        vals = [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]
        info.update(power_limit_w=vals[0], clocks_max_sm_mhz=vals[1])
    except Exception as e:  # noqa: BLE001 -- the times are still useful without the card's settings
        info["nvidia_smi_error"] = repr(e)
    return info


class ReplayTimer:
    """Brackets every CUDAGraph.replay with CUDA events while active."""

    def __init__(self):
        self.events = []

    def __enter__(self):
        self.orig = torch.cuda.CUDAGraph.replay
        timer = self

        def replay(graph):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            timer.orig(graph)
            b.record()
            timer.events.append((a, b))

        torch.cuda.CUDAGraph.replay = replay
        return self

    def __exit__(self, *exc):
        torch.cuda.CUDAGraph.replay = self.orig
        return False

    def times_ms(self):
        torch.cuda.synchronize()
        return [a.elapsed_time(b) for a, b in self.events]


def fresh_blocks(dev):
    """Both decoder blocks with their initial weights (tuning writes the fake-quant weights into the layers)."""
    model = bench.build_llama(2, dev)
    blocks = [model.model.layers[j].to(dev) for j in range(2)]
    for blk in blocks:
        for p in blk.parameters():
            p.requires_grad_(False)
    return model, blocks


def main():
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    model, blocks = fresh_blocks(dev)
    torch.manual_seed(0)
    xs = [torch.randn(1, SEQ, HIDDEN, device=dev).bfloat16() * 0.05 for _ in range(SAMPLES)]
    pos = torch.arange(SEQ, device=dev).unsqueeze(0)
    cos, sin = model.model.rotary_emb.to(dev)(xs[0], pos)
    pe = (cos.bfloat16(), sin.bfloat16())
    others = {"position_embeddings": [pe], "position_ids": [pos], "attention_mask": None}

    def fp_forward(blk, inputs):
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            outs = [blk(x, position_embeddings=pe) for x in inputs]
        return [(o[0] if isinstance(o, (tuple, list)) else o).reshape(1, SEQ, HIDDEN).bfloat16() for o in outs]

    h1 = fp_forward(blocks[0], xs)
    h2 = fp_forward(blocks[1], h1)
    del model, blocks
    cases = {"block0": (lambda b: b[0], xs, h1), "block1": (lambda b: b[1], h1, h2),
             "group01": (lambda b: BlockGroup(b, ["model.layers.0", "model.layers.1"]), xs, h2)}
    out = {}
    for name, (make, inputs, refs) in cases.items():
        _, blocks = fresh_blocks(dev)
        unit = make(blocks)
        random.seed(0)
        q = SignRoundQuantizer(parse_scheme("W4A16"), iters=args.iters, batch_size=BATCH)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        with ReplayTimer() as t:
            q.quantize_block(unit, inputs, others, refs, None, None, input_ids=None)
        times = t.times_ms()[args.skip:]
        res = q.last_result
        del unit, blocks
        if not res.used_cuda_graph or len(times) < 30:
            raise RuntimeError(f"{name}: {len(times)} timed replays (graph={res.used_cuda_graph}); need a captured graph "
                               "and >= 30 replays after warm-up")
        out[name] = {"ms_per_iter_median": statistics.median(times), "ms_min": min(times), "ms_max": max(times),
                     "replays_timed": len(times), "peak_allocated_gib": torch.cuda.max_memory_allocated(dev) / 2 ** 30,
                     "layers": len(res.quantized_layers), "loss_iter0": res.losses[0], "best_loss": res.best_loss}
    out["sum_of_blocks_ms"] = out["block0"]["ms_per_iter_median"] + out["block1"]["ms_per_iter_median"]
    out["group_minus_sum_ms"] = out["group01"]["ms_per_iter_median"] - out["sum_of_blocks_ms"]
    rec = {"card": card_info(), "shape": "llama3_8b block (4096 hidden, 14336 ffn, 32/8 heads)", "samples": SAMPLES,
           "seq": SEQ, "batch_size": BATCH, "tokens_per_iter": BATCH * SEQ, "scheme": "W4A16 g128", "iters": args.iters,
           "skip": args.skip, "results": out}
    print(json.dumps(rec), flush=True)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "nblocks_rate.json"), "w") as f:
        json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
