"""Time of one lm_head tuning iteration (`quant_lm_head=True`) at the Llama-3-8B shape (a development probe, not the bench).

    python tools/lm_head_rate.py [--root DIR] [--iters 10] [--reps 3] [--out DIR]

Runs `SignRoundQuantizer.quantize_layer` on a seeded 128256 x 4096 bf16 lm_head with 8 calibration samples of 2048 tokens,
batch_size 8, W4A16 g128.  Each repetition makes two calls, with 2 and with 2 + `--iters` iterations, timed on the host
around a device synchronise; their difference over `--iters` is the time of one iteration (8 micro-batches: target,
forward and grad-w GEMMs each, then one fused update), free of the per-call set-up.  A first 2-iteration call warms up.
Prints one JSON line with the card name and power limit read in the same run, the per-iteration times and the loss of
every iteration of the last long call, and writes it to DIR/lm_head_rate.json.

`--root` imports `auto_round_b200` from another checkout (with its library built), so two versions can be compared by
running this script alternately on each.  Needs a CUDA device: there is no CPU path.
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import time

ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--iters", type=int, default=10)
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--out", default="lm_head_rate_out")
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))

import torch  # noqa: E402

from auto_round_b200.quantizer import SignRoundQuantizer  # noqa: E402
from auto_round_b200.schemes import parse_scheme  # noqa: E402

N, K, SAMPLES, SEQ, BATCH, WARM = 128256, 4096, 8, 2048, 8, 2


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


def main():
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    w0 = (torch.randn(N, K, device=dev) * 0.02).bfloat16()
    fp = [torch.randn(1, SEQ, K, device=dev).bfloat16() for _ in range(SAMPLES)]
    qin = [(x.float() + 0.01 * torch.randn_like(x, dtype=torch.float32)).bfloat16() for x in fp]   # the quantised chain
    lin = torch.nn.Linear(K, N, bias=False, device=dev, dtype=torch.bfloat16)
    lin.weight.requires_grad_(False)

    def call(iters):
        lin.weight.copy_(w0)                        # quantize_layer writes the fake-quant weight back into the layer
        random.seed(0)                              # the sampler draws from python's global `random`
        q = SignRoundQuantizer(parse_scheme("W4A16"), iters=iters, batch_size=BATCH)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        q.quantize_layer(lin, fp, qin)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, q.last_result.losses

    call(WARM)
    per_iter, losses = [], None
    for _ in range(args.reps):
        t_short, _ = call(WARM)
        t_long, losses = call(WARM + args.iters)
        per_iter.append((t_long - t_short) / args.iters * 1e3)
    rec = {"card": card_info(), "root": os.path.abspath(args.root), "shape": [N, K], "samples": SAMPLES, "seq": SEQ,
           "batch_size": BATCH, "scheme": "W4A16 g128", "iters_timed": args.iters, "ms_per_iter": per_iter,
           "ms_per_iter_median": statistics.median(per_iter), "losses": losses}
    print(json.dumps(rec), flush=True)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "lm_head_rate.json"), "w") as f:
        json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
