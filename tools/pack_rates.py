"""Achieved HBM rate of the checkpoint pack kernels at the Llama-3-8B layer shapes (a development probe, not the bench).

    python tools/pack_rates.py [--out DIR] [--reps 30]

Times `ar_pack_int` (W4 g128, zp-1 layout), `ar_pack_awq` (W4 g128 asymmetric), `ar_pack_fp4_nv` and `ar_pack_fp4_mx` on
each of the seven linears of one decoder layer with CUDA events: median of `--reps` (>= 30) launches after 5 warm-up
launches.  The rate is the bytes the algorithm has to move, computed from the shapes (weight read in bf16, scales and
zero-points read, packed words and transposed scales written), over that time; it is not a share of peak.  Prints the card
name and power limit read in the same run and writes DIR/pack_rates.json.  Needs a CUDA device: there is no CPU path.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from auto_round_b200 import ops  # noqa: E402

LLAMA = [("q", 4096, 4096), ("k", 1024, 4096), ("v", 1024, 4096), ("o", 4096, 4096), ("gate", 14336, 4096),
         ("up", 14336, 4096), ("down", 4096, 14336)]


def card_info():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        vals = [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]
        info.update(power_limit_w=vals[0], clocks_max_sm_mhz=vals[1])
    except Exception as e:  # noqa: BLE001 -- the numbers are still useful without the card's settings
        info["nvidia_smi_error"] = repr(e)
    return info


def cases(n, k, dev):
    """(kernel, algorithmic bytes, call) per pack kernel for one [n, k] layer; inputs come from the fake-quant kernels."""
    w = (torch.randn(n, k, device=dev) * 0.02).bfloat16()
    out = []
    g = 128
    for name, asym in (("int_sym", False), ("int_asym", True)):
        spec = ops.make_spec(name, 4, g, n, k)
        wq, sc, zp = ops.qdq_fwd(spec, w, want_scale=True)
        sc = sc.reshape(n, -1).contiguous()
        groups = n * (k // g)
        packed = n * k // 2 + groups // 2 + groups * 2                     # words + zero words + fp16 scales written
        if asym:
            zp = zp.reshape(n, -1).contiguous()
            out.append(("ar_pack_awq", n * k * 2 + groups * 6 + packed, lambda wq=wq, sc=sc, zp=zp: ops.pack_awq(wq, sc, zp, g)))
        else:
            out.append(("ar_pack_int", n * k * 2 + groups * 2 + packed + k * 4,
                        lambda wq=wq, sc=sc: ops.pack_int(wq, sc, None, 4, g, True, zp_const=8)))
    spec = ops.make_spec("nv_fp4", 4, 16, n, k)
    gs = ops.nv_global_scale(w)
    wq, sc, _ = ops.qdq_fwd(spec, w, gscale=gs, want_scale=True)
    sc = sc.to(torch.float32).reshape(n, -1).contiguous()
    out.append(("ar_pack_fp4_nv", n * k * 2 + (n * k // 16) * 4 + n * k // 2 + n * k // 16,
                lambda wq=wq, sc=sc, gs=gs: ops.pack_fp4_nv(wq, sc, gs)))
    spec = ops.make_spec("mx_fp4", 4, 32, n, k)
    wq, e, _ = ops.qdq_fwd(spec, w, want_scale=True)
    e = e.to(torch.bfloat16).reshape(n, -1).contiguous()
    out.append(("ar_pack_fp4_mx", n * k * 2 + (n * k // 32) * 2 + n * k // 2 + n * k // 32,
                lambda wq=wq, e=e: ops.pack_fp4_mx(wq, e)))
    return out


def time_ms(call, reps):
    for _ in range(5):
        call()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times), min(times), max(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="pack_rates_out")
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pack_rates: a CUDA device is required (the pack kernels have no CPU path)")
    if args.reps < 30:
        raise SystemExit("pack_rates: --reps must be at least 30")
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    result = {"card": card_info(), "reps": args.reps, "rows": []}
    print(json.dumps(result["card"]))
    for layer, n, k in LLAMA:
        for kernel, nbytes, call in cases(n, k, dev):
            med, lo, hi = time_ms(call, args.reps)
            row = {"layer": layer, "n": n, "k": k, "kernel": kernel, "bytes": nbytes, "median_ms": med, "min_ms": lo, "max_ms": hi,
                   "achieved_GBps": nbytes / (med * 1e-3) / 1e9}
            result["rows"].append(row)
            print(f"{kernel:16s} {layer:5s} n={n:5d} k={k:5d}  {med * 1e3:8.1f} us (min {lo * 1e3:.1f}, max {hi * 1e3:.1f})  "
                  f"{row['achieved_GBps']:7.0f} GB/s")
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "pack_rates.json"), "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
