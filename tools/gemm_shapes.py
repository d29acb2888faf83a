"""Per-shape timing of the bf16 GEMM launches of one Llama-3-8B calibration iteration (a development probe, not the bench).

    python tools/gemm_shapes.py [--out DIR] [--reps 30] [--baseline-lib PATH/libar_b200.so]

Times each of the 18 `ar_gemm_bf16` launches of one sign-SGD iteration at T = 16384 tokens (the shapes and operand
majorness of bench._gemm_mix: forward, grad-in for o / gate / up / down, grad-w) separately with CUDA events, plus the
grouped MoE launches (GROUP_M forward and grad-in, GROUP_K grad-w) at one Mixtral-8x7B shape.  With --baseline-lib a second
build of the library is loaded through ctypes and timed with alternating runs on the same seeded operands; the outputs of
the two builds are compared bit for bit (mismatch count and maximum bf16 ulp distance per shape).
Prints the card name, power limit and clocks, and writes DIR/gemm_shapes.json.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from auto_round_b200 import _lib, ops  # noqa: E402

T = 16384
LLAMA = [("q", 4096, 4096, False), ("k", 1024, 4096, False), ("v", 1024, 4096, False), ("o", 4096, 4096, True),
         ("gate", 14336, 4096, True), ("up", 14336, 4096, True), ("down", 4096, 14336, True)]
MIXTRAL = dict(hidden=4096, inter=14336, experts=8, topk=2)


def load_lib(path):
    lib = C.CDLL(os.path.abspath(path))
    lib.ar_last_error.restype = C.c_char_p
    for name, args in _lib.SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = C.c_int
    return lib


def card_info():
    info = {"name": torch.cuda.get_device_name(0)}
    q = "power.limit,clocks.max.sm,clocks.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        vals = [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]
        info.update(power_limit_w=vals[0], clocks_max_sm_mhz=vals[1], clocks_sm_mhz_idle=vals[2])
    except Exception as e:  # noqa: BLE001 -- the numbers are still useful without the card's settings
        info["nvidia_smi_error"] = repr(e)
    return info


def _p(t):
    return C.c_void_p(t.data_ptr() if t is not None else 0)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def llama_cases(dev):
    """(name, flops, out tensor, call(lib, out) -> rc) for the 18 launches, in bench._gemm_mix order."""
    cases = []
    for name, n, k, dx in LLAMA:
        w = (torch.randn(n, k, device=dev) * 0.02).bfloat16()
        x = torch.randn(T, k, device=dev).bfloat16()
        dy = torch.randn(T, n, device=dev).bfloat16()

        def call(lib, out, a, b, m_, n_, k_, a_mn, b_mn):
            return lib.ar_gemm_bf16(_p(a), _p(b), _p(out), m_, n_, k_, a_mn, b_mn, a.stride(0), b.stride(0), out.stride(0),
                                    C.c_void_p(0), _stream())

        fl = 2 * T * n * k
        cases.append((f"{name}.fwd T={T} n={n} k={k} (K,K)", fl, torch.empty(T, n, device=dev, dtype=torch.bfloat16),
                      lambda lib, out, a=x, b=w, n=n, k=k: call(lib, out, a, b, T, n, k, 0, 0)))
        if dx:
            cases.append((f"{name}.grad_in T={T} n={k} k={n} (K,MN)", fl, torch.empty(T, k, device=dev, dtype=torch.bfloat16),
                          lambda lib, out, a=dy, b=w, n=n, k=k: call(lib, out, a, b, T, k, n, 0, 1)))
        cases.append((f"{name}.grad_w m={n} n={k} k={T} (MN,MN)", fl, torch.empty(n, k, device=dev, dtype=torch.bfloat16),
                      lambda lib, out, a=dy, b=x, n=n, k=k: call(lib, out, a, b, n, k, T, 1, 1)))
    return cases


def moe_cases(dev):
    h, inter, e, topk = MIXTRAL["hidden"], MIXTRAL["inter"], MIXTRAL["experts"], MIXTRAL["topk"]
    pairs = T * topk
    route = ops.MoeRoute(pairs, e, dev)
    ops.moe_route(route, torch.randint(0, e, (pairs,), device=dev, dtype=torch.int64))
    rows = route.max_rows
    xp = torch.randn(rows, h, device=dev).bfloat16()
    dg = torch.randn(rows, inter, device=dev).bfloat16()
    wg = (torch.randn(e, inter, h, device=dev) * 0.02).bfloat16()           # gate: [E, n=inter, k=h]
    wd = (torch.randn(e, h, inter, device=dev) * 0.02).bfloat16()           # down: [E, n=h, k=inter]
    bf = dict(device=dev, dtype=torch.bfloat16)

    def grouped_m(lib, out, a, b, n, k, b_mn):
        return lib.ar_gemm_bf16_grouped(_p(a), _p(b), _p(out), 1, rows, n, k, 0, int(b_mn), a.stride(0), b.stride(1),
                                        out.stride(0), k if b_mn else n, e, _p(route.mtab), _p(route.num_mt), rows // 256, 0,
                                        _stream())

    def grouped_k(lib, out, dy, x):
        n_out, k_out = dy.shape[1], x.shape[1]
        return lib.ar_gemm_bf16_grouped(_p(dy), _p(x), _p(out), 2, rows, k_out, rows, 1, 1, dy.stride(0), x.stride(0), k_out,
                                        out.shape[1], e, _p(route.ktab), _p(route.num_active), e, n_out, _stream())

    fl = 2 * pairs * h * inter                                              # FLOPs of the routed (unpadded) rows
    return [
        (f"moe.gate.fwd GROUP_M rows={rows} n={inter} k={h}", fl, torch.zeros(rows, inter, **bf),
         lambda lib, out: grouped_m(lib, out, xp, wg, inter, h, False)),
        (f"moe.down.fwd GROUP_M rows={rows} n={h} k={inter}", fl, torch.zeros(rows, h, **bf),
         lambda lib, out: grouped_m(lib, out, dg, wd, h, inter, False)),
        (f"moe.down.grad_in GROUP_M rows={rows} n={inter} k={h} (B MN)", fl, torch.zeros(rows, inter, **bf),
         lambda lib, out: grouped_m(lib, out, xp, wd, inter, h, True)),
        (f"moe.gate.grad_w GROUP_K rows={rows} m={inter} n={h}", fl, torch.zeros(e, inter, h, **bf),
         lambda lib, out: grouped_k(lib, out, dg, xp)),
    ]


def time_one(lib, call, out, s, e):
    s.record()
    rc = call(lib, out)
    e.record()
    if rc != 0:
        raise RuntimeError(f"GEMM launch failed (status {rc}): {lib.ar_last_error().decode(errors='replace')}")
    return s, e


def ulp_stats(a, b):
    def ordered(t):
        u = t.view(torch.int16).to(torch.int32) & 0xFFFF
        return torch.where(u >= 0x8000, 0x8000 - u, u)
    diff = (ordered(a) - ordered(b)).abs()
    return int((diff != 0).sum()), int(diff.max()) if diff.numel() else 0


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", default="gemm_shapes_out", help="output directory (gemm_shapes.json)")
    ap.add_argument("--reps", type=int, default=30, help="timed launches per shape and library (after 3 warm-ups)")
    ap.add_argument("--baseline-lib", default=None, help="a second libar_b200.so to time against and compare with")
    ap.add_argument("--no-moe", action="store_true", help="skip the grouped MoE shapes")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gemm_shapes: no CUDA device")
    dev = "cuda"
    os.makedirs(args.out, exist_ok=True)
    card = card_info()
    print(json.dumps({"card": card}), flush=True)

    libs = {"new": _lib.load()}
    if args.baseline_lib:
        libs["baseline"] = load_lib(args.baseline_lib)
    torch.manual_seed(0)
    cases = llama_cases(dev) + ([] if args.no_moe else moe_cases(dev))
    torch.cuda.synchronize()

    rows, tot = [], {k: 0.0 for k in libs}
    for name, flops, out, call in cases:
        outs = {k: out if k == "new" else out.clone() for k in libs}
        for _ in range(3):
            for k, lib in libs.items():
                time_one(lib, call, outs[k], torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        torch.cuda.synchronize()
        evs = {k: [] for k in libs}
        for _ in range(args.reps):                          # alternate the libraries launch by launch
            for k, lib in libs.items():
                evs[k].append(time_one(lib, call, outs[k], torch.cuda.Event(enable_timing=True),
                                       torch.cuda.Event(enable_timing=True)))
        torch.cuda.synchronize()
        rec = {"shape": name, "flops": flops}
        for k in libs:
            ms = sorted(s.elapsed_time(e) for s, e in evs[k])
            med = statistics.median(ms)
            tot[k] += med if not name.startswith("moe.") else 0.0
            rec[k] = {"ms_median": round(med, 4), "ms_min": round(ms[0], 4), "ms_max": round(ms[-1], 4),
                      "tflops": round(flops / (med / 1e3) / 1e12, 1)}
        if "baseline" in libs:
            bad, ulp = ulp_stats(outs["new"], outs["baseline"])
            rec["identical"] = bool(torch.equal(outs["new"], outs["baseline"]))
            rec["mismatches"], rec["max_ulp"] = bad, ulp
            rec["speedup"] = round(rec["baseline"]["ms_median"] / rec["new"]["ms_median"], 4)
        rows.append(rec)
        print(json.dumps(rec), flush=True)
        del outs

    llama_flops = sum(r["flops"] for r in rows if not r["shape"].startswith("moe."))
    summary = {"card": card, "reps": args.reps, "tokens": T,
               "llama_18_launches": {k: {"ms": round(v, 3), "tflops": round(llama_flops / (v / 1e3) / 1e12, 1)}
                                     for k, v in tot.items()},
               "shapes": rows}
    if "baseline" in libs:
        summary["all_identical"] = all(r["identical"] for r in rows)
        summary["baseline_lib"] = os.path.abspath(args.baseline_lib)
    card_after = card_info()
    summary["clocks_sm_mhz_after"] = card_after.get("clocks_sm_mhz_idle")
    with open(os.path.join(args.out, "gemm_shapes.json"), "w") as f:
        json.dump(summary, f, indent=1)
    print(json.dumps({k: v for k, v in summary.items() if k != "shapes"}), flush=True)


if __name__ == "__main__":
    main()
