"""One-shot GPU diagnostics (run on a GPU machine): correctness of every GEMM variant + timing vs cuBLAS.
Writes gpurun_out/diag.json.  Not a test and not the bench: a development probe."""
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from auto_round_b200 import ops  # noqa: E402

out = {"device": torch.cuda.get_device_name(0), "gemm": [], "timing": []}
dev = "cuda"


def ref(a, b, a_mn, b_mn):
    A = a.float().t() if a_mn else a.float()
    B = b.float().t() if b_mn else b.float()
    return A @ B.t()


for (m, n, k) in [(128, 256, 64), (128, 256, 256), (256, 512, 512), (200, 328, 136), (1024, 1536, 2048)]:
    for a_mn in (False, True):
        for b_mn in (False, True):
            torch.manual_seed(1)
            a = torch.randn((k, m) if a_mn else (m, k), device=dev).bfloat16()
            b = torch.randn((k, n) if b_mn else (n, k), device=dev).bfloat16()
            rec = {"m": m, "n": n, "k": k, "a_mn": a_mn, "b_mn": b_mn}
            try:
                d = ops.gemm(a, b, a_mn, b_mn)
                torch.cuda.synchronize()
                r = ref(a, b, a_mn, b_mn)
                rec["err_over_rms"] = float((d.float() - r).abs().max() / r.pow(2).mean().sqrt())
                rec["nan"] = bool(torch.isnan(d.float()).any())
            except Exception as e:  # noqa: BLE001
                rec["error"] = repr(e)
            out["gemm"].append(rec)
            print(rec, flush=True)


def timeit(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


T = 16384
for (n, k, tag) in [(4096, 4096, "q_proj"), (14336, 4096, "gate_proj"), (4096, 14336, "down_proj")]:
    x = torch.randn(T, k, device=dev).bfloat16()
    w = (torch.randn(n, k, device=dev) * 0.02).bfloat16()
    dy = torch.randn(T, n, device=dev).bfloat16()
    fl = 2.0 * T * n * k
    try:
        t_fwd = timeit(lambda: ops.gemm(x, w))
        t_dx = timeit(lambda: ops.gemm(dy, w, False, True))
        t_dw_plain = timeit(lambda: ops.gemm(dy, x, True, True))
        t_cublas = timeit(lambda: torch.matmul(x, w.t()))
        t_cublas_dw = timeit(lambda: torch.matmul(dy.t(), x))
        rec = {"layer": tag, "fwd_ms": t_fwd, "dx_ms": t_dx, "dw_ms": t_dw_plain, "cublas_fwd_ms": t_cublas,
               "cublas_dw_ms": t_cublas_dw, "fwd_tflops": fl / t_fwd / 1e9, "dx_tflops": fl / t_dx / 1e9,
               "dw_tflops": fl / t_dw_plain / 1e9, "cublas_tflops": fl / t_cublas / 1e9}
        spec = ops.make_spec("int_sym", 4, 128, n, k)
        v = torch.zeros(n, k, device=dev)
        mn = torch.ones(spec.groups, device=dev)
        mx = torch.ones(spec.groups, device=dev)
        wmin, wmax = ops.group_minmax(spec, w)
        wq = torch.empty_like(w)
        t_qdq = timeit(lambda: ops.qdq_fwd(spec, w, v, mn, mx, wmin, wmax, None, out_wq=wq))
        rec.update(qdq_ms=t_qdq, qdq_gbs=(n * k * 8) / t_qdq / 1e6)
    except Exception as e:  # noqa: BLE001
        rec = {"layer": tag, "error": repr(e)}
    out["timing"].append(rec)
    print(rec, flush=True)

os.makedirs("gpurun_out", exist_ok=True)
json.dump(out, open("gpurun_out/diag.json", "w"), indent=1)
