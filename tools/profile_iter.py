"""In-context kernel timeline of the sign-SGD iteration (torch.profiler / CUPTI) on one Llama-3-8B block.
Unlike the ncu launch list (kernels serialised, cold caches) this shows durations while the GPU is busy back to back,
plus the idle gaps.  Writes gpurun_out/iter_timeline.txt.  Development probe, not the bench."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from auto_round_b200.quantizer import SignRoundQuantizer  # noqa: E402
from auto_round_b200.schemes import parse_scheme  # noqa: E402

dev = torch.device("cuda", 0)
graph = "--graph" in sys.argv
model = bench.build_llama(1, dev)
blk = model.model.layers[0].to(dev)
for p in blk.parameters():
    p.requires_grad_(False)
ns, S, H = 16, bench.SEQLEN, 4096
torch.manual_seed(0)
xs = [torch.randn(1, S, H, device=dev).bfloat16() * 0.05 for _ in range(ns)]
pos = torch.arange(S, device=dev).unsqueeze(0)
cos, sin = model.model.rotary_emb.to(dev)(xs[0], pos)
others = {"position_embeddings": [(cos.bfloat16(), sin.bfloat16())], "position_ids": [pos], "attention_mask": None}
with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
    refs = [blk(x, position_embeddings=others["position_embeddings"][0])[0:1].reshape(1, S, H) if False else
            blk(x, position_embeddings=others["position_embeddings"][0]) for x in xs]
refs = [(r[0] if isinstance(r, (tuple, list)) else r).reshape(1, S, H) for r in refs]
iters = 14
q = SignRoundQuantizer(parse_scheme("W4A16"), iters=iters, batch_size=8, use_cuda_graph=graph)
from torch.profiler import ProfilerActivity, profile

torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
    q.quantize_block(blk, xs, others, refs, None, None, input_ids=None)
    torch.cuda.synchronize()
ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
ev.sort(key=lambda e: e.time_range.start)
# isolate steady-state iterations: between consecutive iter_advance kernels
idx = [i for i, e in enumerate(ev) if "iter_advance" in e.name]
lines = []
if len(idx) >= 8:
    a, b = idx[5], idx[6]
    it = ev[a + 1:b + 1]
    span = it[-1].time_range.end - it[0].time_range.start
    busy = sum(e.time_range.end - e.time_range.start for e in it)
    lines.append(f"mode={'graph' if graph else 'eager'} one iteration: {len(it)} kernels, span {span/1e3:.2f} ms, busy {busy/1e3:.2f} ms, idle {(span-busy)/1e3:.2f} ms")
    agg = {}
    for e in it:
        k = e.name[:90]
        c, t = agg.get(k, (0, 0.0))
        agg[k] = (c + 1, t + (e.time_range.end - e.time_range.start))
    for k, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:30]:
        lines.append(f"{t/1e3:8.3f} ms  n={c:2d}  {k}")
    gaps = sorted(((it[i + 1].time_range.start - it[i].time_range.end, it[i].name[:50], it[i + 1].name[:50]) for i in range(len(it) - 1)), reverse=True)[:8]
    lines.append("largest gaps (us): " + "; ".join(f"{g:.0f} after {a_}" for g, a_, _ in gaps))
os.makedirs("gpurun_out", exist_ok=True)
open("gpurun_out/iter_timeline%s.txt" % ("_graph" if graph else ""), "w").write("\n".join(lines) + "\n")
print("\n".join(lines))
