"""Differential fuzz of the oracle against the UNMODIFIED reference (intel/auto-round v0.15.0).

TEST INFRASTRUCTURE ONLY.  The committed fixtures under tests/golden/ pin the oracle on a fixed set of inputs; this script
draws seeded random weights / rounding offsets / scales / importance vectors for many seeds and shapes and demands bit-exact
agreement of values AND autograd gradients between `oracle/qdq.py`, `oracle/pack.py` and the reference's registered
functions and packers.  With the reference importable (`--record`, see oracle/ref_shim.py) it runs both sides and stores
what the reference computed under tests/golden/: a canonical SHA-256 of every reference tensor (the comparison is bit-exact,
so a digest decides it as well as the tensor would) and, for the loop replays, the recorded runs themselves.  Without
`--record` the oracle side is checked against those stored results; tests/test_oracle_vs_reference_live.py runs it:

    python -m oracle.diff_fuzz --seeds 6 [--record]     -> prints one JSON line {"cases": N, "failures": [...]}
    python -m oracle.diff_fuzz --loops [--record]
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import sys

import torch

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
DIGESTS = os.path.join(GOLDEN, "diff_fuzz_reference.json")
LOOPS = os.path.join(GOLDEN, "diff_fuzz_loops.pt")


def _digest(t):
    """Canonical digest of a tensor's VALUES: float64, flat, -0.0 folded into +0.0, one NaN pattern -- equal digests iff
    the values are equal element for element (NaN matching NaN), whatever the dtype or shape."""
    if t is None:
        return None
    t = torch.as_tensor(t).detach().cpu()
    t = t.view(torch.uint8) if t.dtype == torch.float8_e4m3fn else t
    x = t.reshape(-1).to(torch.float64) + 0.0
    x[torch.isnan(x)] = float("nan")
    return hashlib.sha256(x.numpy().tobytes()).hexdigest()[:32]


def _weights(n, k, gen, dtype=torch.bfloat16):
    w = (torch.randn(n, k, generator=gen) * (0.02 + 0.1 * float(torch.rand(1, generator=gen)))).to(dtype)
    if n > 2:
        w[0, : min(16, k)] = 0
        w[1, 0], w[1, 1] = 0.25, -0.25
        w[2, min(7, k - 1)] = 6.0
    return w


def run(seeds: int, record: bool = False):
    """record=True: run the reference live, compare, and return its digests; otherwise compare with the stored ones."""
    from oracle import qdq as Q

    if record:
        from oracle.ref_shim import import_reference

        import_reference()
        from auto_round.data_type import QUANT_FUNC_WITH_DTYPE as REF
        ref_digests = {}
    else:
        REF = None
        ref_digests = json.load(open(DIGESTS))

    def check(key, ref_value, got):
        """ref_value: a zero-argument callable computing the reference's tensor (only called when recording)."""
        if record:
            ref_digests[key] = _digest(ref_value())
        return key in ref_digests and ref_digests[key] == _digest(got)

    failures, cases = [], 0
    shapes = [(8, 128), (5, 200), (16, 256), (3, 64)]
    for seed in range(seeds):
        gen = torch.Generator().manual_seed(1000 + seed)
        n, k = shapes[seed % len(shapes)]
        for name, bits, g in (("int_sym", 4, 128), ("int_sym", 2, 32), ("int_sym", 3, 64), ("int_sym", 8, 32), ("int_asym", 2, 32),
                              ("int_asym", 4, 64), ("mx_fp4", 4, 32), ("nv_fp4", 4, 16)):
            w = _weights(n, k, gen)
            grp, _, _ = Q.to_groups(w, g)
            G = grp.shape[0]
            v0 = (torch.rand(grp.shape, generator=gen) - 0.5).float()
            mn0 = (0.4 + 0.6 * torch.rand(G, generator=gen)).float()
            mx0 = (0.4 + 0.6 * torch.rand(G, generator=gen)).float()
            gq = torch.randn(w.shape, generator=gen).to(w.dtype)
            outs = []
            for which in (("ref", "oracle") if record else ("oracle",)):
                v, mn, mx = (t.clone().requires_grad_(True) for t in (v0, mn0, mx0))
                if name.startswith("int"):
                    wmin = torch.clamp(grp.min(1)[0], max=0)
                    wmax = torch.clamp(grp.max(1)[0], min=0)
                    if which == "ref":
                        q, s, z = REF[name](w, bits=bits, group_size=g, v=v, min_scale=mn, max_scale=mx, scale_dtype=torch.float16,
                                            tensor_min=wmin, tensor_max=wmax, q_scale_thresh=1e-5)
                    else:
                        fn = Q.int_sym if name == "int_sym" else Q.int_asym
                        q, s, z = fn(w, bits, g, v, mn, mx, wmin, wmax, torch.float16, 1e-5)
                elif name == "mx_fp4":
                    if which == "ref":
                        q, s, z = REF["mx_fp4"](w, bits=4, group_size=32, v=v, max_scale=mx, data_type="mx_fp")
                    else:
                        q, s, z = Q.mx_fp4(w, 32, v, mx)
                else:
                    gs = Q.nv_global_scale(w) * 0.95
                    if which == "ref":
                        q, s, z = REF["nv_fp4"](w, bits=4, group_size=16, v=v, global_scale=gs, max_scale=mx)
                    else:
                        q, s, z = Q.nv_fp4(w, 16, v, gs, mx)
                (q.float() * gq.float()).sum().backward()
                outs.append((q, s, z if isinstance(z, torch.Tensor) else None, v.grad, mx.grad, mn.grad))
            cases += 1
            labels = ("qdq", "scale", "zp", "dV", "d max_scale", "d min_scale")
            for i, (lab, b) in enumerate(zip(labels, outs[-1])):
                if not check(f"fq/{seed}/{name}/w{bits}/g{g}/{lab}", lambda: outs[0][i], b):
                    failures.append(f"seed {seed} {name} w{bits} g{g} [{n}x{k}]: {lab} differs")
        # RTN variants and the optimized-RTN searches
        for name, bits, g in (("rtn_int_sym", 4, 128), ("opt_rtn_int_sym", 4, 32), ("opt_rtn_int_sym", 2, 32), ("opt_rtn_int_sym", 3, 128),
                              ("opt_rtn_nv_fp4", 4, 16), ("opt_rtn_mx_fp4", 4, 32)):
            w = _weights(n, k, gen)
            im = (torch.rand(k, generator=gen) ** 2 * 30 + 0.01).float() if seed % 3 else None
            if im is not None and seed % 5 == 0:
                im[: max(1, k // 10)] = 0
            kw = dict(bits=bits, group_size=g)
            a = None
            if name == "rtn_int_sym":
                if record:
                    a = REF[name](w.clone(), **kw)
                b = Q.rtn_int_sym(w.clone(), bits, g)
            elif name == "opt_rtn_int_sym":
                if record:
                    a = REF[name](w.clone(), imatrix=None if im is None else im.clone(), **kw)
                b = Q.opt_rtn_int_sym(w.clone(), bits, g, im)
            elif name == "opt_rtn_nv_fp4":
                gs = Q.nv_global_scale(w) * 0.9
                if record:
                    a = REF[name](w.clone(), global_scale=gs, **({} if im is None else {"imatrix": im.clone()}), **kw)
                b = Q.opt_rtn_nv_fp4(w.clone(), 16, gs, 1.0, im)[:3]
            else:
                if record:
                    a = REF[name](w.clone(), data_type="mx_fp4", imatrix=None if im is None else im.clone(), **kw)
                b = Q.opt_rtn_mx_fp4(w.clone(), 32, im)[:3]
            cases += 1
            key = f"rtn/{seed}/{name}/w{bits}/g{g}"
            if not check(key + "/qdq", lambda: a[0], b[0]):
                failures.append(f"seed {seed} {name} w{bits} g{g} [{n}x{k}] imatrix={'yes' if im is not None else 'no'}: qdq differs")
            if not check(key + "/scale", lambda: a[1], b[1]):
                failures.append(f"seed {seed} {name} w{bits} g{g} [{n}x{k}]: scale differs")
    # packers: reference QuantLinear.pack vs oracle/pack.py on fresh qdq weights (every bit of every buffer)
    import torch.nn as nn

    from oracle import pack as P

    if record:
        from auto_round.export.export_to_autoround.qlinear_fp import QuantLinear as FpQL
        from auto_round_extension.torch.qlinear_torch import QuantLinear as PlainQL
        from auto_round_extension.torch.qlinear_torch_zp import QuantLinear as ZpQL
    else:
        class _NoRef:                       # replay: the reference's packers are not called (check() never reads them)
            def __init__(self, *a, **k):
                self.device = None

            def pack(self, *a, **k):
                return None
        FpQL = PlainQL = ZpQL = _NoRef

    def lin(wq):
        m = nn.Linear(wq.shape[1], wq.shape[0], bias=False)
        m.weight.data = wq.clone()
        return m

    def cmp(tag, got: dict, ref_obj, keys):
        for key in keys:
            if not check(f"pack/{tag}/{key}", lambda: getattr(ref_obj, key), got[key]):
                failures.append(f"{tag}: packed buffer {key} differs")

    for seed in range(seeds):
        gen = torch.Generator().manual_seed(5000 + seed)
        for bits, g in ((4, 128), (2, 32), (8, 64), (3, 128)):
            n, k = 32 * (1 + seed % 2), 256
            w = _weights(n, k, gen)
            v = torch.rand(n * k // g, g, generator=gen) - 0.5
            wq, sc, zp = Q.int_sym(w, bits, g, v)
            ql = ZpQL(bits, g, k, n, False, g_idx=True)
            ql.pack(lin(wq.detach()), sc.reshape(n, -1).detach().clone(), int(zp), None, "cpu")
            cmp(f"seed {seed} pack int_sym w{bits} g{g}", P.pack_int(wq.detach(), sc.reshape(n, -1).detach(), int(zp), bits, g, True), ql,
                ("qweight", "qzeros", "scales"))
            cases += 1
            if bits != 4:
                wq, sc, zp = Q.int_asym(w, bits, g, v)
                ql = PlainQL(bits, g, k, n, False)
                ql.device = "cpu"
                ql.pack(lin(wq.detach()), sc.reshape(n, -1).detach().clone(), zp.reshape(n, -1).detach().clone(), None, "cpu")
                cmp(f"seed {seed} pack int_asym w{bits} g{g}",
                    P.pack_int(wq.detach(), sc.reshape(n, -1).detach(), zp.reshape(n, -1).detach(), bits, g, False), ql,
                    ("qweight", "qzeros", "scales"))
                cases += 1
        n, k = 32, 128
        w = _weights(n, k, gen)
        gs = Q.nv_global_scale(w)
        wq, sc, _ = Q.nv_fp4(w, 16, torch.rand(n * k // 16, 16, generator=gen) - 0.5, gs)
        ql = FpQL(4, 16, k, n, False, data_type="nv_fp", act_bits=16)
        ql.pack(lin(wq), sc.reshape(n, -1), global_scale=gs, device="cpu")
        cmp(f"seed {seed} pack nv_fp4", P.pack_nvfp4(wq, sc.reshape(n, -1), gs), ql, ("weight_packed", "weight_scale"))
        wq, e, _ = Q.mx_fp4(w, 32, torch.rand(n * k // 32, 32, generator=gen) - 0.5)
        ql = FpQL(4, 32, k, n, False, data_type="mx_fp", act_bits=16)
        ql.pack(lin(wq), e.reshape(n, -1), device="cpu")
        cmp(f"seed {seed} pack mx_fp4", P.pack_mxfp4(wq, e.reshape(n, -1)), ql, ("weight_packed", "weight_scale"))
        cases += 2
    if record:
        with open(DIGESTS, "w") as f:
            json.dump(ref_digests, f, indent=0, sort_keys=True)
    return {"cases": cases, "failures": failures}


def run_loops(record: bool = False):
    """Whole tuning runs with NON-default loop options (the committed block fixtures all use the defaults): the reference's
    AutoRound on the tiny Llama, recorded by oracle/gen_golden.gen_block (record=True: live, and stored under tests/golden/),
    replayed by oracle/signround.tune_block."""
    from oracle import signround as S

    if record:
        from oracle.ref_shim import import_reference

        import_reference()
        import oracle.gen_golden as G
        recs = {}
    else:
        recs = torch.load(LOOPS, weights_only=False)

    configs = [
        ("minmax_off", dict(scheme="W4A16", group_size=32, enable_minmax_tuning=False), S.LayerScheme(4, 32, True, "int"),
         dict(enable_minmax_tuning=False)),
        ("last_iter", dict(scheme="W4A16", group_size=32, not_use_best_mse=True), S.LayerScheme(4, 32, True, "int"),
         dict(not_use_best_mse=True)),
        ("custom_lr", dict(scheme="W2A16", group_size=32, sym=False, lr=0.01, minmax_lr=0.02), S.LayerScheme(2, 32, False, "int"),
         dict(lr=0.01, minmax_lr=0.02)),
        ("nvfp4_bs2", dict(scheme="NVFP4", act_bits=16, act_data_type="float"), S.LayerScheme(4, 16, True, "nv_fp"), dict()),
        # gradient accumulation: 2 micro-batches of 2 per iteration, MSELoss('sum'), one step (quantizer.py:436-452)
        ("accum2_bs2", dict(scheme="W4A16", group_size=32, gradient_accumulate_steps=2), S.LayerScheme(4, 32, True, "int"),
         dict(gradient_accumulate_steps=2)),
    ]
    failures, cases = [], 0
    for tag, kw, sc, okw in configs:
        bs = 2 if tag.endswith("bs2") else 4
        if record:
            recs[tag] = _compact(G.gen_block(tag, kw, iters=5, batch_size=bs, save=False))
        rec = recs[tag]
        for bi, b in enumerate(rec["blocks"]):
            from oracle.tests_support import tiny_block
            blk = tiny_block(b["block_state"])
            masks = [(ids != -100).to(torch.long) for ids in b["input_ids"]]
            res = S.tune_block(blk, b["inputs"], b["others"], b["fp_outputs"], lambda n, m: sc, iters=rec["iters"], batch_size=bs,
                               token_masks=masks, nv_global_scales=b["nv_gs"] or None, sampler=S.ReplaySampler(b["batches"]), **okw)
            nvalid = [sum(int(masks[i].sum()) for i in batch) for batch in b["batches"]]
            got = [l * n for l, n in zip(res.losses, nvalid)]
            if okw.get("gradient_accumulate_steps", 1) != 1:       # the reference logs one (sum-reduced) loss per micro-batch
                got = list(res.micro_losses)
            cases += 1
            if any(abs(a - e) > 1e-6 * abs(e) for a, e in zip(got, b["losses"])) or len(got) != len(b["losses"]):
                failures.append(f"loop {tag} block {bi}: losses differ")
            for name, digest in b["weight_digests"].items():
                if _digest(blk.get_submodule(name).weight.data) != digest:
                    failures.append(f"loop {tag} block {bi}: final weight of {name} differs")
                    break
    if record:
        seen = {}

        def dedup(o):                   # the runs share their inputs: store each distinct tensor once
            if isinstance(o, torch.Tensor):
                return seen.setdefault((o.dtype, tuple(o.shape), _digest(o)), o)
            if isinstance(o, (list, tuple)):
                return type(o)(dedup(v) for v in o)
            return {k: dedup(v) for k, v in o.items()} if isinstance(o, dict) else o
        torch.save(dedup(recs), LOOPS, _use_new_zipfile_serialization=False)
    return {"cases": cases, "failures": failures}


def _compact(rec):
    """What the replay reads of a recorded run: per block its inputs and the reference's losses, and a digest of every final
    weight (compared bit for bit)."""
    keep = ("block_state", "inputs", "others", "fp_outputs", "input_ids", "batches", "losses", "nv_gs")
    blocks = [dict({k: b[k] for k in keep}, weight_digests={n: _digest(l["weight"]) for n, l in b["layers"].items()})
              for b in rec["blocks"]]
    return {"iters": rec["iters"], "blocks": blocks}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--seeds", type=int, default=8)
    ap.add_argument("--loops", action="store_true", help="replay whole tuning runs with non-default loop options")
    ap.add_argument("--record", action="store_true", help="run the reference live and store its results under tests/golden/")
    args = ap.parse_args()
    if args.loops:
        res = run_loops(args.record)
        print(json.dumps(res))
        sys.exit(1 if res["failures"] else 0)
    res = run(args.seeds, args.record)
    print(json.dumps(res))
    sys.exit(1 if res["failures"] else 0)
