"""enable_alg_ext on the GPU (SURVEY.md 8 rows a10 / a19): searched init scale, max_scale in [0, 2], outlier-suppressed loss.

The all-zero-group NaN of the reference's autograd (DESIGN.md 5b #2) is masked in the comparison.

What they state (same bars as tests/test_gpu_kernels.py / test_gpu_engine.py):
  * fake-quant forward with an init scale: bit-exact to the oracle (int sym, MXFP4, NVFP4)
  * backward: dV bit-exact (bf16-rounded Gq), d max_scale within 2e-3 of the oracle's fp32-graph value, d min_scale == 0
  * outlier loss: threshold selection exact (count dropped == numel // 1000), loss within 1e-5 of the oracle on tie-free
    data, gradient bf16-equal on >= 99.9 % of the elements
  * quantize_block with enable_alg_ext: iteration-0 loss within 2e-2 of the oracle's, final block MSE within +-25 %
"""
import os
import random

import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("CUDA device required", allow_module_level=True)

from auto_round_b200 import ops  # noqa: E402
from auto_round_b200.quantizer import SignRoundQuantizer  # noqa: E402
from auto_round_b200.schemes import parse_scheme  # noqa: E402
from oracle import qdq as Q  # noqa: E402
from oracle import signround as S  # noqa: E402

DEV = torch.device("cuda", 0)

CASES = {"int_sym_w2g32": ("int_sym", 2, 32), "int_sym_w4g128": ("int_sym", 4, 128), "mx_fp4": ("mx_fp4", 4, 32),
         "nv_fp4": ("nv_fp4", 4, 16)}


def _setup(name, n=16, k=256, seed=0):
    qname, bits, g = CASES[name]
    gen = torch.Generator().manual_seed(seed)
    w = (torch.randn(n, k, generator=gen) * 0.05).bfloat16()
    w[0, :g] = 0
    im = (torch.rand(k, generator=gen) ** 2 * 40 + 0.01).float()
    sc = S.LayerScheme(bits, g, True, {"int_sym": "int", "mx_fp4": "mx_fp", "nv_fp4": "nv_fp"}[qname])
    init = S.search_init_scale(w, sc, im, 1e-5)
    groups = n * k // g
    v = (torch.rand(groups, g, generator=gen) - 0.5).float()
    mx = (0.6 + 1.2 * torch.rand(groups, generator=gen)).float()          # inside [0, 2]
    return qname, bits, g, w, im, sc, init, v, mx


def _oracle_qdq(qname, w, bits, g, v, mx, init, gs):
    if qname == "int_sym":
        return Q.int_sym(w, bits, g, v, 1.0, mx, init_scale=init)
    if qname == "mx_fp4":
        return Q.mx_fp4(w, g, v, mx, init_scale=init)
    return Q.nv_fp4(w, g, v, gs, mx, init_scale=init)


@pytest.mark.parametrize("name", list(CASES))
def test_init_scale_search_and_forward_bit_exact(name):
    qname, bits, g, w, im, sc, init, v, mx = _setup(name)
    n, k = w.shape
    spec = ops.make_spec(qname, bits, g, n, k, 1e-5, 2.0)
    q = SignRoundQuantizer(parse_scheme("W4A16"), iters=1, enable_alg_ext=True)
    wd = w.to(DEV)
    got_init = q.search_init_scale(spec, type("S", (), {"qdq_name": qname})(), wd, im.to(DEV))
    assert torch.equal(got_init.cpu().reshape(-1), init.float().reshape(-1)), name
    gs = Q.nv_global_scale(w).reshape(1) if qname == "nv_fp4" else None
    ref_q, ref_s, _ = _oracle_qdq(qname, w, bits, g, v, mx, init, gs)
    wq, scale, _ = ops.qdq_fwd(spec, wd, v.reshape(n, k).to(DEV).contiguous(), None, mx.to(DEV), None, None,
                               None if gs is None else gs.to(DEV), want_scale=True, init_scale=got_init)
    assert torch.equal(wq.cpu(), ref_q), name
    assert torch.equal(scale.float().cpu().reshape(-1), ref_s.float().reshape(-1)), name


@pytest.mark.parametrize("name", list(CASES))
def test_init_scale_backward(name):
    qname, bits, g, w, im, sc, init, v, mx = _setup(name, seed=3)
    n, k = w.shape
    gs = Q.nv_global_scale(w).reshape(1) if qname == "nv_fp4" else None
    vp = v.clone().requires_grad_(True)
    mp = mx.clone().requires_grad_(True)
    out, _, _ = _oracle_qdq(qname, w, bits, g, vp, mp, init, gs)
    gq = torch.randn(n, k, generator=torch.Generator().manual_seed(9)).bfloat16()
    (out.float() * gq.float()).sum().backward()
    spec = ops.make_spec(qname, bits, g, n, k, 1e-5, 2.0)
    wmin = wmax = None
    if qname == "int_sym":
        wmin, wmax = ops.group_minmax(spec, w.to(DEV))
    dv, dmin, dmax = ops.qdq_bwd(spec, w.to(DEV), gq.float().to(DEV).contiguous(), v.reshape(n, k).to(DEV).contiguous(), None,
                                 mx.to(DEV), wmin, wmax, None if gs is None else gs.to(DEV), init_scale=init.float().reshape(-1).to(DEV))
    ref_dv = vp.grad.reshape(n, k)
    assert torch.allclose(dv.cpu(), ref_dv, rtol=2e-5, atol=1e-9), name
    ref_dm = mp.grad
    # row 0's first group is all-zero: the reference's autograd yields NaN there for mx/nv (0 * inf), the CUDA path defines
    # d(max_scale) = 0 (DESIGN.md 5b #2) -- compare the finite positions, require 0 at the NaN ones
    nan = torch.isnan(ref_dm)
    assert int(nan.sum()) <= 1 and float(dmax.cpu()[nan].abs().sum()) == 0.0, name
    denom = ref_dm[~nan].abs().max().clamp_min(1e-12)
    assert float((dmax.cpu() - ref_dm)[~nan].abs().max() / denom) <= 2e-3, name
    if dmin is not None:
        assert float(dmin.abs().max()) == 0.0


@pytest.mark.parametrize("rows,cols,masked", [(64, 64, True), (4096, 4096, True), (1000, 128, False)])
def test_outlier_loss_matches_oracle(rows, cols, masked):
    gen = torch.Generator().manual_seed(rows + cols)
    ref = torch.randn(rows, cols, generator=gen).bfloat16()
    pred = (ref.float() + 0.05 * torch.randn(rows, cols, generator=gen)).bfloat16()
    pred[3, 5] += 2.0                                                       # a few unmistakable outliers
    pred[rows // 2, cols // 2] -= 3.0
    mask = None
    if masked:
        mask = (torch.rand(rows, generator=gen) > 0.1).to(torch.uint8)
    p32 = pred.clone().requires_grad_(True)
    m3 = None if mask is None else mask.reshape(rows, 1).long()
    loss = S.outlier_suppressed_loss(p32, ref, m3)
    (loss * 1000).backward()
    scratch = ops.OutlierSelect(DEV)
    loss_sum = torch.zeros(1, dtype=torch.float64, device=DEV)
    dpred = ops.mse_outlier_fwd_bwd(pred.to(DEV), ref.to(DEV), None if mask is None else mask.to(DEV), 1000.0, loss_sum, scratch)
    torch.cuda.synchronize()
    numel = rows * cols
    k = max(1, int(numel / 1000))
    sel = scratch.sel.cpu().tolist()
    diff_bits = (torch.abs(pred - ref).view(torch.int16).int() & 0x7FFF).reshape(-1)
    above = int((diff_bits > sel[0]).sum())
    assert above < k <= above + int((diff_bits == sel[0]).sum())           # the threshold is the k-th largest pattern
    assert sel[1] == k - above and sel[2] >= sel[1]                         # exactly k elements are dropped
    assert int(scratch.hist.abs().sum()) == 0                               # histogram re-armed for the next iteration
    got = float(loss_sum) / numel
    assert got == pytest.approx(float(loss), rel=1e-4)
    same = (dpred.cpu() == p32.grad.to(torch.bfloat16))
    assert float(same.float().mean()) >= 0.999


ALGEXT = {
    "algext_w2a16_sym_g32": (dict(scheme="W2A16", group_size=32), S.LayerScheme(2, 32, True, "int")),
    "algext_w4a16_sym_g32": (dict(scheme="W4A16", group_size=32), S.LayerScheme(4, 32, True, "int")),
    "algext_mxfp4": (dict(scheme="MXFP4", act_bits=16), S.LayerScheme(4, 32, True, "mx_fp")),
    "algext_nvfp4": (dict(scheme="NVFP4", act_bits=16, act_data_type="float"), S.LayerScheme(4, 16, True, "nv_fp")),
    "algext_w2a16_asym_g32": (dict(scheme="W2A16", group_size=32, sym=False), S.LayerScheme(2, 32, False, "int")),
}


@pytest.mark.parametrize("tag", list(ALGEXT))
def test_quantize_block_alg_ext_vs_oracle(golden_dir, tag):
    from test_gpu_engine import _block_mse, _tiny_block      # tests/ is on sys.path (pytest rootdir import mode)

    rec = torch.load(os.path.join(golden_dir, f"block_{tag}.pt"), weights_only=False)
    kw, osc = ALGEXT[tag]
    scheme = parse_scheme(kw["scheme"], {k: v for k, v in kw.items() if k != "scheme"})
    b = rec["blocks"][0]
    masks = [(ids != -100).to(torch.long) for ids in b["input_ids"]]
    iters = 40
    random.seed(1234)
    oblk = _tiny_block(b["block_state"])
    ores = S.tune_block(oblk, b["inputs"], b["others"], b["fp_outputs"], lambda n, m: osc, iters=iters,
                        batch_size=rec["batch_size"], token_masks=masks, nv_global_scales=b["nv_gs"] or None, alg_ext=True,
                        imatrices=b["imatrix"])
    o_mse = _block_mse(oblk, b["inputs"], b["others"], b["fp_outputs"], masks, "cpu")
    blk = _tiny_block(b["block_state"], DEV)
    for p in blk.parameters():
        p.requires_grad_(False)
    q = SignRoundQuantizer(scheme, iters=iters, batch_size=rec["batch_size"], enable_alg_ext=True)
    nv = {n: g.to(DEV).reshape(1) for n, g in b["nv_gs"].items()} if b["nv_gs"] else None
    q.quantize_block(blk, [t.to(DEV) for t in b["inputs"]], b["others"], [t.to(DEV) for t in b["fp_outputs"]], None, None,
                     input_ids=b["input_ids"], nv_global_scales=nv, sampler=S.ReplaySampler(ores.batches),
                     imatrices={n: t.to(DEV) for n, t in b["imatrix"].items()})
    res = q.last_result
    assert res.losses[0] == pytest.approx(ores.losses[0], rel=2e-2)
    n0 = sum(int(masks[i].sum()) for i in ores.batches[0])
    assert res.losses[0] * n0 == pytest.approx(rec["blocks"][0]["losses"][0], rel=2e-2) or ores.batches[0] != b["batches"][0]
    g_mse = _block_mse(blk, b["inputs"], b["others"], b["fp_outputs"], masks, DEV)
    assert res.best_loss <= res.losses[0] + 1e-12
    assert g_mse == pytest.approx(o_mse, rel=0.25), (g_mse, o_mse)
    for name, lay in b["layers"].items():
        mod = blk.get_submodule(name)
        assert type(mod) is torch.nn.Linear and tuple(mod.scale.shape) == tuple(lay["scale"].shape)
