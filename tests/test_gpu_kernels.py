"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle and the committed golden
fixtures of the reference.  Run on an H100:  python -m pytest tests -m gpu -q

Tolerances (stated per check):
  * integer / byte outputs (packed words, codes, nibbles, e4m3/e8m0 scales): bit-exact;
  * fake-quant forward (Wq bf16, scale, zp) and dV: bit-exact (same fp32 op sequence, no FMA contraction);
  * d(min/max_scale): fp32 group sums vs the reference's fp16-rounded autograd -> |err| <= 2e-3*|ref| + 1e-3*scale;
  * bf16 tensor-core GEMMs: fp32-accumulated bf16 products vs an fp32 torch reference ->
    |d - ref| <= 2^-7*|ref| + 2e-3*rms(ref)  (one bf16 output rounding = 2^-9 relative, plus summation order).
"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():  # the whole module needs a device; `-m "not gpu"` deselects it anyway
    pytest.skip("CUDA device required", allow_module_level=True)

from auto_round_b200 import ops  # noqa: E402
from oracle import pack as P  # noqa: E402
from oracle import qdq as Q  # noqa: E402

DEV = "cuda"


def _load(golden_dir, name):
    return torch.load(os.path.join(golden_dir, name), weights_only=False)


def _spec_for(name, kw, n, k):
    base = name.split("_w")[0] if name.startswith("int") else ("mx_fp4" if name.startswith("mx") else "nv_fp4")
    return ops.make_spec(base, kw["bits"], kw["group_size"], n, k)


def _close_scalegrad(got, ref):
    """d(min/max_scale): the reference rounds the two partial sums of dL/ds to fp16 SEPARATELY (the scale tensor is
    fp16, so autograd accumulates its gradient in fp16) before they cancel; we keep fp32.  Bound: 1e-2 relative
    + 5e-3 of the mean magnitude, and identical sign wherever the value is not at that noise floor."""
    ref = torch.nan_to_num(ref.float(), nan=0.0)
    got = got.float().cpu()
    floor = 2e-2 * (ref.abs().mean() + 1e-12)           # fp16 cancellation noise of the REFERENCE's own value
    ok = bool(((got - ref).abs() <= 1e-2 * ref.abs() + floor).all())
    big = ref.abs() > 4 * floor
    return ok and bool((torch.sign(got)[big] == torch.sign(ref)[big]).all())


def _tight_scalegrad(got, exact):
    """against the exact-arithmetic (fp32-accumulated) gradient of the same graph (oracle grad_fp32=True)."""
    exact = torch.nan_to_num(exact.float(), nan=0.0)
    got = got.float().cpu()
    return bool(((got - exact).abs() <= 2e-4 * exact.abs() + 2e-5 * (exact.abs().mean() + 1e-12)).all())


# ------------------------------------------------------------------------------------------------ qdq
def test_qdq_golden_fwd_bwd(golden_dir):
    gold = _load(golden_dir, "qdq.pt")
    for key, rec in gold.items():
        if key.startswith("rtn"):
            continue
        name = key.split("/")[0]
        w = rec["w"].to(DEV)
        n, k = w.shape
        spec = _spec_for(name, rec["kw"], n, k)
        v = rec["v"].to(DEV).contiguous()
        mn = rec["min_scale"].to(DEV) if spec.is_int else None
        mx = rec["max_scale"].to(DEV)
        wmin = wmax = gs = None
        if spec.is_int:
            wmin, wmax = ops.group_minmax(spec, w)
            rmin, rmax = Q.group_minmax(rec["w"], rec["kw"]["group_size"])
            assert torch.equal(wmin.cpu(), rmin) and torch.equal(wmax.cpu(), rmax), key
        if name.startswith("nv"):
            gs = ops.nv_global_scale(w)
            assert torch.equal(gs.cpu().reshape(()), rec["global_scale"].reshape(())), key
        wq, scale, zp = ops.qdq_fwd(spec, w, v, mn, mx, wmin, wmax, gs, want_scale=True)
        assert torch.equal(wq.cpu(), rec["wq"]), key
        assert torch.equal(scale.cpu().float().reshape(-1), rec["scale"].float().reshape(-1)), key
        if isinstance(rec["zp"], torch.Tensor):
            assert torch.equal(zp.cpu().reshape(-1), rec["zp"].reshape(-1)), key
        # recomputing min/max inside the kernel must give the same answer
        wq2, _, _ = ops.qdq_fwd(spec, w, v, mn, mx, None, None, gs)
        assert torch.equal(wq2.cpu(), rec["wq"]), key
        # autograd hands the qdq graph a bf16-rounded dL/dWq (Wq is a bf16 tensor): feed the kernel the same values
        gq = rec["gq"].to(torch.bfloat16).float().to(DEV).contiguous()
        dv, dmin, dmax = ops.qdq_bwd(spec, w, gq, v, mn, mx, wmin, wmax, gs)
        ref_dv = rec["dv"].reshape(n, -1)
        ok = ~torch.isnan(ref_dv)
        if name.startswith("mx"):   # closed form o/t vs autograd's (1 - y*dP/dt) + o*dP/dt: 1e-5 relative
            torch.testing.assert_close(dv.cpu()[ok], ref_dv[ok], rtol=2e-5, atol=1e-7)
        else:
            assert torch.equal(dv.cpu()[ok], ref_dv[ok]), key
        if rec["dmax"] is not None:
            assert _close_scalegrad(dmax, rec["dmax"]), key
        if rec["dmin"] is not None:
            assert _close_scalegrad(dmin, rec["dmin"]), key


def test_rtn_golden(golden_dir):
    rec = _load(golden_dir, "qdq.pt")["rtn_int_sym_w4g128"]
    w = rec["w"].to(DEV)
    spec = ops.make_spec("int_sym", 4, 128, *w.shape)
    wq, scale, _ = ops.qdq_fwd(spec, w, want_scale=True)         # V=0, scales=1, min/max recomputed: plain RTN
    assert torch.equal(wq.cpu(), rec["wq"])
    assert torch.equal(scale.cpu().reshape(-1), rec["scale"].reshape(-1))


@pytest.mark.parametrize("name,bits,g", [("int_sym", 4, 128), ("int_sym", 2, 32), ("int_asym", 2, 32),
                                         ("int_asym", 4, 64), ("mx_fp4", 4, 32), ("nv_fp4", 4, 16),
                                         ("int_sym", 8, 256), ("int_sym", 3, 128)])
def test_qdq_vs_oracle_random(name, bits, g):
    torch.manual_seed(hash((name, bits, g)) % 1000)
    n, k = 192, 1024
    w = (torch.randn(n, k) * 0.03).bfloat16()
    w[5, :g] = 0
    grp, _, _ = Q.to_groups(w, g)
    v = (torch.rand(grp.shape) - 0.5) * 1.004
    mn = 0.3 + 0.7 * torch.rand(grp.shape[0])
    mx = 0.3 + 0.7 * torch.rand(grp.shape[0])
    gq = torch.randn(n, k)
    vr, mnr, mxr = v.clone().requires_grad_(), mn.clone().requires_grad_(), mx.clone().requires_grad_()
    if name == "int_sym":
        wmin, wmax = Q.group_minmax(w, g)
        wq, sc, zp = Q.int_sym(w, bits, g, vr, mnr, mxr, wmin, wmax)
    elif name == "int_asym":
        wmin, wmax = Q.group_minmax(w, g)
        wq, sc, zp = Q.int_asym(w, bits, g, vr, mnr, mxr, wmin, wmax)
    elif name == "mx_fp4":
        wq, sc, zp = Q.mx_fp4(w, g, vr, mxr)
    else:
        gsr = Q.nv_global_scale(w)
        wq, sc, zp = Q.nv_fp4(w, g, vr, gsr, mxr)
    (wq.float() * gq).sum().backward()
    spec = ops.make_spec(name, bits, g, n, k)
    wd = w.to(DEV)
    gs = ops.nv_global_scale(wd) if name == "nv_fp4" else None
    wmin_d = wmax_d = None
    if spec.is_int:
        wmin_d, wmax_d = ops.group_minmax(spec, wd)
    mn_d = mn.to(DEV) if spec.is_int else None
    out, sc_d, zp_d = ops.qdq_fwd(spec, wd, v.to(DEV).contiguous(), mn_d, mx.to(DEV), wmin_d, wmax_d, gs, want_scale=True)
    assert torch.equal(out.cpu(), wq.detach())
    assert torch.equal(sc_d.cpu().float().reshape(-1), sc.detach().float().reshape(-1))
    if isinstance(zp, torch.Tensor):
        assert torch.equal(zp_d.cpu().reshape(-1), zp.detach().reshape(-1))
    gq_d = gq.to(torch.bfloat16).float().to(DEV)      # grad w.r.t. the bf16 Wq is bf16-rounded in autograd
    dv, dmin, dmax = ops.qdq_bwd(spec, wd, gq_d, v.to(DEV).contiguous(), mn_d, mx.to(DEV), wmin_d, wmax_d, gs)
    ref_dv = vr.grad.reshape(n, -1)
    ok = ~torch.isnan(ref_dv)
    if name in ("int_sym", "int_asym", "nv_fp4"):
        assert torch.equal(dv.cpu()[ok], ref_dv[ok])
    else:  # mx: autograd evaluates (1 - y*dP/dt) + o*dP/dt in fp32; we use the closed form o/t -> 1e-5 relative
        torch.testing.assert_close(dv.cpu()[ok], ref_dv[ok], rtol=2e-5, atol=1e-7)
    assert _close_scalegrad(dmax, mxr.grad)
    if spec.is_int:
        assert _close_scalegrad(dmin, mnr.grad)
        # tight check against the exact-arithmetic gradient of the same graph (forward values bit-identical)
        v2, mn2, mx2 = v.clone().requires_grad_(), mn.clone().requires_grad_(), mx.clone().requires_grad_()
        fn = Q.int_sym if name == "int_sym" else Q.int_asym
        wq2, _, _ = fn(w, bits, g, v2, mn2, mx2, wmin, wmax, grad_fp32=True)
        assert torch.equal(wq2.detach(), wq.detach())
        (wq2.float() * gq).sum().backward()
        assert _tight_scalegrad(dmax, mx2.grad)
        assert _tight_scalegrad(dmin, mn2.grad)


# ----------------------------------------------------------------------------------------------- pack
def test_pack_golden(golden_dir):
    gold = _load(golden_dir, "pack.pt")
    for key, rec in gold.items():
        wq = rec["wq"].to(DEV)
        n, k = wq.shape
        if key.startswith("int"):
            sym = key.endswith("gptq_zp")
            zp = None if sym else rec["zp"].float().to(DEV).contiguous()
            qw, qz, st, gi = ops.pack_int(wq, rec["scale"].to(DEV).contiguous(), zp, rec["bits"], rec["group_size"],
                                          zp_minus_one=sym, zp_const=rec["zp"] if sym else 0)
            assert torch.equal(qw.cpu(), rec["qweight"]), key
            assert torch.equal(qz.cpu(), rec["qzeros"]), key
            assert torch.equal(st.cpu(), rec["scales"]), key
            if "g_idx" in rec:
                assert torch.equal(gi.cpu(), rec["g_idx"]), key
            # round trip through the unpacker: codes -> dequant == qdq weight
            wback, codes = ops.unpack_int(qw, qz, st, n, k, rec["bits"], rec["group_size"], sym, want_codes=True)
            assert torch.equal(wback.cpu(), rec["wq"]), key
        elif key == "nv_fp4":
            pk, sc = ops.pack_fp4_nv(wq, rec["scale"].to(DEV).contiguous(), rec["global_scale"].reshape(1).to(DEV))
            assert torch.equal(pk.cpu(), rec["weight_packed"])
            assert torch.equal(sc.cpu(), rec["weight_scale"])
        else:
            pk, sc = ops.pack_fp4_mx(wq, rec["scale"].to(DEV).contiguous())
            assert torch.equal(pk.cpu(), rec["weight_packed"])
            assert torch.equal(sc.cpu(), rec["weight_scale"])


def test_pack_int4_llama_shape_vs_oracle():
    """q_proj-sized layer (4096x4096, W4 g128): packed words bit-exact against the numpy oracle."""
    torch.manual_seed(3)
    n, k, g = 4096, 4096, 128
    w = (torch.randn(n, k) * 0.02).bfloat16()
    spec = ops.make_spec("int_sym", 4, g, n, k)
    wd = w.to(DEV)
    v = ((torch.rand(n, k) - 0.5)).to(DEV)
    wq, scale, _ = ops.qdq_fwd(spec, wd, v, want_scale=True)
    scale2 = scale.reshape(n, -1)
    qw, qz, st, gi = ops.pack_int(wq, scale2.contiguous(), None, 4, g, True, zp_const=8)
    ref = P.pack_int(wq.cpu(), scale2.cpu(), 8, 4, g, zp_minus_one=True)
    assert np.array_equal(qw.cpu().numpy(), ref["qweight"])
    assert np.array_equal(qz.cpu().numpy(), ref["qzeros"])
    assert np.array_equal(st.cpu().numpy(), ref["scales"])
    assert int(qz.cpu()[0, 0]) == 0x77777777
    # size-independent property: unpack(pack(x)) == x and codes in range
    wback, codes = ops.unpack_int(qw, qz, st, n, k, 4, g, True, want_codes=True)
    assert torch.equal(wback, wq)
    assert int(codes.min()) >= 0 and int(codes.max()) <= 15


def test_fp4_nibble_known_answers_gpu():
    # reference literals: test/unit/test_cpu/export/test_qlinear_fp_helpers.py:174-221
    for val, byte in [(6.0, 0x77), (-6.0, 0xFF), (0.5, 0x11), (0.0, 0x00)]:
        wq = torch.full((1, 32), val, dtype=torch.bfloat16, device=DEV)
        e = torch.zeros(1, 1, dtype=torch.bfloat16, device=DEV)
        pk, sc = ops.pack_fp4_mx(wq, e)
        assert int(pk[0, 0]) == byte and int(sc[0, 0]) == 127
    back = ops.unpack_fp4(pk, 1, 32)
    assert torch.equal(back, torch.zeros_like(back))


# ----------------------------------------------------------------------------------------------- GEMM
def _gemm_close(d, ref):
    ref = ref.float()
    d = d.float().to(ref.device)
    rms = ref.pow(2).mean().sqrt()
    bad = (d - ref).abs() > (2.0 ** -7) * ref.abs() + 2e-3 * rms
    assert not bool(bad.any()), f"{int(bad.sum())} elements off; max abs err {float((d - ref).abs().max())}, rms {float(rms)}"


def _gemm_ref(a, b, a_mn, b_mn, bias=None):
    A = a.float().t() if a_mn else a.float()
    B = b.float().t() if b_mn else b.float()
    out = A @ B.t()
    if bias is not None:
        out = out + bias.float()
    return out


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("m,n,k", [(128, 256, 64), (256, 512, 256), (200, 328, 136), (1024, 1536, 2048)])
def test_gemm_all_majors(a_mn, b_mn, m, n, k):
    torch.manual_seed(m + n + k)
    a = torch.randn((k, m) if a_mn else (m, k), device=DEV).bfloat16()
    b = torch.randn((k, n) if b_mn else (n, k), device=DEV).bfloat16()
    bias = torch.randn(n, device=DEV).bfloat16()
    _gemm_close(ops.gemm(a, b, a_mn, b_mn), _gemm_ref(a, b, a_mn, b_mn))
    _gemm_close(ops.gemm(a, b, a_mn, b_mn, bias=bias), _gemm_ref(a, b, a_mn, b_mn, bias))


def test_gemm_llama_shapes_linearity():
    """Full-size shapes (T=16384 tokens): linearity D(a1+a2) == D(a1)+D(a2) within bf16 rounding, plus a sampled
    fp32 check of 64 rows."""
    torch.manual_seed(0)
    t, n, k = 16384, 4096, 4096
    x = torch.randn(t, k, device=DEV).bfloat16()
    w = (torch.randn(n, k, device=DEV) * 0.02).bfloat16()
    y = ops.gemm(x, w)
    rows = torch.randint(0, t, (64,), device=DEV)
    _gemm_close(y[rows], x[rows].float() @ w.float().t())
    y2 = ops.gemm((x * 2).contiguous(), w)
    assert torch.equal(y2, (y.float() * 2).bfloat16())      # scaling by 2 is exact in bf16


# ------------------------------------------------------------------------------- fake-quant linear
@pytest.mark.parametrize("name,bits,g", [("int_sym", 4, 128), ("int_asym", 2, 32), ("mx_fp4", 4, 32), ("nv_fp4", 4, 16),
                                         ("int_sym", 4, 32), ("int_asym", 4, 64)])
def test_fake_quant_linear_vs_oracle(name, bits, g):
    """The product's fake-quant linear: forward = ar_qdq_fwd + wgmma GEMM, grad-in GEMM, and the weight gradient of the
    bf16 grad-w GEMM through the fused update's fake-quant backward."""
    torch.manual_seed(11)
    t, n, k = 384, 256, 512
    w = (torch.randn(n, k) * 0.03).bfloat16()
    x = torch.randn(t, k).bfloat16()
    dy = (torch.randn(t, n) * 0.01).bfloat16()
    grp, _, _ = Q.to_groups(w, g)
    v = (torch.rand(grp.shape) - 0.5)
    mn = 0.5 + 0.5 * torch.rand(grp.shape[0])
    mx = 0.5 + 0.5 * torch.rand(grp.shape[0])
    vr, mnr, mxr = v.clone().requires_grad_(), mn.clone().requires_grad_(), mx.clone().requires_grad_()
    xr = x.float().requires_grad_()
    if name == "int_sym":
        wmin, wmax = Q.group_minmax(w, g)
        wq, _, _ = Q.int_sym(w, bits, g, vr, mnr, mxr, wmin, wmax)
    elif name == "int_asym":
        wmin, wmax = Q.group_minmax(w, g)
        wq, _, _ = Q.int_asym(w, bits, g, vr, mnr, mxr, wmin, wmax)
    elif name == "mx_fp4":
        wq, _, _ = Q.mx_fp4(w, g, vr, mxr)
    else:
        wq, _, _ = Q.nv_fp4(w, g, vr, Q.nv_global_scale(w), mxr)
    y_ref = xr @ wq.float().t()                        # fp32 reference of the bf16-input GEMM
    (y_ref * dy.float()).sum().backward()

    spec = ops.make_spec(name, bits, g, n, k)
    wd, xd, dyd = w.to(DEV), x.to(DEV), dy.to(DEV)
    gs = ops.nv_global_scale(wd) if name == "nv_fp4" else None
    wmin_d = wmax_d = None
    if spec.is_int:
        wmin_d, wmax_d = ops.group_minmax(spec, wd)
    vd, mxd = v.to(DEV).contiguous(), mx.to(DEV)
    mnd = mn.to(DEV) if spec.is_int else None
    wqd, _, _ = ops.qdq_fwd(spec, wd, vd, mnd, mxd, wmin_d, wmax_d, gs)
    assert torch.equal(wqd.cpu(), wq.detach())
    y = ops.gemm(xd, wqd)
    _gemm_close(y.cpu(), y_ref.detach())
    dx = ops.fq_linear_bwd_dx(spec, dyd, wqd)
    _gemm_close(dx.cpu(), xr.grad)
    # weight gradient: bf16 dWq of the grad-w GEMM -> the fake-quant backward of ar_fq_update (its pre-sign outputs)
    gq = ops.gemm(dyd, xd, a_mn_major=True, b_mn_major=True)
    dv = torch.empty(n, spec.kpad, dtype=torch.float32, device=DEV)
    dmn = torch.empty(spec.groups, dtype=torch.float32, device=DEV)
    dmx = torch.empty(spec.groups, dtype=torch.float32, device=DEV)
    lr_tab = torch.tensor([0.005, 0.005], device=DEV)
    ops.fq_update(spec, wd, vd, mnd, mxd, wmin_d, wmax_d, gs, gq, torch.empty_like(wd), lr_tab, dbg=(dv, dmn, dmx))
    # it agrees in SIGN with the oracle's autograd wherever the gradient is not at the noise floor
    ref = vr.grad.reshape(n, -1)[:, :k]
    big = ref.abs() > 1e-3 * ref.abs().max()
    agree = (torch.sign(dv[:, :k].cpu())[big] == torch.sign(ref)[big]).float().mean()
    assert agree > 0.9999


# ----------------------------------------------------------------------------------------- loop glue
def test_mse_best_gather():
    torch.manual_seed(5)
    rows, cols = 64, 256
    pred = torch.randn(rows, cols).bfloat16()
    ref = torch.randn(rows, cols).bfloat16()
    mask = (torch.rand(rows) > 0.2)
    m = mask.to(torch.long).unsqueeze(-1)
    pr = pred.clone().requires_grad_()
    loss = torch.nn.functional.mse_loss((pr * m).float(), (ref * m).float())
    (loss * 1000).backward()
    loss_sum = torch.zeros(1, dtype=torch.float64, device=DEV)
    dp = ops.mse_fwd_bwd(pred.to(DEV), ref.to(DEV), mask.to(torch.uint8).to(DEV), 1.0 / (rows * cols), 1000.0, loss_sum)
    assert float(loss_sum) / (rows * cols) == pytest.approx(float(loss), rel=1e-6)
    assert torch.equal(dp.cpu(), pr.grad)
    state = torch.zeros(4, dtype=torch.float64, device=DEV)
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    hist = torch.zeros(8, dtype=torch.float32, device=DEV)
    ops.best_update(loss_sum, 1.0 / (rows * cols), 1.0 / 7.0, 0, state, flag, hist)
    assert int(flag) == 1 and float(loss_sum) == 0.0
    assert float(state[0]) == pytest.approx(float(loss) / 7.0, rel=1e-6) and float(hist[0]) == pytest.approx(float(loss) / 7, rel=1e-6)
    loss_sum.fill_(1e9)
    ops.best_update(loss_sum, 1.0, 1.0, 1, state, flag, hist)
    assert int(flag) == 0 and float(state[2]) == 0.0
    src = torch.randn(6, 4, 64, device=DEV).bfloat16()
    idx = torch.tensor([5, 0, 3], dtype=torch.int32, device=DEV)
    assert torch.equal(ops.gather_rows(src, idx), src[[5, 0, 3]])
