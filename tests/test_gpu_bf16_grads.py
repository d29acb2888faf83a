"""bf16 pre-sign gradient path used under data parallelism: the fused dW epilogue can emit dV in bf16 (half the NVLink
exchange); the update only uses the sign.  Checks: bf16 dV == bf16-rounded fp32 dV and an identical sign-SGD step."""
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("CUDA device required", allow_module_level=True)

from auto_round_b200 import ops  # noqa: E402

DEV = "cuda"


@pytest.mark.parametrize("name,bits,g", [("int_sym", 4, 128), ("nv_fp4", 4, 16)])
def test_dv_bf16_matches_fp32(name, bits, g):
    torch.manual_seed(2)
    t, n, k = 512, 256, 512
    w = (torch.randn(n, k, device=DEV) * 0.03).bfloat16()
    x = torch.randn(t, k, device=DEV).bfloat16()
    dy = (torch.randn(t, n, device=DEV) * 0.01).bfloat16()
    spec = ops.make_spec(name, bits, g, n, k)
    v = torch.rand(n, k, device=DEV) - 0.5
    mx = 0.5 + 0.5 * torch.rand(spec.groups, device=DEV)
    mn = 0.5 + 0.5 * torch.rand(spec.groups, device=DEV) if spec.is_int else None
    wmin = wmax = gs = None
    if spec.is_int:
        wmin, wmax = ops.group_minmax(spec, w)
    else:
        gs = ops.nv_global_scale(w)
    dv32 = torch.empty(n, k, device=DEV)
    dv16 = torch.empty(n, k, device=DEV, dtype=torch.bfloat16)
    dmx = torch.empty(spec.groups, device=DEV)
    dmn = torch.empty(spec.groups, device=DEV) if spec.is_int else None
    ops.fq_linear_bwd_dw(spec, dy, x, w, v, mn, mx, wmin, wmax, gs, dv32, dmn, dmx)
    ops.fq_linear_bwd_dw(spec, dy, x, w, v, mn, mx, wmin, wmax, gs, dv16, dmn, dmx)
    assert torch.equal(dv16, dv32.to(torch.bfloat16))
    # accumulate in bf16
    ops.fq_linear_bwd_dw(spec, dy, x, w, v, mn, mx, wmin, wmax, gs, dv16, dmn, dmx, accumulate=True)
    torch.testing.assert_close(dv16.float(), 2 * dv32, rtol=2 ** -7, atol=1e-6)
    # the same sign-SGD step from either gradient
    p1 = torch.rand(n * k + 4 * ((spec.groups + 3) // 4), device=DEV)
    p2 = p1.clone()
    gsc = torch.randn(p1.numel() - n * k, device=DEV)
    lr = torch.tensor([0.005, 0.005], device=DEV)
    ops.signsgd_step(p1, dv32.view(-1), None, None, lr, 0, clamp_begin=n * k, g_scales=gsc)
    ops.signsgd_step(p2, dv16.view(-1)[: n * k].contiguous(), None, None, lr, 0, clamp_begin=n * k, g_scales=gsc)
    # dv16 now holds 2*dv (same signs, except where bf16 rounding of tiny values hit zero)
    same = (p1 == p2).float().mean()
    assert same > 0.9999
