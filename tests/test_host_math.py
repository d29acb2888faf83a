"""CPU tier: the PRODUCT's device math (auto_round_b200/csrc/ar_qdq_math.cuh -- the struct every CUDA kernel and the fused
GEMM epilogue call) compiled as host C++ (tests/host_math/math_host.cpp, g++) and checked against the oracle.

This does not replace the GPU parity tests (the kernels' indexing, reductions and launches only run on the GPU); it pins the
formulas themselves without a GPU -- in particular the enable_alg_ext `init_scale` branches written after round 1's GPU
budget was spent."""
import ctypes as C
import os
import subprocess

import pytest
import torch

from oracle import qdq as Q
from oracle import signround as S

HERE = os.path.dirname(os.path.abspath(__file__))
CUDA_INC = "/usr/local/cuda/include"


@pytest.fixture(scope="session")
def host_math(tmp_path_factory):
    if not os.path.isdir(CUDA_INC):
        pytest.skip("CUDA headers not found")
    out = str(tmp_path_factory.mktemp("hostmath") / "libmath_host.so")
    src = os.path.join(HERE, "host_math", "math_host.cpp")
    subprocess.run(["g++", "-std=c++17", "-O1", "-fopenmp", "-ffp-contract=off", "-fPIC", "-shared", f"-I{CUDA_INC}", src, "-o", out],
                   check=True)
    lib = C.CDLL(out)
    F = C.POINTER(C.c_float)
    lib.host_qdq.argtypes = [C.c_int, C.c_int, C.c_int, C.c_long, F, F, F, F, F, C.c_float, C.c_float, F, F, F, F, F, F, F]
    lib.host_qdq.restype = C.c_int
    return lib


def _ptr(t):
    return None if t is None else C.cast(t.data_ptr(), C.POINTER(C.c_float))


def run_host(lib, dtype, bits, g, w, v, mn, mx, init, gscale, gq, thr=1e-5):
    groups = w.numel() // g
    wf = w.float().contiguous()
    outs = {k: torch.empty(wf.numel()) for k in ("wq", "dv")}
    outs.update({k: torch.empty(groups) for k in ("scale", "zp", "dmin", "dmax")})
    args = [t if t is None else t.float().contiguous() for t in (v, mn, mx, init, gq)]
    rc = lib.host_qdq(dtype, bits, g, groups, _ptr(wf), _ptr(args[0]), _ptr(args[1]), _ptr(args[2]), _ptr(args[3]),
                      float(gscale), thr, _ptr(args[4]), _ptr(outs["wq"]), _ptr(outs["scale"]), _ptr(outs["zp"]),
                      _ptr(outs["dv"]) if gq is not None else None, _ptr(outs["dmin"]) if gq is not None else None,
                      _ptr(outs["dmax"]) if gq is not None else None)
    assert rc == 0
    return outs


CASES = [  # name, dtype id, oracle name, bits, g, init?
    ("int_sym_w4g128", 0, "int_sym", 4, 128, False), ("int_sym_w2g32", 0, "int_sym", 2, 32, False),
    ("int_asym_w2g32", 1, "int_asym", 2, 32, False), ("mx_fp4", 2, "mx_fp4", 4, 32, False), ("nv_fp4", 3, "nv_fp4", 4, 16, False),
    ("int_sym_w2g32_init", 0, "int_sym", 2, 32, True), ("int_sym_w4g128_init", 0, "int_sym", 4, 128, True),
    ("mx_fp4_init", 2, "mx_fp4", 4, 32, True), ("nv_fp4_init", 3, "nv_fp4", 4, 16, True),
]


def _inputs(qname, bits, g, with_init, seed):
    gen = torch.Generator().manual_seed(seed)
    n, k = 24, 256
    w = (torch.randn(n, k, generator=gen) * 0.05).bfloat16()
    w[0, :g] = 0                                    # an all-zero group
    w[1, :4] = torch.tensor([0.25, -0.25, 0.1, 0.0]).bfloat16()
    w[2, 7] = 4.0                                   # an outlier
    groups = n * k // g
    v = (torch.rand(groups, g, generator=gen) - 0.5).float()
    hi = 2.0 if with_init else 1.0
    mn = (0.5 + 0.5 * torch.rand(groups, generator=gen)).float()
    mx = (0.4 * hi + 0.6 * hi * torch.rand(groups, generator=gen)).float()
    init = None
    if with_init:
        sc = S.LayerScheme(bits, g, True, {"int_sym": "int", "mx_fp4": "mx_fp", "nv_fp4": "nv_fp"}[qname])
        im = (torch.rand(k, generator=gen) ** 2 * 40 + 0.01).float()
        init = S.search_init_scale(w, sc, im, 1e-5)
    gs = Q.nv_global_scale(w).reshape(1) if qname == "nv_fp4" else None
    gq = torch.randn(n, k, generator=gen).bfloat16()
    return w, v, mn, mx, init, gs, gq


def _oracle(qname, w, bits, g, v, mn, mx, init, gs, grad_fp32=False):
    if qname == "int_sym":
        if init is not None:
            return Q.int_sym(w, bits, g, v, mn, mx, init_scale=init)
        return Q.int_sym(w, bits, g, v, mn, mx, grad_fp32=grad_fp32)
    if qname == "int_asym":
        return Q.int_asym(w, bits, g, v, mn, mx, grad_fp32=grad_fp32)
    if qname == "mx_fp4":
        return Q.mx_fp4(w, g, v, mx, init_scale=init)
    return Q.nv_fp4(w, g, v, gs, mx, init_scale=1.0 if init is None else init)


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("name,dt,qname,bits,g,with_init", CASES)
def test_device_math_on_host_matches_oracle(host_math, name, dt, qname, bits, g, with_init, seed):
    w, v, mn, mx, init, gs, gq = _inputs(qname, bits, g, with_init, seed=100 * seed + len(name))
    is_int = qname.startswith("int")
    vp, mnp, mxp = v.clone().requires_grad_(True), mn.clone().requires_grad_(True), mx.clone().requires_grad_(True)
    out, scale, zp = _oracle(qname, w, bits, g, vp, mnp, mxp, init, gs, grad_fp32=True)
    (out.float() * gq.float()).sum().backward()
    got = run_host(host_math, dt, bits, g, w, v.reshape(-1), mn if is_int else None, mx,
                   None if init is None else init.float().reshape(-1), 0.0 if gs is None else float(gs), gq.float().reshape(-1))
    # forward: bit-exact (values and scale / exponent / zero point)
    assert torch.equal(got["wq"].reshape(w.shape).bfloat16(), out.detach()), name
    assert torch.equal(got["scale"], scale.detach().float().reshape(-1)), name
    if qname == "int_asym":
        assert torch.equal(got["zp"], zp.detach().float().reshape(-1)), name
    # dL/dV: same closed form as autograd
    assert torch.allclose(got["dv"].reshape(vp.shape), vp.grad, rtol=2e-5, atol=1e-9), name
    # scale gradients.  The reference's graph rounds the scale through fp16/e4m3 with straight-through casts; with an init
    # scale the oracle keeps the plain `.to(fp16)` (its gradient is then fp16-rounded): loose bound there, tight otherwise
    ref_dm = mxp.grad
    tol = 2e-3 if (with_init and is_int) else 2e-5
    finite = torch.isfinite(ref_dm)                        # all-zero fp4 group: reference NaN (0 * inf), ours 0 (DESIGN.md 5b)
    scale_ref = ref_dm[finite].abs().max().clamp_min(1e-12)
    assert float(((got["dmax"] - ref_dm).abs()[finite]).max() / scale_ref) <= tol, name
    assert bool((got["dmax"][~finite] == 0).all())
    if is_int:
        if with_init:
            assert float(got["dmin"].abs().max()) == 0.0 and (mnp.grad is None or float(mnp.grad.abs().max()) == 0.0)
        else:
            ref_dn = mnp.grad
            assert float((got["dmin"] - ref_dn).abs().max() / ref_dn.abs().max().clamp_min(1e-12)) <= tol, name


def _bits_of_absdiff(pred, ref):
    """bf16 bit pattern (15 bits) of |pred - ref| as `torch.abs(pred - ref)` holds it -- absdiff_bits() in ar_outlier.cu."""
    return (torch.abs(pred - ref).view(torch.int16).to(torch.int32) & 0x7FFF).reshape(-1)


@pytest.mark.parametrize("rows,cols,seed", [(64, 64, 0), (512, 1024, 1), (37, 8, 2)])
def test_histogram_threshold_selects_the_topk_set(rows, cols, seed):
    """The algorithm of ar_outlier.cu restated with numpy-level ops (histogram of the bf16 pattern -> suffix scan ->
    threshold + tie budget), against torch.topk as the reference's _get_loss uses it: same number of dropped elements, same
    set above the threshold, and -- because elements AT the threshold have the same |bf16 diff| -- the same bf16-level loss
    up to which tie members are dropped."""
    gen = torch.Generator().manual_seed(seed)
    ref = torch.randn(rows, cols, generator=gen).bfloat16()
    pred = (ref.float() + 0.05 * torch.randn(rows, cols, generator=gen)).bfloat16()
    numel = rows * cols
    k = max(1, int(numel / 1000))
    bits = _bits_of_absdiff(pred, ref)
    hist = torch.bincount(bits, minlength=32768)
    suffix = torch.flip(torch.cumsum(torch.flip(hist, [0]), 0), [0])          # suffix[t] = count(pattern >= t)
    thr = int(torch.nonzero(suffix >= k).max())                                # largest t with count(>= t) >= k
    above = int(suffix[thr + 1]) if thr + 1 < 32768 else 0
    need = k - above
    assert above < k <= above + int(hist[thr]) and 1 <= need <= int(hist[thr])
    # torch.topk's choice
    _, top = torch.topk(torch.abs(pred - ref).view(-1).abs(), k)
    dropped = torch.zeros(numel, dtype=torch.bool)
    dropped[top] = True
    assert bool(dropped[bits > thr].all())                                    # everything above the threshold is dropped
    assert not bool(dropped[bits < thr].any())                                # nothing below it
    assert int(dropped[bits == thr].sum()) == need                            # and exactly `need` of the ties
    # loss: dropping ANY `need` tie members changes the sum only through the fp32 |diff| of members with equal bf16 |diff|
    d = (pred.float() - ref.float()).abs().reshape(-1)
    mine = dropped.clone()
    mine[bits == thr] = False
    tie_idx = torch.nonzero(bits == thr).reshape(-1)[:need]                    # first-come choice, as the kernel's counter
    mine[tie_idx] = True
    l_ref = float(((d * (~dropped)) ** 2).mean())
    l_mine = float(((d * (~mine)) ** 2).mean())
    assert l_mine == pytest.approx(l_ref, rel=1e-3)
    assert l_mine == pytest.approx(float(S.outlier_suppressed_loss(pred, ref, None)), rel=1e-3)
