"""GPU checks of what the 128 x 256 store tiles and the register-to-global epilogue of ar::gemm_kernel can break: ragged
edges in n (not a multiple of the 256-wide tile), m and k, bias, column-slice outputs with a row pitch wider than n,
run-to-run determinism under the dynamic tile scheduler, a launch from a thread without a current CUDA context, and the
grouped MoE launches with ragged n.

Tolerance (same as the GEMM checks of test_gpu_kernels.py): fp32-accumulated bf16 products against an fp32 torch
reference, |d - ref| <= 2^-7*|ref| + 2e-3*rms(ref)."""
import ctypes as C
import threading

import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("CUDA device required", allow_module_level=True)

from auto_round_b200 import _lib, ops  # noqa: E402

DEV = "cuda"
MAJORS = [(False, False), (False, True), (True, False), (True, True)]
SENTINEL = -1234.0                                       # exact in bf16


def _close(d, ref):
    ref = ref.float()
    d = d.float().to(ref.device)
    rms = ref.pow(2).mean().sqrt()
    bad = (d - ref).abs() > (2.0 ** -7) * ref.abs() + 2e-3 * rms
    assert not bool(bad.any()), f"{int(bad.sum())} elements off; max abs err {float((d - ref).abs().max())}, rms {float(rms)}"


def _operands(m, n, k, a_mn, b_mn, seed):
    torch.manual_seed(seed)
    a = torch.randn((k, m) if a_mn else (m, k), device=DEV).bfloat16()
    b = torch.randn((k, n) if b_mn else (n, k), device=DEV).bfloat16()
    return a, b


def _ref(a, b, a_mn, b_mn, bias=None):
    A = a.float().t() if a_mn else a.float()
    B = b.float().t() if b_mn else b.float()
    out = A @ B.t()
    return out + bias.float() if bias is not None else out


@pytest.mark.parametrize("a_mn,b_mn", MAJORS)
@pytest.mark.parametrize("n", [200, 1152, 4160])
def test_ragged_n_m_k(a_mn, b_mn, n):
    m, k = 328, 200                                      # m % 128 != 0, k % 64 != 0 (both multiples of 8 for TMA pitches)
    a, b = _operands(m, n, k, a_mn, b_mn, seed=n)
    bias = torch.randn(n, device=DEV).bfloat16()
    _close(ops.gemm(a, b, a_mn, b_mn), _ref(a, b, a_mn, b_mn))
    _close(ops.gemm(a, b, a_mn, b_mn, bias=bias), _ref(a, b, a_mn, b_mn, bias))


@pytest.mark.parametrize("a_mn,b_mn", MAJORS)
@pytest.mark.parametrize("bias_on", [False, True])
def test_column_slice_output_leaves_the_rest(a_mn, b_mn, bias_on):
    m, n, k = 328, 200, 136
    a, b = _operands(m, n, k, a_mn, b_mn, seed=7)
    bias = torch.randn(n, device=DEV).bfloat16() if bias_on else None
    buf = torch.full((m + 9, 1024), SENTINEL, device=DEV, dtype=torch.bfloat16)
    c0 = 136                                             # 272-byte offset: 16-byte aligned, not tile aligned
    view = buf[:m, c0:c0 + n]
    # ops.gemm takes contiguous outputs only; the C ABI takes any 16-byte aligned output with a row pitch ldd >= n
    rc = _lib.load().ar_gemm_bf16(C.c_void_p(a.data_ptr()), C.c_void_p(b.data_ptr()), C.c_void_p(view.data_ptr()), m, n, k,
                                  int(a_mn), int(b_mn), a.stride(0), b.stride(0), view.stride(0),
                                  C.c_void_p(bias.data_ptr() if bias is not None else 0),
                                  C.c_void_p(torch.cuda.current_stream().cuda_stream))
    _lib.check(rc, "ar_gemm_bf16")
    _close(view, _ref(a, b, a_mn, b_mn, bias))
    outside = torch.ones_like(buf, dtype=torch.bool)
    outside[:m, c0:c0 + n] = False
    assert bool((buf[outside] == SENTINEL).all()), f"{int((buf[outside] != SENTINEL).sum())} elements outside the slice written"


@pytest.mark.parametrize("a_mn,b_mn", MAJORS)
def test_repeat_launch_bit_identical(a_mn, b_mn):
    m, n, k = 2048, 4160, 1024                           # 16 x 17 tiles: more tiles than SMs, a ragged last column tile
    a, b = _operands(m, n, k, a_mn, b_mn, seed=3)
    d1 = ops.gemm(a, b, a_mn, b_mn)
    d2 = ops.gemm(a, b, a_mn, b_mn)
    assert torch.equal(d1, d2)
    rows = torch.randint(0, m, (64,), device=DEV)
    _close(d1[rows], _ref(a, b, a_mn, b_mn)[rows])


def test_launch_from_a_thread_without_a_context():
    """The first GEMM of a thread that has made no CUDA runtime call, as PyTorch's autograd device threads start: encoding
    the TMA descriptors needs a current context, and the launch makes the device's primary context current itself."""
    a, b = _operands(256, 512, 128, False, False, seed=4)
    want = ops.gemm(a, b)
    got = torch.empty_like(want)
    err = []

    def run():
        try:
            ops.gemm(a, b, out=got)
        except Exception as e:  # noqa: BLE001 -- reported by the assertion below
            err.append(e)

    t = threading.Thread(target=run)
    t.start()
    t.join()
    assert not err, err[0]
    torch.cuda.synchronize()
    assert torch.equal(got, want)


def _route(tokens, e, topk, skip):
    g = torch.Generator().manual_seed(tokens)
    logits = torch.randn(tokens, e, generator=g)
    logits[:, skip] = -1e9                               # an expert without tokens
    idx = torch.topk(logits, topk, dim=-1).indices
    route = ops.moe_route(ops.MoeRoute(tokens * topk, e, DEV), idx.reshape(-1).to(DEV))
    torch.cuda.synchronize()
    return route, route.offsets.cpu().tolist()


@pytest.mark.parametrize("b_mn", [False, True])
def test_grouped_m_ragged_n(b_mn):
    tokens, e, topk, n, k = 700, 4, 2, 200, 136
    route, offs = _route(tokens, e, topk, skip=1)
    rows = route.max_rows
    torch.manual_seed(5)
    a = torch.randn(rows, k, device=DEV).bfloat16()
    b_stack = torch.randn((e, k, n) if b_mn else (e, n, k), device=DEV).bfloat16()
    out = torch.full((rows, n), SENTINEL, device=DEV, dtype=torch.bfloat16)
    ops.gemm_grouped_m(a, b_stack, route, n=n, k=k, b_mn_major=b_mn, out=out)
    for j in range(e):
        lo, hi = offs[j], offs[j + 1]
        if hi == lo:
            continue
        bj = b_stack[j].float()
        _close(out[lo:hi], a[lo:hi].float() @ (bj if b_mn else bj.t()))
    assert bool((out[offs[-1]:] == SENTINEL).all())     # rows past the last expert's segment are not written


def test_grouped_k_ragged_n():
    tokens, e, topk, n_out, k_out = 700, 4, 2, 328, 200
    route, offs = _route(tokens, e, topk, skip=2)
    rows = route.max_rows
    torch.manual_seed(6)
    dy = torch.randn(rows, n_out, device=DEV).bfloat16()
    x = torch.randn(rows, k_out, device=DEV).bfloat16()
    pitch = 512                                          # n_out rounded up to 256
    out = torch.full((e, pitch, k_out), SENTINEL, device=DEV, dtype=torch.bfloat16)
    ops.gemm_grouped_k(dy, x, route, out)
    for j in range(e):
        lo, hi = offs[j], offs[j + 1]
        if hi == lo:
            assert bool((out[j] == SENTINEL).all())      # an expert without tokens keeps its slab
            continue
        _close(out[j, :n_out], dy[lo:hi].float().t() @ x[lo:hi].float())
