"""ar_pack_awq / ar_unpack_awq on the GPU: bit-exact against the reference's WQLinear_GEMM.from_linear outputs
(tests/golden/pack_awq.pt) and against the CPU oracle (oracle/pack_awq.py) at tile edges and at one Llama-3-8B shape."""
import ctypes
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("CUDA device required", allow_module_level=True)

from auto_round_b200 import _lib, ops  # noqa: E402
from oracle import pack_awq as A  # noqa: E402

DEV = torch.device("cuda", 0)


def _gpu_pack(wq, scale, zp, g):
    if isinstance(zp, torch.Tensor):
        return ops.pack_awq(wq.to(DEV), scale.to(DEV), zp.to(DEV).contiguous(), g)
    return ops.pack_awq(wq.to(DEV), scale.to(DEV), None, g, zp_const=int(zp))


def _assert_same(got, want, what):
    for key, t in zip(("qweight", "qzeros", "scales"), got):
        assert t.dtype == want[key].dtype and tuple(t.shape) == tuple(want[key].shape), (what, key)
        assert torch.equal(t.cpu(), want[key]), (what, key)


def _asym_qdq(n, k, g, seed, tuned=True):
    """A weight the int-asym fake-quant kernel produced, with its fp16 scales and fp32 zero-points [N, G]."""
    gen = torch.Generator().manual_seed(seed)
    w = (torch.randn(n, k, generator=gen) * 0.03).bfloat16()
    w[0, : min(k, 8)] = w[0, : min(k, 8)].abs()
    if n > 4:
        ge = k if g == -1 else g
        w[4, :ge] = w[4, :ge].abs() + 0.01                      # zero-point 0
    spec = ops.make_spec("int_asym", 4, g, n, k)
    v = ((torch.rand(n, spec.kpad, generator=gen) - 0.5).to(DEV)) if tuned else None
    wq, scale, zp = ops.qdq_fwd(spec, w.to(DEV), v, want_scale=True)
    return wq, scale.reshape(n, -1).contiguous(), zp.reshape(n, -1).contiguous()


def test_fixtures_bit_exact(golden_dir):
    golden = torch.load(os.path.join(golden_dir, "pack_awq.pt"), weights_only=False)
    assert len(golden) == 5
    for name, rec in golden.items():
        _assert_same(_gpu_pack(rec["wq"], rec["scale"], rec["zp"], rec["group_size"]), rec, name)


@pytest.mark.parametrize("n", [8, 24, 128, 4096 + 8])
@pytest.mark.parametrize("kg", [(32, 32), (96, 32), (64, 64), (192, 64), (128, 128), (384, 128), (136, -1), (200, -1)])
def test_tile_edges_vs_oracle(n, kg):
    k, g = kg
    wq, scale, zp = _asym_qdq(n, k, g, seed=n * 1000 + k)
    want = A.pack_awq(wq.cpu(), scale.cpu(), zp.cpu(), g)
    _assert_same(ops.pack_awq(wq, scale, zp, g), want, (n, k, g))
    assert int((zp == 0).sum()) > 0 or n <= 4
    # symmetric: no zero-point tensor, the constant in every nibble
    spec = ops.make_spec("int_sym", 4, g, n, k)
    wqs, ss, _ = ops.qdq_fwd(spec, wq, want_scale=True)
    ss = ss.reshape(n, -1).contiguous()
    _assert_same(ops.pack_awq(wqs, ss, None, g, zp_const=8), A.pack_awq(wqs.cpu(), ss.cpu(), 8, g), ("sym", n, k, g))


def test_llama3_8b_down_proj_shape_vs_oracle():
    n, k, g = 4096, 14336, 128
    wq, scale, zp = _asym_qdq(n, k, g, seed=11)
    _assert_same(ops.pack_awq(wq, scale, zp, g), A.pack_awq(wq.cpu(), scale.cpu(), zp.cpu(), g), (n, k, g))


@pytest.mark.parametrize("shape", [(64, 256, 128), (24, 96, 32), (520, 320, 64), (40, 160, -1)])
def test_round_trip_returns_the_fake_quant_weight(shape):
    n, k, g = shape
    wq, scale, zp = _asym_qdq(n, k, g, seed=5)
    qw, qz, st = ops.pack_awq(wq, scale, zp, g)
    back, codes = ops.unpack_awq(qw, qz, st, n, k, g, want_codes=True)
    assert torch.equal(back, wq)
    ocodes, _ = A.unpack_awq(qw.cpu(), qz.cpu(), st.cpu(), g)
    assert torch.equal(codes.cpu(), ocodes) and int(codes.min()) >= 0 and int(codes.max()) <= 15


def test_shape_errors():
    lib = _lib.load()
    wq = torch.zeros(12, 64, dtype=torch.bfloat16, device=DEV)
    sc = torch.ones(12, 2, dtype=torch.float16, device=DEV)
    out = torch.zeros(64 * 2, dtype=torch.int32, device=DEV)
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    rc = lib.ar_pack_awq(p(wq), p(sc), None, 8, 12, 64, 32, p(out), p(out), p(out), None)
    assert rc == -1 and b"out_features (12) shape mismatch" in lib.ar_last_error()
    rc = lib.ar_pack_awq(p(wq), p(sc), None, 8, 16, 48, 32, p(out), p(out), p(out), None)
    assert rc == -1 and b"in_features (48) shape mismatch" in lib.ar_last_error()
    with pytest.raises(ValueError, match=r"out_features \(12\) shape mismatch"):
        ops.pack_awq(wq, sc, None, 32, zp_const=8)
    with pytest.raises(ValueError, match=r"in_features \(48\) shape mismatch"):
        ops.pack_awq(torch.zeros(16, 48, dtype=torch.bfloat16, device=DEV), sc, None, 32, zp_const=8)
