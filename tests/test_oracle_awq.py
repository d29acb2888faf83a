"""Pins the CPU oracle of the AWQ GEMM layout (oracle/pack_awq.py) against tests/golden/pack_awq.pt, written by the
unmodified reference's WQLinear_GEMM.from_linear (oracle/gen_golden_formats.py)."""
import os

import pytest
import torch

from oracle import pack_awq as A

CASES = ("asym_g128", "asym_g32", "sym_g128", "asym_gm1", "asym_g64_bias")


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(os.path.join(golden_dir, "pack_awq.pt"), weights_only=False)


@pytest.mark.parametrize("case", CASES)
def test_pack_matches_reference(golden, case):
    rec = golden[case]
    out = A.pack_awq(rec["wq"], rec["scale"], rec["zp"], rec["group_size"])
    for key in ("qweight", "qzeros", "scales"):
        assert out[key].dtype == rec[key].dtype and tuple(out[key].shape) == tuple(rec[key].shape), key
        assert torch.equal(out[key], rec[key]), key


@pytest.mark.parametrize("case", CASES)
def test_unpack_returns_the_codes_and_the_weight(golden, case):
    rec = golden[case]
    codes, w = A.unpack_awq(rec["qweight"], rec["qzeros"], rec["scales"], rec["group_size"])
    from oracle.pack import int_codes
    assert torch.equal(codes, torch.from_numpy(int_codes(rec["wq"], rec["scale"], rec["zp"], rec["group_size"])))
    assert codes.min() >= 0 and codes.max() <= 15
    assert torch.equal(w.to(torch.bfloat16), rec["wq"])          # the fake-quant weight is (code - zero) * scale


def test_fixture_has_zero_point_zero_groups(golden):
    """A group without negative weights has zero-point 0: the lowest nibble value must survive the packing."""
    assert int((golden["asym_g128"]["zp"] == 0).sum()) > 0
    assert int((A.unpack_cols(golden["asym_g128"]["qzeros"]) == 0).sum()) > 0


def test_nibble_order_literal():
    """Columns 0..7 hold the codes 0..7: column i lands at nibble [0, 4, 1, 5, 2, 6, 3, 7][i], so the nibbles read
    from the top are 7 5 3 1 6 4 2 0."""
    vals = torch.arange(8, dtype=torch.int32).reshape(1, 8)
    assert A._pack_cols(vals).tolist() == [[0x75316420]]
    assert A.unpack_cols(torch.tensor([[0x75316420]], dtype=torch.int32)).tolist() == [list(range(8))]
    # a high nibble of 8..15 in the top position sets the sign bit of the int32 word
    top = torch.tensor([[0, 0, 0, 0, 0, 0, 0, 15]], dtype=torch.int32)
    assert A._pack_cols(top).tolist() == [[-(1 << 28)]]


def test_shape_preconditions():
    w = torch.zeros(12, 64, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match=r"out_features \(12\) shape mismatch"):
        A.pack_awq(w, torch.ones(12, 2, dtype=torch.float16), 8, 32)
    w = torch.zeros(16, 48, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match=r"in_features \(48\) shape mismatch"):
        A.pack_awq(w, torch.ones(16, 2, dtype=torch.float16), 8, 32)
