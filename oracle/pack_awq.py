"""CPU oracle for the AWQ "GEMM" layout (4 bit), torch integer work.

TEST INFRASTRUCTURE ONLY (see oracle/qdq.py header).  Restates, from the layout they produce:
  * auto_round/export/export_to_awq/utils.py:197-273  WQLinear_GEMM.from_linear  (pack)
  * auto_round/export/export_to_awq/utils.py:45-101   unpack_awq / reverse_awq_order / dequantize_gemm  (unpack)
Pinned by tests/golden/pack_awq.pt (outputs of the reference).

Layout: qweight i32 [K, N/8], word j of row k = sum_i code[8j+i, k] << 4*ORDER[i]; qzeros i32 [G, N/8] packs the
zero-points of the same eight columns the same way (a symmetric layer: the constant in every nibble); scales fp16 [G, N].
"""
from __future__ import annotations

import torch

from .pack import int_codes

ORDER = (0, 4, 1, 5, 2, 6, 3, 7)          # nibble position of column 8j+i


def _pack_cols(vals: torch.Tensor) -> torch.Tensor:
    """int32 [R, N] -> int32 [R, N/8]: eight consecutive columns per word; the shifted int32 lanes are summed (wrapping),
    which is an OR for in-range nibbles."""
    r, n = vals.shape
    sh = torch.tensor(ORDER, dtype=torch.int32) * 4
    return (vals.to(torch.int32).reshape(r, n // 8, 8) << sh).sum(dim=-1).to(torch.int32)


def check_shapes(n: int, k: int, group_size: int) -> int:
    """The reference's preconditions (utils.py:150-158) -> effective group size."""
    g = k if group_size == -1 else group_size
    if k % g != 0:
        raise ValueError(f"in_features ({k}) shape mismatch")
    if n % 8 != 0:
        raise ValueError(f"out_features ({n}) shape mismatch")
    return g


def pack_awq(w_qdq: torch.Tensor, scale: torch.Tensor, zp, group_size: int) -> dict:
    """w_qdq [N,K], scale [N,G], zp fp32 [N,G] or a python int -> dict(qweight, qzeros, scales)."""
    n, k = w_qdq.shape
    g = check_shapes(n, k, group_size)
    codes = torch.from_numpy(int_codes(w_qdq, scale, zp, g))                     # [N, K] = round(W / s + zp)
    if isinstance(zp, torch.Tensor):
        qzeros = _pack_cols(zp.t().contiguous().to(torch.int32))
    else:
        word = 0
        for i in range(8):
            word |= int(zp) << (4 * i)
        word = word - (1 << 32) if word >= (1 << 31) else word
        qzeros = torch.full((k // g, n // 8), word, dtype=torch.int32)
    return {"qweight": _pack_cols(codes.t().contiguous()), "qzeros": qzeros,
            "scales": scale.t().contiguous().to(torch.float16)}


def unpack_cols(words: torch.Tensor) -> torch.Tensor:
    """int32 [R, N/8] -> nibbles int32 [R, N] in column order."""
    sh = torch.tensor(ORDER, dtype=torch.int32) * 4
    return ((words[:, :, None] >> sh) & 15).reshape(words.shape[0], -1)


def unpack_awq(qweight: torch.Tensor, qzeros: torch.Tensor, scales: torch.Tensor, group_size: int):
    """-> (codes int32 [N,K], W' fp32 [N,K] = (code - zero) * scale)."""
    k = qweight.shape[0]
    g = k if group_size == -1 else group_size
    codes = unpack_cols(qweight)                                                  # [K, N]
    zeros = unpack_cols(qzeros).repeat_interleave(g, dim=0)
    w = (codes - zeros).to(torch.float32) * scales.to(torch.float32).repeat_interleave(g, dim=0)
    return codes.t().contiguous(), w.t().contiguous()
