"""Quantisation schemes -- host-side mirror of auto_round/schemes.py:197-210 (QuantizationScheme) and the
presets used by the hot path (:538-707).  Only weight-only tuning of int (sym/asym), MXFP4 and NVFP4 weights is
in scope; activation quantisation fields are carried for config fidelity and rejected if they would change math.
"""
from __future__ import annotations

from dataclasses import asdict, dataclass, fields, replace
from typing import Optional


@dataclass
class QuantizationScheme:
    bits: int = 4
    group_size: int = 128
    sym: bool = True
    data_type: str = "int"
    act_bits: Optional[int] = 16
    act_group_size: Optional[int] = None
    act_sym: Optional[bool] = None
    act_data_type: Optional[str] = None
    act_dynamic: Optional[bool] = None
    super_bits: Optional[int] = None
    super_group_size: Optional[int] = None

    @classmethod
    def from_dict(cls, d: dict) -> "QuantizationScheme":
        names = {f.name for f in fields(cls)}
        return cls(**{k: v for k, v in d.items() if k in names})

    def to_dict(self) -> dict:
        return asdict(self)

    # --- the fake-quant function this scheme resolves to (auto_round/data_type/utils.py:105-176)
    @property
    def qdq_name(self) -> str:
        dt = self.data_type
        if dt == "int":
            return "int_sym" if self.sym else "int_asym"
        if dt in ("mx_fp", "mx_fp4") and self.bits == 4:
            return "mx_fp4"
        if dt in ("nv_fp", "nv_fp4") and self.bits == 4:
            return "nv_fp4"
        raise NotImplementedError(f"data_type={dt!r} bits={self.bits} is outside the H100 hot path "
                                  "(int 2/3/4/8, mx_fp4, nv_fp4)")

    @property
    def weight_only(self) -> bool:
        return self.act_bits is None or self.act_bits >= 16


PRESETS = {
    "W4A16": dict(bits=4, sym=True, group_size=128, data_type="int", act_bits=16),
    "W2A16": dict(bits=2, sym=True, group_size=128, data_type="int", act_bits=16),
    "W2A16G64": dict(bits=2, sym=True, group_size=64, data_type="int", act_bits=16),
    "W2A16G32": dict(bits=2, sym=True, group_size=32, data_type="int", act_bits=16),
    "W3A16": dict(bits=3, sym=True, group_size=128, data_type="int", act_bits=16),
    "W8A16": dict(bits=8, sym=True, group_size=128, data_type="int", act_bits=16),
    "MXFP4": dict(bits=4, group_size=32, data_type="mx_fp", act_bits=4, act_data_type="mx_fp", act_group_size=32,
                  act_sym=True, act_dynamic=True),
    "NVFP4": dict(bits=4, group_size=16, data_type="nv_fp", act_bits=4, act_data_type="nv_fp4_with_static_gs",
                  act_group_size=16, act_sym=True, act_dynamic=True),
}

_SCHEME_FIELDS = tuple(f.name for f in fields(QuantizationScheme))


def parse_scheme(scheme, overrides: Optional[dict] = None) -> QuantizationScheme:
    """auto_round/schemes.py:496-535: preset name / dict / QuantizationScheme + per-field keyword overrides."""
    if isinstance(scheme, QuantizationScheme):
        s = replace(scheme)
    elif isinstance(scheme, dict):
        s = QuantizationScheme.from_dict(scheme)
    elif isinstance(scheme, str):
        key = scheme.upper()
        if key not in PRESETS:
            raise ValueError(f"unknown scheme {scheme!r}; supported presets: {sorted(PRESETS)}")
        s = QuantizationScheme.from_dict(PRESETS[key])
    else:
        raise TypeError(f"scheme must be str, dict or QuantizationScheme, got {type(scheme)}")
    for k, v in (overrides or {}).items():
        if k in _SCHEME_FIELDS and v is not None:
            setattr(s, k, v)
    # auto_round/schemes.py:395-422 (_reconcile_bits_and_dtype): a float activation dtype means "not quantised"
    if s.act_data_type in ("float", "fp", "bf16", "fp16") and (s.act_bits is None or s.act_bits >= 16):
        s.act_bits = 16
    if not s.weight_only:
        raise NotImplementedError(
            "activation quantisation (act_bits < 16) is outside the H100 hot path; pass act_bits=16 "
            "(and act_data_type='float' for NVFP4) for weight-only tuning, as BASELINE.json's configs do")
    s.qdq_name  # validates the weight data type
    return s
