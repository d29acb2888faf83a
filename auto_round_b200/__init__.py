"""auto_round_b200 -- H100-native (sm_90a) engine for the AutoRound block-wise SignRound calibration path.

Public surface mirrors the reference for this path only: `AutoRound(...).quantize()/quantize_and_save()`,
`QuantizationScheme` presets, the `auto_round` checkpoint format.  Compute is hand-written CUDA behind the C ABI
in include/ar_b200.h; PyTorch is used for memory, streams, autograd plumbing of the non-linear block ops and NCCL.
"""
from .schemes import PRESETS, QuantizationScheme, parse_scheme  # noqa: F401

__version__ = "0.1.0"


def __getattr__(name):
    # lazy: importing the package must not require a GPU or the built library
    import importlib
    if name == "AutoRound":
        return importlib.import_module(".autoround", __name__).AutoRound
    if name == "SignRoundQuantizer":
        return importlib.import_module(".quantizer", __name__).SignRoundQuantizer
    if name in ("ops", "export", "quantizer", "autoround", "wrapper", "build", "_lib", "parallel"):
        return importlib.import_module("." + name, __name__)
    raise AttributeError(name)
