"""Crash-resume of the block-sequential tuning run (SURVEY.md 8 f4) -- host-side mirror of auto_round/utils/resume.py.

Activated exactly like the reference: set `AR_RESUME_DIR`.  After every block the run persists
  * the block's RESULT (packed `QuantLinear` buffers, or the qdq weight + scale / zp / global scale of each tuned linear),
  * the two chain values the next block needs verbatim -- the full-precision block outputs (next block's reference input)
    and, with `enable_quanted_input`, the quantised block's outputs (utils/resume.py:8-22 explains why both must be the live
    values, not recomputed ones),
  * a manifest `{signature, completed_blocks}` written atomically (tmp file + os.replace), trusted only when the signature
    (model id, scheme + per-layer config, dataset, nsamples, seqlen, block list) matches and `completed_blocks` is a PREFIX
    of the current block order (utils/resume.py:96-119).
The reference keeps finished blocks in its ShardWriter / offloader directories; this engine has neither, so the per-block
result files live in the resume directory itself.

Everything here is plain torch / json on host tensors: no CUDA, covered by tests/test_resume.py in the CPU tier.
"""
from __future__ import annotations

import hashlib
import json
import os
import tempfile
from pathlib import Path
from typing import Optional

import torch
import torch.nn as nn

MANIFEST = "resume_manifest.json"
Q_INPUT = "resume_q_input.pt"
FP_INPUT = "resume_input_ids.pt"      # the reference's name for the chained full-precision hidden states

_SCALARS = (int, float, bool, str, type(None))


def host_copy(tree):
    """Detached CPU copy of every tensor in a (possibly nested) list / tuple / dict; other leaves pass through."""
    if torch.is_tensor(tree):
        return tree.detach().cpu()
    if isinstance(tree, dict):
        return {key: host_copy(val) for key, val in tree.items()}
    if isinstance(tree, (list, tuple)):
        return type(tree)(map(host_copy, tree))
    return tree


_to_cpu = host_copy


def _write_atomically(target: Path, emit, binary: bool) -> None:
    """Write through a temporary sibling and rename it over `target`, so that a crash never leaves a torn file."""
    handle, scratch = tempfile.mkstemp(dir=str(target.parent), prefix=".tmp_resume_")
    try:
        with os.fdopen(handle, "wb" if binary else "w") as stream:     # a stream, not a path: torch.save names its archive
            emit(stream)                                                # after the path otherwise
        os.replace(scratch, target)
    except BaseException:
        if os.path.exists(scratch):
            os.remove(scratch)
        raise


def _atomic_write_json(path: Path, data: dict) -> None:
    _write_atomically(path, lambda stream: json.dump(data, stream), binary=False)


def _atomic_save(obj, path: Path) -> None:
    _write_atomically(path, lambda stream: torch.save(obj, stream), binary=True)


def _scalar_items(cfg: dict):
    for key in sorted(cfg, key=str):
        if isinstance(cfg[key], _SCALARS):
            yield f"{key}={cfg[key]}"


def layer_config_fingerprint(layer_config) -> str:
    """Same string as utils/resume.py:185-222 builds: per layer (sorted) its scalar settings (sorted), nothing else."""
    if not layer_config:
        return "<no-layer-config>"
    rows = []
    for layer in sorted(layer_config):
        cfg = layer_config[layer]
        cfg = cfg.to_dict() if hasattr(cfg, "to_dict") else cfg
        rows.append(f"{layer}:" + (",".join(_scalar_items(cfg)) if isinstance(cfg, dict) else str(cfg)))
    return ";".join(rows)


def compute_run_signature(model_id: Optional[str], scheme_desc: str, dataset_desc: str, nsamples: int, seqlen: int,
                          block_names: list) -> str:
    """sha256 over the NUL-terminated identifying strings -- the digest utils/resume.py:166-182 produces."""
    fields_ = (model_id or "", scheme_desc, dataset_desc, str(nsamples), str(seqlen), "|".join(block_names))
    return hashlib.sha256(b"".join(f.encode("utf-8") + b"\x00" for f in fields_)).hexdigest()


def dataset_fingerprint(dataset) -> str:
    """Token-tensor datasets have no stable `str()`: hash their contents instead."""
    if dataset is None or isinstance(dataset, str):
        return str(dataset)
    h = hashlib.sha256()
    for t in dataset:
        t = torch.as_tensor(t).detach().to("cpu", torch.int64).contiguous()
        h.update(str(tuple(t.shape)).encode())
        h.update(t.numpy().tobytes())
    return "tokens:" + h.hexdigest()


# ------------------------------------------------------------------------------------------ per-block result snapshot
_LAYER_ATTRS = ("scale", "zp", "weight_global_scale")


def snapshot_block(block: nn.Module) -> dict:
    """Host copy of what tuning changed in `block`: for packed layers every buffer of the QuantLinear holder (plus the
    constructor facts), for unpacked ones the qdq weight and the scale / zp / global-scale attributes."""
    from .export import QuantLinear

    out = {}
    for name, m in block.named_modules():
        if isinstance(m, QuantLinear):
            out[name] = {"kind": "packed", "in_features": m.in_features, "out_features": m.out_features,
                         "buffers": {k: v.detach().cpu() for k, v in m._buffers.items() if v is not None},
                         "non_persistent": sorted(m._non_persistent_buffers_set)}
        elif isinstance(m, nn.Linear) and hasattr(m, "scale"):
            rec = {"kind": "qdq", "weight": m.weight.detach().cpu()}
            for a in _LAYER_ATTRS:
                if hasattr(m, a):
                    rec[a] = _to_cpu(getattr(m, a))
            out[name] = rec
    return out


def restore_block(block: nn.Module, snap: dict, scheme_for) -> list:
    """Inverse of snapshot_block on a freshly loaded (unquantised) `block`.  `scheme_for(name, module)` supplies the
    QuantizationScheme a packed holder is labelled with.  Returns the restored layer names."""
    from .export import QuantLinear
    from .wrapper import set_module

    done = []
    for name, rec in snap.items():
        lin = block.get_submodule(name)
        if rec["kind"] == "packed":
            bias = rec["buffers"].get("bias")
            bufs = {k: v for k, v in rec["buffers"].items() if k != "bias"}
            set_module(block, name, QuantLinear(rec["in_features"], rec["out_features"], scheme_for(name, lin), bufs, bias,
                                                persist_g_idx="g_idx" not in rec.get("non_persistent", ["g_idx"])))
        else:
            lin.weight.data = rec["weight"].to(lin.weight.dtype)
            for a in _LAYER_ATTRS:
                if a in rec:
                    setattr(lin, a, rec[a])
        done.append(name)
    return done


class ResumeState:
    """utils/resume.py:74-164 plus the per-block result files described in the module docstring."""

    def __init__(self, resume_dir: str, signature: str, block_names: list):
        self.dir = Path(resume_dir)
        self.dir.mkdir(parents=True, exist_ok=True)
        self.signature = signature
        self.block_names = list(block_names)
        self.manifest_path = self.dir / MANIFEST
        self.completed_blocks: list = []
        self._load()

    def _block_path(self, name: str) -> Path:
        return self.dir / ("block_" + name.replace("/", "_") + ".pt")

    def _trusted_prefix(self) -> list:
        """The finished blocks a manifest may vouch for: same run signature, a PREFIX of the current block order
        (utils/resume.py:96-119), and every result file still on disk.  Anything else means "start from block 0"."""
        try:
            manifest = json.loads(self.manifest_path.read_text())
        except (OSError, ValueError):
            return []
        if manifest.get("signature") != self.signature:
            return []
        done = list(manifest.get("completed_blocks", []))
        if done != self.block_names[:len(done)]:
            return []
        return done if all(self._block_path(name).exists() for name in done) else []

    def _load(self) -> None:
        self.completed_blocks = self._trusted_prefix()

    @property
    def resume_index(self) -> int:
        return len(self.completed_blocks)

    def _load_tensor(self, name: str):
        p = self.dir / name
        if not self.completed_blocks or not p.exists():
            return None
        try:
            return torch.load(p, map_location="cpu", weights_only=False)
        except Exception:  # noqa: BLE001
            return None

    def load_q_input(self):
        return self._load_tensor(Q_INPUT)

    def load_input_ids(self):
        return self._load_tensor(FP_INPUT)

    def load_block(self, name: str) -> dict:
        return torch.load(self._block_path(name), map_location="cpu", weights_only=False)

    def mark_block_done(self, block_name: str, block_snapshot: dict, q_input, fp_input) -> None:
        expected = self.block_names[len(self.completed_blocks)]
        if block_name != expected:
            raise AssertionError(f"ResumeState.mark_block_done out of order: expected {expected!r}, got {block_name!r}")
        _atomic_save(block_snapshot, self._block_path(block_name))
        qp = self.dir / Q_INPUT
        if q_input is not None:
            _atomic_save(_to_cpu(q_input), qp)
        elif qp.exists():
            qp.unlink()
        _atomic_save(_to_cpu(fp_input), self.dir / FP_INPUT)       # required: the FP reference chain always exists
        self.completed_blocks.append(block_name)
        # the manifest is written LAST: a crash before this line re-does the block instead of skipping it
        _atomic_write_json(self.manifest_path, {"signature": self.signature, "completed_blocks": self.completed_blocks})

    def clear(self) -> None:
        for p in [self.manifest_path, self.dir / Q_INPUT, self.dir / FP_INPUT] + [self._block_path(n) for n in self.block_names]:
            if p.exists():
                try:
                    p.unlink()
                except OSError:
                    pass
        self.completed_blocks = []
