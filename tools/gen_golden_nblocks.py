"""Fixtures for `nblocks=2`: the unmodified reference's `AutoRound(..., nblocks=2).quantize()` on a 3-layer tiny Llama, so the
blocks are tuned as the groups [0, 1] and [2].  Writes tests/golden/block_nblocks2_<scheme>.pt with the layout of
oracle/gen_golden.py's block_*.pt fixtures, one record per group: the group's inputs, kwargs, FP outputs, label ids,
state dict (keys `layers.<j>.…`), sampled batches, per-iteration losses, the best iteration and the final qdq weight /
scale / zp of every layer (block-relative names `layers.<j>.…`).

    python tools/gen_golden_nblocks.py

Needs the reference checkout that oracle/ref_shim.py imports; the fixtures it writes are plain tensors.

The reference's public constructor files `nblocks` under its SignRoundConfig, which its compressor never reads: its
`BaseOrchestrator.nblocks` stays 1 and `AutoRound(..., nblocks=2)` tunes block by block.  Its group path (the
orchestrator's `nblocks > 1` branch) runs only when that attribute is set, so this script sets it after construction."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import gen_golden as G  # noqa: E402
from oracle.ref_shim import import_reference  # noqa: E402

SCHEMES = {
    "w4a16_sym_g32": dict(scheme="W4A16", group_size=32),
    "w2a16_asym_g32": dict(scheme="W2A16", group_size=32, sym=False),
}


def best_iter(group) -> int:
    """The reference keeps the first iteration whose loss.item() / num_elm is strictly below every earlier one."""
    masks = [(ids != -100) for ids in group["input_ids"]]
    best, at = float("inf"), 0
    for it, (loss, batch) in enumerate(zip(group["losses"], group["batches"])):
        num_elm = sum(int(masks[i].sum()) for i in batch) or 1
        if loss / num_elm < best:
            best, at = loss / num_elm, it
    return at


def main():
    import_reference()
    from auto_round.compressors.base import BaseOrchestrator

    orig_init = BaseOrchestrator.__init__

    def init_with_nblocks(self, *a, **k):
        orig_init(self, *a, **k)
        self.nblocks = 2

    BaseOrchestrator.__init__ = init_with_nblocks
    for tag, kw in SCHEMES.items():
        rec = G.gen_block(f"nblocks2_{tag}", dict(kw, nblocks=2), model_factory=lambda: G.tiny_llama(layers=3), save=False)
        rec["nblocks"] = 2
        for g in rec["blocks"]:
            g["best_iter"] = best_iter(g)
        path = os.path.join(G.GOLDEN, f"block_nblocks2_{tag}.pt")
        torch.save(rec, path)
        print(f"{os.path.basename(path)}: {len(rec['blocks'])} groups, layers per group",
              [len(g["layers"]) for g in rec["blocks"]], "best_iter", [g["best_iter"] for g in rec["blocks"]])


if __name__ == "__main__":
    main()
