"""CPU oracle of the reference's un-fused MoE experts.

TEST INFRASTRUCTURE ONLY (see oracle/qdq.py header).  Restates, in plain torch on the CPU:
  * auto_round/modeling/fused_moe/replace_modules.py + moe_experts_interface.py:120-171   fused 3-D expert parameters
    (`gate_up_proj [E, 2I, H]`, `down_proj [E, H, I]`) -> per-expert nn.Linear containers "0".."E-1"
  * auto_round/modeling/fused_moe/moe_experts_interface.py:173-260 (`linear_loop_experts_forward` /
    `_run_experts_with_routes`): loop over the experts, gather the (token, slot) pairs routed to each, run its three
    linears, scale by the routing weight, sum the k slots per token.
Used by tests/test_oracle_golden.py to replay a reference Mixtral tuning run bit-for-bit (tests/golden/block_mixtral_mxfp4.pt)
and by the GPU parity tests as the reference the product's grouped wgmma path (auto_round_b200/moe.py) is checked against.
The product never imports this module."""
import torch
import torch.nn as nn


class _Expert(nn.Module):
    def __init__(self, gate: nn.Linear, up: nn.Linear, down: nn.Linear):
        super().__init__()
        self.gate_proj, self.up_proj, self.down_proj = gate, up, down


class LoopExperts(nn.Module):
    def __init__(self, fused: nn.Module):
        super().__init__()
        gu, dn = fused.gate_up_proj.data, fused.down_proj.data
        e, two_i, h = gu.shape
        inter = two_i // 2
        self.num_experts, self.act_fn = e, fused.act_fn
        for i in range(e):
            gate = nn.Linear(h, inter, bias=False, device=gu.device, dtype=gu.dtype)
            up = nn.Linear(h, inter, bias=False, device=gu.device, dtype=gu.dtype)
            down = nn.Linear(inter, h, bias=False, device=gu.device, dtype=gu.dtype)
            gate.weight.data.copy_(gu[i, :inter])
            up.weight.data.copy_(gu[i, inter:])
            down.weight.data.copy_(dn[i])
            self.add_module(str(i), _Expert(gate, up, down))

    def forward(self, hidden_states, top_k_index, top_k_weights):
        lead = hidden_states.shape
        x = hidden_states.reshape(-1, lead[-1])
        ids = top_k_index.reshape(x.shape[0], -1)
        k = ids.shape[1]
        w = top_k_weights.reshape(-1).to(x.dtype)
        flat_ids = ids.reshape(-1)
        pair_token = torch.arange(x.shape[0], device=x.device).repeat_interleave(k)
        x_pairs = x[pair_token]
        y_pairs = torch.zeros_like(x_pairs)
        for e in range(self.num_experts):
            sel = (flat_ids == e).nonzero().reshape(-1)
            if sel.numel() == 0:
                continue
            ex = getattr(self, str(e))
            xe = x_pairs.index_select(0, sel)
            y_pairs.index_copy_(0, sel, ex.down_proj(self.act_fn(ex.gate_proj(xe)) * ex.up_proj(xe)).to(y_pairs.dtype))
        out = (y_pairs * w.unsqueeze(-1)).view(x.shape[0], k, -1).sum(dim=1)
        return out.view(lead)


def unfuse_experts_cpu(block: nn.Module) -> int:
    n = 0
    for name, m in list(block.named_modules()):
        gu, dn = getattr(m, "gate_up_proj", None), getattr(m, "down_proj", None)
        if isinstance(gu, nn.Parameter) and isinstance(dn, nn.Parameter) and gu.dim() == 3 and dn.dim() == 3 and hasattr(m, "act_fn"):
            parent = block
            parts = name.split(".")
            for p in parts[:-1]:
                parent = getattr(parent, p)
            setattr(parent, parts[-1], LoopExperts(m))
            n += 1
    return n
