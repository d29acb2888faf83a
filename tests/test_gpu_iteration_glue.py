"""The non-GEMM kernels of one sign-SGD iteration at production shapes: block glue (csrc/ar_block.cu), MoE glue
(csrc/ar_moe.cu), the outlier-suppressed loss and its top-k (csrc/ar_outlier.cu) and the loop schedule (csrc/ar_loop.cu).

Every reference is a restatement of the operation in torch, run on the GPU, of one of two kinds:
  * exact: the same fp32 operations in the same order.  bf16 x bf16 products are exact in fp32 and the library is built
    with -fmad=false, so the outputs must match bit for bit;
  * fp64: where the kernel is free to choose its reduction order, with a bound derived from that order (stated per test).

`ulp` below is the bf16 spacing at a value: 2^(floor(log2|v|) - 7), and 2^-133 (the subnormal spacing) at and below
2^-126.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("CUDA device required", allow_module_level=True)

from auto_round_b200 import _lib, fused, ops  # noqa: E402
from oracle import signround as S  # noqa: E402

DEV = "cuda"


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _bits(t):
    return t.view(torch.int16)


def _bit_equal(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _ulp(v):
    """bf16 spacing at each value of the fp64 tensor `v`."""
    _, e = torch.frexp(v)
    e = torch.where(v == 0, torch.full_like(e, -125), e)
    return torch.ldexp(torch.ones_like(v), (e - 8).clamp(min=-133))


def _check(rc, what):
    _lib.check(rc, what)


# ------------------------------------------------------------------------------------------------------ RMSNorm
RMS_SHAPES = [(rows, h) for h in (72, 512, 2560, 3584, 4096, 5120, 8192) for rows in (1, 37)] + [(16384, 4096)]


def _rms_inputs(rows, hidden, seed):
    gen = _gen(seed)
    x = torch.randn(rows, hidden, device=DEV, generator=gen)
    if rows > 2:
        x[1] = 0.0                                             # rstd = 1/sqrt(eps)
        x[2] *= 1e4 / x[2].abs().max()                         # |x| up to 1e4
        x[rows - 1] *= 1e-3
    w = torch.rand(hidden, device=DEV, generator=gen) * 2.0 - 0.5   # trained norm weights can be negative
    dy = torch.randn(rows, hidden, device=DEV, generator=gen)
    old = torch.randn(rows, hidden, device=DEV, generator=gen)
    return x.bfloat16(), w.bfloat16(), dy.bfloat16(), old.bfloat16()


@pytest.mark.parametrize("eps", [1e-5, 1e-6])
@pytest.mark.parametrize("rows,hidden", RMS_SHAPES)
def test_rmsnorm(rows, hidden, eps):
    """hidden 72 runs one partial warp (VPT 1), 2560 / 3584 / 4096 run VPT 2 (3584 with a partial second vector),
    5120 / 8192 run VPT 4.

    rstd: within 2^-20 relative of the fp64 1/sqrt(mean(x^2) + eps).  The fp32 sum of positive terms runs at most
    8*VPT + 5 + 8 additions deep; its round-to-nearest errors add as a random walk whose spread is far inside 2^-21
    (the linear worst case, every rounding in one direction, would be about 2^-19.4), and rsqrtf adds at most 2 ulp
    (2^-22).
    Forward: y == bf16(w * bf16(x * r)) bit for bit with the kernel's own r.
    Forward vs HF LlamaRMSNorm (eager, on the GPU): HF's r comes from another fp32 reduction order and may differ in the
    last bits, so the inner n = bf16(x * r) may round to the neighbouring bf16 value (rare).  Where the two n agree, y is
    bit-identical; where they differ, they are one step apart and the product with w carries that step:
        |y - y_hf| <= |w| * |n - n_hf| + ulp(max(|y|, |y_hf|))
    which is 1 ulp where n == n_hf and can reach about 2 ulp (n at the bottom of its binade, y at the top of its own)
    where the inner rounding flipped.
    Backward (fp64, with the kernel's r):  dn = bf16(dy*w), n = x*r, ref = r*(dn - n*mean(dn*n)),
        |dx - ref| <= ulp(ref) + 2^-16 * r * |n| * mean|dn*n|
    (one bf16 rounding plus the fp32 dot product over 8*VPT sequential terms and the block tree).
    accumulate=1: dx == bf16(float(dx0) + float(old)) bit for bit, dx0 the accumulate=0 output."""
    from transformers.models.llama.modeling_llama import LlamaRMSNorm

    x, w, dy, old = _rms_inputs(rows, hidden, seed=rows * 7 + hidden)
    y, rstd = ops.rmsnorm_fwd(x, w, eps)

    r64 = 1.0 / torch.sqrt(x.double().pow(2).mean(-1) + eps)
    rel = ((rstd.double() - r64).abs() / r64).max()
    assert float(rel) <= 2.0 ** -20, f"rstd off by {float(rel):.3e} relative"

    r = rstd[:, None]
    assert _bit_equal(y, (w.float() * (x.float() * r).bfloat16().float()).bfloat16())

    hf = LlamaRMSNorm(hidden, eps=eps).to(DEV).to(torch.bfloat16)
    with torch.no_grad():
        hf.weight.copy_(w)
        y_hf = hf(x)
    xf = x.float()
    n_hf = (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)).bfloat16()
    assert _bit_equal(y_hf, w * n_hf)                           # HF's rounding points, restated
    n_k = (xf * r).bfloat16()
    same_n = _bits(n_k) == _bits(n_hf)
    assert bool((_bits(y)[same_n] == _bits(y_hf)[same_n]).all())
    gap = (n_k.double() - n_hf.double()).abs()
    assert bool((gap <= _ulp(n_k.double())).all())
    y64, h64 = y.double(), y_hf.double()
    bound = w.double().abs() * gap + _ulp(torch.maximum(y64.abs(), h64.abs()))
    assert bool(((y64 - h64).abs() <= bound).all())
    same = float((_bits(y) == _bits(y_hf)).double().mean())
    within = float(((y64 - h64).abs() <= _ulp(torch.maximum(y64.abs(), h64.abs()))).double().mean())
    print(f"rmsnorm vs HF LlamaRMSNorm rows={rows} hidden={hidden} eps={eps}: {y.numel()} elements, "
          f"{same:.8f} bit-identical, {within:.8f} within 1 ulp, {int((~same_n).sum())} inner roundings differ")

    dx = ops.rmsnorm_bwd(dy, x, w, rstd)
    r = rstd.double()[:, None]
    dn = (dy.float() * w.float()).bfloat16().double()
    n = x.double() * r
    ref = r * (dn - n * (dn * n).mean(-1, keepdim=True))
    bound = _ulp(ref) + 2.0 ** -16 * r * n.abs() * (dn * n).abs().mean(-1, keepdim=True)
    err = (dx.double() - ref).abs()
    assert bool((err <= bound).all()), f"rmsnorm bwd: worst error {float((err / bound).max()):.3f} of the bound"

    acc = old.clone()
    _check(_lib.load().ar_rmsnorm_bwd(ops._p(dy), ops._p(x), ops._p(w), ops._p(rstd), rows, hidden, ops._p(acc), 1,
                                      ops._stream()), "ar_rmsnorm_bwd")
    assert _bit_equal(acc, (dx.float() + old.float()).bfloat16())


# --------------------------------------------------------------------------------------------------------- RoPE
ROPE_SHAPES = [(2, 2048, 32, 128), (2, 2048, 8, 128), (1, 333, 28, 128), (3, 48, 4, 64)]


def _rope_tables(b, s, d, table_batch, split, gen):
    """cos/sin [table_batch, S, D] bf16.  'hf': LlamaRotaryEmbedding's cat(f, f) tables (each sample of a batch table at
    its own positions); 'split': arbitrary full-width tables whose halves differ (c1 != c2, s1 != s2)."""
    if split:
        cos = torch.rand(table_batch, s, d, device=DEV, generator=gen) * 2 - 1
        sin = torch.rand(table_batch, s, d, device=DEV, generator=gen) * 2 - 1
        return cos.bfloat16(), sin.bfloat16()
    inv_freq = 1.0 / (500000.0 ** (torch.arange(0, d, 2, device=DEV, dtype=torch.float32) / d))
    pos = torch.arange(s, device=DEV, dtype=torch.float32)[None].repeat(table_batch, 1)
    pos = pos + torch.randint(0, 4096, (table_batch, 1), device=DEV, generator=gen).float()   # per-sample offsets
    freqs = pos[:, :, None] * inv_freq[None, None, :]
    emb = torch.cat([freqs, freqs], -1)
    return emb.cos().bfloat16(), emb.sin().bfloat16()


@pytest.mark.parametrize("split", [False, True], ids=["hf_table", "split_halves"])
@pytest.mark.parametrize("per_sample", [False, True], ids=["table_batch_1", "table_batch_B"])
@pytest.mark.parametrize("b,s,h,d", ROPE_SHAPES)
def test_rope(b, s, h, d, per_sample, split):
    """Forward: bit-equal to HF apply_rotary_pos_emb (called eagerly) on the [B,H,S,D] view of [B,S,H,D] memory, directly
    and through the patched helper of fused.py (q and a GQA k with fewer heads).
    Backward: bit-equal to bf16(g1*c1 + g2*s2) | bf16(g2*c2 - g1*s1) (exact products, one fp32 add, one rounding),
    directly and through fused._RopeFn's autograd, and within 1 ulp of the fp64 transpose (autograd of the fp64 forward)."""
    from transformers.models.llama import modeling_llama as ml

    gen = _gen(b * 1000 + s + h + d)
    tb = b if per_sample else 1
    cos, sin = _rope_tables(b, s, d, tb, split, gen)
    hk = max(1, h // 4)
    x = torch.randn(b, s, h, d, device=DEV, generator=gen).bfloat16()
    xk = torch.randn(b, s, hk, d, device=DEV, generator=gen).bfloat16()
    q_v, k_v = x.transpose(1, 2), xk.transpose(1, 2)            # what the attention module hands to the helper

    ref_q, ref_k = ml.apply_rotary_pos_emb(q_v, k_v, cos, sin)
    assert _bit_equal(ops.rope(x, cos, sin).transpose(1, 2), ref_q)
    assert _bit_equal(ops.rope(xk, cos, sin).transpose(1, 2), ref_k)
    pq, pk = fused._make_fused_rope(ml.apply_rotary_pos_emb)(q_v, k_v, cos, sin)
    assert _bit_equal(pq, ref_q) and _bit_equal(pk, ref_k)

    g = torch.randn(b, s, h, d, device=DEV, generator=gen).bfloat16()
    c, sn = cos.float()[:, :, None, :], sin.float()[:, :, None, :]
    half = d // 2
    c1, c2, s1, s2 = c[..., :half], c[..., half:], sn[..., :half], sn[..., half:]
    g1, g2 = g.float()[..., :half], g.float()[..., half:]
    want = torch.cat([g1 * c1 + g2 * s2, g2 * c2 - g1 * s1], -1).bfloat16()
    dx = ops.rope(g, cos, sin, backward=True)
    assert _bit_equal(dx, want)

    leaf = x.clone().requires_grad_(True)
    fused._RopeFn.apply(leaf.transpose(1, 2), cos, sin).backward(g.transpose(1, 2))
    assert _bit_equal(leaf.grad, want)

    x64 = torch.zeros(b, s, h, d, dtype=torch.float64, device=DEV, requires_grad=True)
    c64, s64 = cos.double()[:, :, None, :], sin.double()[:, :, None, :]
    x1, x2 = x64[..., :half], x64[..., half:]
    out = torch.cat([x1 * c64[..., :half] - x2 * s64[..., :half], x2 * c64[..., half:] + x1 * s64[..., half:]], -1)
    out.backward(g.double())
    t = x64.grad
    assert bool(((dx.double() - t).abs() <= _ulp(t)).all())


# ------------------------------------------------------------------------------------------------------- SwiGLU
SPECIAL_G = [0.0, -0.0, 1e-3, -1e-3, 20.0, -20.0, 90.0, -90.0]


@pytest.mark.parametrize("numel", [8, 2048 * 14336, 4096 * 18944, 16384 * 14336])
def test_swiglu(numel):
    """16384*14336 (235 M elements) runs the grid-stride loop past the sm_count*16 block cap.  g holds +-0, +-1e-3, +-20
    and +-90 (at g = -90, expf(-g) overflows: silu is -0 and the sigmoid 0).
    Forward: bit-equal to F.silu(g) * u.   du: bit-equal to bf16(dh * F.silu(g)).
    dg (fp64):  ref = bf16(dh*u) * s*(1 + g*(1 - s)),  |dg - ref| <= ulp(ref) + |bf16(dh*u)| * (1 + |g|) * 2^-126.
    The second term is fp32's range: below g = -88.7 the fp32 sigmoid is 0 where the exact one is under 2^-127, and
    just above that it is subnormal; elsewhere the fp32 chain stays well inside the bf16 rounding."""
    gen = _gen(numel % 100003)
    g = (torch.randn(numel, device=DEV, generator=gen) * 3).bfloat16()
    g[-8:] = torch.tensor(SPECIAL_G[::-1], device=DEV).bfloat16()
    g[:8] = torch.tensor(SPECIAL_G, device=DEV).bfloat16()
    u = torch.randn(numel, device=DEV, generator=gen).bfloat16()
    dh = torch.randn(numel, device=DEV, generator=gen).bfloat16()
    assert int(_bits(F.silu(g[7:8]))) == -0x8000                # g = -90: silu is -0

    h = ops.swiglu_fwd(g, u)
    assert _bit_equal(h, F.silu(g) * u)
    del h
    dg, du = ops.swiglu_bwd(dh, g, u)
    assert _bit_equal(du, dh * F.silu(g))
    chunk = 1 << 25
    for i in range(0, numel, chunk):
        gd = g[i:i + chunk].double()
        s = torch.sigmoid(gd)
        dhu = (dh[i:i + chunk].float() * u[i:i + chunk].float()).bfloat16().double()
        ref = dhu * s * (1 + gd * (1 - s))
        bound = _ulp(ref) + dhu.abs() * (1 + gd.abs()) * 2.0 ** -126
        err = (dg[i:i + chunk].double() - ref).abs()
        assert bool((err <= bound).all()), f"swiglu dg: worst error {float((err / bound).max()):.3f} of the bound"


# ------------------------------------------------------------------------------------------------------ MoE glue
# (tokens, experts, topk, e_begin, e_local, cols): one GPU and expert-parallel ranks (pairs outside [e_begin, e_begin +
# e_local) have no row), Mixtral's hidden 4096 and intermediate 14336, topk 1 / 2 / 8
MOE_CASES = [(300, 4, 1, 0, 4, 64), (2048, 8, 2, 0, 8, 4096), (1024, 8, 2, 0, 8, 14336), (512, 64, 8, 32, 32, 4096),
             (256, 16, 8, 4, 8, 14336), (200, 8, 2, 2, 3, 64)]


def _moe_setup(tokens, e, topk, e_begin, e_local, seed):
    gen = _gen(seed)
    logits = torch.randn(tokens, e, device=DEV, generator=gen)
    w, idx = torch.topk(torch.softmax(logits, -1), topk, dim=-1)
    pair_w = (w / w.sum(-1, keepdim=True)).bfloat16().reshape(-1).contiguous()
    route = ops.moe_route(ops.MoeRoute(tokens * topk, e_local, DEV), idx.reshape(-1).contiguous(), e_begin)
    return route, pair_w, gen


@pytest.mark.parametrize("weighted", [False, True], ids=["plain", "pair_w"])
@pytest.mark.parametrize("tokens,e,topk,e_begin,e_local,cols", MOE_CASES)
def test_moe_gather(tokens, e, topk, e_begin, e_local, cols, weighted):
    """Row r = x[pair // topk], or bf16(x * w[pair]) with pair weights; padding rows and every row past offsets[-1] up to
    max_rows are 0.  Bit-exact."""
    route, pair_w, gen = _moe_setup(tokens, e, topk, e_begin, e_local, seed=tokens + cols + topk)
    x = torch.randn(tokens, cols, device=DEV, generator=gen).bfloat16()
    out = torch.full((route.max_rows, cols), float("nan"), dtype=torch.bfloat16, device=DEV)
    ops.moe_gather(x, route, topk, pair_w if weighted else None, out=out)
    por = route.pair_of_row.long()
    valid = por >= 0
    assert int(route.offsets[-1]) < route.max_rows and int(valid.sum()) < int(route.offsets[-1])   # both kinds of pad rows
    src = x[por.clamp(min=0) // topk]
    if weighted:
        src = (src.float() * pair_w[por.clamp(min=0)].float()[:, None]).bfloat16()
    assert _bit_equal(out, torch.where(valid[:, None], src, torch.zeros_like(src)))


@pytest.mark.parametrize("form", ["forward", "backward"])
@pytest.mark.parametrize("tokens,e,topk,e_begin,e_local,cols", MOE_CASES)
def test_moe_combine(tokens, e, topk, e_begin, e_local, cols, form):
    """out[t] = bf16 of an fp32 accumulation over t's slots in slot order, rows of -1 skipped.  forward (moe.py's expert
    output): each term bf16(d[row] * w[pair]); backward (the grad-in of both expert GEMMs): d[row] then d2[row].
    Bit-exact."""
    route, pair_w, gen = _moe_setup(tokens, e, topk, e_begin, e_local, seed=tokens * 3 + cols + topk)
    d = torch.randn(route.max_rows, cols, device=DEV, generator=gen).bfloat16()
    d2 = torch.randn(route.max_rows, cols, device=DEV, generator=gen).bfloat16() if form == "backward" else None
    out = ops.moe_combine(d, route, tokens, topk, pair_w=pair_w if form == "forward" else None, d2=d2)
    rop = route.row_of_pair.long().view(tokens, topk)
    assert bool((rop < 0).any()) == (e_local < e)             # expert-parallel cases have pairs owned elsewhere
    acc = torch.zeros(tokens, cols, dtype=torch.float32, device=DEV)
    for s in range(topk):
        row = rop[:, s]
        on = (row >= 0)[:, None]
        rc = row.clamp(min=0)
        if form == "forward":
            term = (d[rc].float() * pair_w.view(tokens, topk)[:, s].float()[:, None]).bfloat16().float()
            acc = acc + torch.where(on, term, 0.0)
        else:
            acc = acc + torch.where(on, d[rc].float(), 0.0)
            acc = acc + torch.where(on, d2[rc].float(), 0.0)
    assert _bit_equal(out, acc.bfloat16())


@pytest.mark.parametrize("tokens,e,topk,e_begin,e_local,cols", MOE_CASES)
def test_moe_rowdot(tokens, e, topk, e_begin, e_local, cols):
    """dw[pair] = bf16(<g[token], d[row]>), exactly 0 for pairs without a row.  One warp per pair: each lane sums cols/32
    exact products in fp32, then 5 shuffle levels, so against the fp64 dot product
        |dw - ref| <= ulp(ref) + (cols/32 + 5) * 2^-24 * sum|g*d|."""
    route, _, gen = _moe_setup(tokens, e, topk, e_begin, e_local, seed=tokens * 5 + cols + topk)
    g = torch.randn(tokens, cols, device=DEV, generator=gen).bfloat16()
    d = torch.randn(route.max_rows, cols, device=DEV, generator=gen).bfloat16()
    dw = ops.moe_rowdot(g, d, route, topk)
    rop = route.row_of_pair.long()
    on = rop >= 0
    assert bool((_bits(dw)[~on] == 0).all())
    pairs = torch.nonzero(on).reshape(-1)
    prod = g[pairs // topk].double() * d[rop[pairs]].double()
    ref = prod.sum(-1)
    bound = _ulp(ref) + (cols / 32 + 5) * 2.0 ** -24 * prod.abs().sum(-1)
    err = (dw[pairs].double() - ref).abs()
    assert bool((err <= bound).all()), f"rowdot: worst error {float((err / bound).max()):.3f} of the bound"


def test_moe_route_rejects_more_than_32_local_experts():
    """33 local experts exceed the route kernel's per-thread tables: refused before any launch."""
    route = ops.MoeRoute(64, 33, DEV)
    with pytest.raises(RuntimeError, match="local experts"):
        ops.moe_route(route, torch.zeros(64, dtype=torch.int64, device=DEV))


# ---------------------------------------------------------------------------------- outlier loss and top-k
def _pattern(pred, ref):
    """bf16 bit pattern of |pred - ref| (what the selection orders), int32."""
    return (_bits((pred - ref).abs()).int() & 0x7FFF).reshape(-1)


def _grid_batch(rows, cols, gen, delta_units):
    """pred = ref + delta with ref on a 2^-4 grid in [-2, 2] and delta = delta_units * 2^-6 (|delta_units| < 120): every
    pred - ref is exact in bf16 and in fp32, so elements with one bf16 |d| pattern share their fp32 |d|."""
    ref = (torch.randint(-32, 33, (rows, cols), device=DEV, generator=gen).float() * 2.0 ** -4)
    pred = ref + delta_units.view(rows, cols).float() * 2.0 ** -6
    assert bool((pred.bfloat16().float() == pred).all())
    return pred.bfloat16(), ref.bfloat16()


def _run_ranks(pred, ref, mask, world):
    """One data-parallel iteration of `world` ranks simulated on one GPU: rank r holds rows r::world, the histograms are
    computed with ar_absdiff_hist and handed to every rank by an all_gather that returns them stacked."""
    lib = _lib.load()
    cols = pred.shape[1]
    numel_g = pred.numel()
    shards = []
    for r in range(world):
        p, q = pred[r::world].contiguous(), ref[r::world].contiguous()
        m = None if mask is None else mask[r::world].contiguous()
        shards.append((p, q, m))
    hists = torch.zeros(world, 32768, dtype=torch.int32, device=DEV)
    for r, (p, q, _) in enumerate(shards):
        _check(lib.ar_absdiff_hist(ops._p(p), ops._p(q), p.numel(), ops._p(hists[r]), ops._stream()), "ar_absdiff_hist")
    out = []
    for r, (p, q, m) in enumerate(shards):
        scratch = ops.OutlierSelect(DEV)
        seen = []

        def all_gather(dst, local, r=r, seen=seen):
            seen.append(torch.equal(local, hists[r]))
            dst.copy_(hists)

        loss_sum = torch.zeros(1, dtype=torch.float64, device=DEV)
        dpred = ops.mse_outlier_fwd_bwd(p, q, m, 1000.0, loss_sum, scratch, numel_global=numel_g, all_gather=all_gather,
                                        rank=r, world=world)
        assert seen == [True]                                   # this rank's own histogram went into the exchange
        assert int(scratch.hist.abs().sum()) == 0               # ... and only it is re-armed
        assert torch.equal(scratch.hist_all, hists)
        out.append(dict(sel=scratch.sel.cpu().tolist(), loss=float(loss_sum), dpred=dpred, bits=_pattern(p, q),
                        rows=p.shape[0]))
    cat_p = torch.cat([s[0] for s in shards]).view(-1, cols)
    cat_r = torch.cat([s[1] for s in shards]).view(-1, cols)
    cat_m = None if mask is None else torch.cat([s[2] for s in shards])
    single = torch.zeros(1, dtype=torch.float64, device=DEV)
    ops.mse_outlier_fwd_bwd(cat_p, cat_r, cat_m, 1000.0, single, ops.OutlierSelect(DEV))
    return out, float(single)


def _check_rank_selection(res, k):
    """Exactly k dropped over all ranks, one threshold, ties handed out in rank order."""
    thr = res[0]["sel"][0]
    assert all(x["sel"][0] == thr for x in res)
    above = [int((x["bits"] > thr).sum()) for x in res]
    ties = [int((x["bits"] == thr).sum()) for x in res]
    assert sum(above) + sum(x["sel"][1] for x in res) == k
    need = k - sum(above)
    for r, x in enumerate(res):
        assert x["sel"][1] == min(max(need - sum(ties[:r]), 0), ties[r]), (r, need, ties)
    return thr, need, ties


@pytest.mark.parametrize("world", [2, 3, 4])
def test_outlier_topk_ranks(world):
    """Rows split unevenly (1031 rows, batch[r::world]); 10 % of the rows masked, with pred == ref there so that the
    loss cannot depend on which ties the ranks drop.  The ranks' losses add up to the single-GPU loss of the batch."""
    rows, cols = 1031, 1024
    gen = _gen(world)
    units = torch.randint(-20, 21, (rows * cols,), device=DEV, generator=gen)
    hot = torch.randperm(rows * cols, device=DEV, generator=gen)[:rows * cols // 1500]
    units[hot] = torch.randint(-119, 120, (hot.numel(),), device=DEV, generator=gen)
    mask = (torch.rand(rows, device=DEV, generator=gen) > 0.1).to(torch.uint8)
    units.view(rows, cols)[mask == 0] = 0
    pred, ref = _grid_batch(rows, cols, gen, units)
    k = max(1, int(rows * cols / 1000))
    res, single = _run_ranks(pred, ref, mask, world)
    _check_rank_selection(res, k)
    assert sum(x["loss"] for x in res) == pytest.approx(single, rel=1e-6)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_outlier_topk_ties(world):
    """About 10*k elements share the threshold |d| = 30 * 2^-6; k/2 elements lie above it.  Rank 0 holds k/4 of the
    ties (fewer than needed), the other ranks the rest: rank 0 drops all of its ties, rank 1 the remainder, the others
    none.  The dropped elements are the ones with dpred == 0; the loss equals the fp64 sum of the kept d^2."""
    rows, cols = 1024, 1024
    n = rows * cols
    k = max(1, int(n / 1000))
    gen = _gen(10 + world)
    units = torch.randint(-10, 11, (n,), device=DEV, generator=gen)
    rank_of = (torch.arange(n, device=DEV) // cols) % world
    own0 = torch.nonzero(rank_of == 0).reshape(-1)
    rest = torch.nonzero(rank_of != 0).reshape(-1)
    own0 = own0[torch.randperm(own0.numel(), device=DEV, generator=gen)]
    rest = rest[torch.randperm(rest.numel(), device=DEV, generator=gen)]
    sign = lambda m: torch.randint(0, 2, (m,), device=DEV, generator=gen) * 2 - 1   # noqa: E731
    n_above = k // 2
    units[rest[:n_above]] = torch.randint(31, 61, (n_above,), device=DEV, generator=gen) * sign(n_above)
    units[own0[:k // 4]] = 30 * sign(k // 4)
    units[rest[n_above:n_above + 10 * k]] = 30 * sign(10 * k)
    pred, ref = _grid_batch(rows, cols, gen, units)
    res, single = _run_ranks(pred, ref, None, world)
    thr, need, ties = _check_rank_selection(res, k)
    assert thr == int(_bits(torch.tensor(30 * 2.0 ** -6, dtype=torch.bfloat16)))
    assert need == k - n_above and ties[0] == k // 4 < need and sum(ties) > 10 * k
    for x in res:
        dropped_ties = int(((x["bits"] == thr) & (x["dpred"].reshape(-1) == 0)).sum())
        assert dropped_ties == x["sel"][1]
        assert int(((x["bits"] > thr) & (x["dpred"].reshape(-1) != 0)).sum()) == 0
    d2 = (units.double() * 2.0 ** -6) ** 2
    kept = d2.sum() - d2[units.abs() > 30].sum() - need * (30 * 2.0 ** -6) ** 2
    assert sum(x["loss"] for x in res) == pytest.approx(float(kept), rel=1e-6)
    assert single == pytest.approx(float(kept), rel=1e-6)


def test_outlier_loss_production_shape():
    """16384 x 4096 with 10 % of the rows masked against the oracle (SignRoundV2Quantizer._get_loss) on the GPU: exactly
    k = numel // 1000 dropped, loss within 1e-4 relative, dpred bf16-equal on >= 99.9 % of the elements.  Ties at the
    threshold pattern cannot be avoided here; which of them are dropped changes only the fp32 residue inside one bf16
    bucket."""
    rows, cols = 16384, 4096
    gen = _gen(77)
    ref = torch.randn(rows, cols, device=DEV, generator=gen).bfloat16()
    pred = (ref.float() + 0.05 * torch.randn(rows, cols, device=DEV, generator=gen)).bfloat16()
    pred[3, 5] += 2.0
    pred[rows // 2, cols // 2] -= 3.0
    mask = (torch.rand(rows, device=DEV, generator=gen) > 0.1).to(torch.uint8)
    p32 = pred.clone().requires_grad_(True)
    loss = S.outlier_suppressed_loss(p32, ref, mask.reshape(rows, 1).long())
    (loss * 1000).backward()
    scratch = ops.OutlierSelect(DEV)
    loss_sum = torch.zeros(1, dtype=torch.float64, device=DEV)
    dpred = ops.mse_outlier_fwd_bwd(pred, ref, mask, 1000.0, loss_sum, scratch)
    k = rows * cols // 1000
    sel = scratch.sel.cpu().tolist()
    bits = _pattern(pred, ref)
    assert int((bits > sel[0]).sum()) + sel[1] == k
    assert float(loss_sum) / (rows * cols) == pytest.approx(float(loss.detach()), rel=1e-4)
    assert float((dpred == p32.grad).float().mean()) >= 0.999


def test_outlier_edges():
    """pred == ref: loss 0, sel = [0, k].  numel < 2000: k = 1, the largest |d| is the one dropped.  A few +-inf and NaN
    differences (fewer than k): ordered above every finite pattern, NaN highest, as torch.topk orders them, so all are
    dropped and the threshold is finite.

    The kernel writes 0 for a dropped element, so its loss stays finite.  The reference computes d * keep with a boolean
    keep, and a dropped inf gives inf * 0 = NaN (DESIGN.md 5b #10): the kernel's loss equals that formula with
    torch.where(keep, d, 0)."""
    scratch = ops.OutlierSelect(DEV)
    gen = _gen(5)

    # pred == ref
    x = torch.randn(64, 256, device=DEV, generator=gen).bfloat16()
    loss_sum = torch.zeros(1, dtype=torch.float64, device=DEV)
    dpred = ops.mse_outlier_fwd_bwd(x, x.clone(), None, 1000.0, loss_sum, scratch)
    sel = scratch.sel.cpu().tolist()
    assert float(loss_sum) == 0.0 and sel[:2] == [0, 64 * 256 // 1000] and int(dpred.count_nonzero()) == 0

    # numel < 2000: k = 1
    ref = torch.randn(13, 152, device=DEV, generator=gen).bfloat16()
    pred = (ref.float() + 0.1 * torch.randn(13, 152, device=DEV, generator=gen)).bfloat16()
    pred[7, 100] = ref[7, 100] + 5.0
    loss_sum.zero_()
    dpred = ops.mse_outlier_fwd_bwd(pred, ref, None, 1000.0, loss_sum, scratch)
    bits = _pattern(pred, ref)
    sel = scratch.sel.cpu().tolist()
    assert int((bits > sel[0]).sum()) + sel[1] == 1 and sel[0] == int(bits.max())
    assert float(dpred[7, 100]) == 0.0 and int(dpred.count_nonzero()) == int(((pred - ref) != 0).sum()) - 1
    assert float(loss_sum) / pred.numel() == pytest.approx(float(S.outlier_suppressed_loss(pred, ref, None)), rel=1e-5)

    # +-inf and NaN differences, fewer than k
    rows, cols = 256, 1024
    units = torch.randint(-40, 41, (rows * cols,), device=DEV, generator=gen)
    pred, ref = _grid_batch(rows, cols, gen, units)
    pred[0, 0] = float("inf")
    pred[1, 1] = float("-inf")
    ref[2, 2] = float("inf")
    pred[3, 3] = float("nan")
    ref[4, 4] = float("nan")
    k = rows * cols // 1000
    loss_sum.zero_()
    dpred = ops.mse_outlier_fwd_bwd(pred, ref, None, 1000.0, loss_sum, scratch)
    sel = scratch.sel.cpu().tolist()
    bits = _pattern(pred, ref)
    flat = (pred - ref).abs().reshape(-1)
    top_v, top_i = torch.topk(flat, k)
    nonfinite = ~torch.isfinite(flat)
    assert int(nonfinite.sum()) == 5 and bool(nonfinite[top_i].sum() == 5)
    assert sel[0] < 0x7F80 and sel[0] == int(_bits(top_v[-1:]).int() & 0x7FFF)
    assert bool((bits[nonfinite] > sel[0]).all())
    assert int((bits > sel[0]).sum()) + sel[1] == k
    assert bool(torch.isfinite(dpred.float()).all()) and bool((dpred.reshape(-1)[nonfinite] == 0).all())
    keep = torch.ones_like(flat, dtype=torch.bool)
    keep[top_i] = False
    d = (pred.float() - ref.float()).abs().reshape(-1)
    want = torch.mean(torch.where(keep, d, 0.0).double() ** 2)
    assert float(loss_sum) / flat.numel() == pytest.approx(float(want), rel=1e-6)
    assert bool(torch.isnan(S.outlier_suppressed_loss(pred, ref, None)))


# ------------------------------------------------------------------------------------------------ loop schedule
def test_mse_fwd_bwd_production_shape():
    """16384 x 4096, 10 % of the rows masked.  loss_sum within 1e-6 relative of fp64 and accumulating over two calls;
    dpred value-equal (a masked zero may be -0) to autograd of test_gpu_kernels.py::test_mse_best_gather's expression."""
    rows, cols = 16384, 4096
    gen = _gen(11)
    pred = torch.randn(rows, cols, device=DEV, generator=gen).bfloat16()
    ref = torch.randn(rows, cols, device=DEV, generator=gen).bfloat16()
    mask = torch.rand(rows, device=DEV, generator=gen) > 0.1
    m = mask.to(torch.long).unsqueeze(-1)
    pr = pred.clone().requires_grad_(True)
    loss = F.mse_loss((pr * m).float(), (ref * m).float())
    (loss * 1000).backward()
    exact = float((((pred.double() - ref.double()) * m) ** 2).sum())
    loss_sum = torch.zeros(1, dtype=torch.float64, device=DEV)
    m8 = mask.to(torch.uint8)
    dp = ops.mse_fwd_bwd(pred, ref, m8, 1.0 / (rows * cols), 1000.0, loss_sum)
    assert float(loss_sum) == pytest.approx(exact, rel=1e-6)
    assert torch.equal(dp, pr.grad)
    dp2 = ops.mse_fwd_bwd(pred, ref, m8, 1.0 / (rows * cols), 1000.0, loss_sum)
    assert float(loss_sum) == pytest.approx(2 * exact, rel=1e-6)
    assert torch.equal(dp2, pr.grad)


def test_best_update_device_overrides():
    """The CUDA graph passes the iteration and 1/num_elm through device memory: they override the by-value arguments.
    Iteration 0 resets the best, a loss equal to the best is not better, loss_hist is written at the device iteration."""
    state = torch.zeros(4, dtype=torch.float64, device=DEV)
    state[0] = 1e-30                                            # lower than any loss below: only a reset replaces it
    flag = torch.full((1,), 7, dtype=torch.int32, device=DEV)
    hist = torch.zeros(8, dtype=torch.float32, device=DEV)
    it = torch.zeros(1, dtype=torch.int32, device=DEV)
    inv_dev = torch.tensor([1.0 / 7.0], dtype=torch.float64, device=DEV)
    loss_sum = torch.zeros(1, dtype=torch.float64, device=DEV)
    inv_numel = 1.0 / 4096

    def total(ls):
        return float(torch.tensor(ls * inv_numel, dtype=torch.float32)) * (1.0 / 7.0)

    def step(ls, host_it):
        loss_sum.fill_(ls)
        ops.best_update(loss_sum, inv_numel, 1.0, host_it, state, flag, hist, inv_num_elm_dev=inv_dev, it_dev=it)
        torch.cuda.synchronize()
        assert float(loss_sum) == 0.0

    step(1234.5, host_it=5)                                     # device iteration 0
    assert int(flag) == 1 and float(state[0]) == total(1234.5) and float(state[2]) == 0.0
    assert float(state[1]) == total(1234.5) and float(hist[0]) == pytest.approx(total(1234.5), rel=1e-7)
    assert float(hist[5]) == 0.0
    it.fill_(1)
    step(1234.5, host_it=0)                                     # equal to the best: not better; host iteration 0 ignored
    assert int(flag) == 0 and float(state[0]) == total(1234.5) and float(state[2]) == 0.0
    assert float(hist[1]) == pytest.approx(total(1234.5), rel=1e-7)
    it.fill_(2)
    step(1000.0, host_it=0)
    assert int(flag) == 1 and float(state[0]) == total(1000.0) and float(state[2]) == 2.0
    assert float(hist[2]) == pytest.approx(total(1000.0), rel=1e-7)
    it.fill_(3)
    step(5000.0, host_it=0)
    assert int(flag) == 0 and float(state[0]) == total(1000.0) and float(state[1]) == total(5000.0)
    assert float(state[2]) == 2.0 and float(hist[3]) == pytest.approx(total(5000.0), rel=1e-7)


@pytest.mark.parametrize("count", [3, 200])
def test_sched_load_iter_advance(count):
    """Three sched_load -> iter_advance rounds reproduce the schedule table's rows in cur32 / cur64 / cur_inv (200
    entries: more than the kernel's 64 threads)."""
    gen = _gen(count)
    iters = 5
    table = torch.randint(0, 1 << 30, (iters, count), dtype=torch.int32, device=DEV, generator=gen)
    inv_table = torch.rand(iters, dtype=torch.float64, device=DEV, generator=gen)
    it = torch.zeros(1, dtype=torch.int32, device=DEV)
    cur32 = torch.empty(count, dtype=torch.int32, device=DEV)
    cur64 = torch.empty(count, dtype=torch.int64, device=DEV)
    cur_inv = torch.empty(1, dtype=torch.float64, device=DEV)
    for r in range(3):
        cur32.fill_(-1)
        cur64.fill_(-1)
        cur_inv.fill_(-1.0)
        ops.sched_load(table, inv_table, it, count, cur32, cur64, cur_inv)
        assert torch.equal(cur32, table[r]) and torch.equal(cur64, table[r].long())
        assert float(cur_inv) == float(inv_table[r])
        ops.iter_advance(it)
        assert int(it) == r + 1


@pytest.mark.parametrize("row_elems", [8, 2048 * 4096])
def test_gather_rows(row_elems):
    """count 8 with repeated indices; 2048*4096-element rows run the grid-capped loop.  Raw bits (NaN payloads
    included) are copied exactly."""
    gen = _gen(row_elems % 1009)
    src = torch.randint(-32768, 32768, (10, row_elems), dtype=torch.int32, device=DEV, generator=gen)
    src = src.to(torch.int16).view(torch.bfloat16)
    idx = torch.tensor([3, 3, 0, 9, 3, 7, 0, 1], dtype=torch.int32, device=DEV)
    out = ops.gather_rows(src, idx)
    assert _bit_equal(out, src[idx.long()])
