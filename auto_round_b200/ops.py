"""Thin torch-tensor front end over the C ABI (include/ar_b200.h).  PyTorch only owns the memory and the
stream; every function below enqueues hand-written sm_90a kernels from libar_b200.so and returns.

No function here has a CPU / eager fallback: tensors must be CUDA tensors and the library must load.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import torch

from . import _lib
from ._lib import DT_INT_ASYM, DT_INT_SYM, DT_MX_FP4, DT_NV_FP4, QSpec

# number of kernels of libar_b200.so launched through this module (bench.py reports it as `gpu_launches`)
LAUNCHES = [0]
_KERNELS_PER_CALL = {"ar_group_minmax": 1, "ar_absmax": 1, "ar_nv_global_scale": 1, "ar_qdq_fwd": 1, "ar_qdq_bwd": 1,
                     "ar_gemm_bf16": 1, "ar_fq_linear_bwd_dx": 1,
                     "ar_mse_fwd_bwd": 1, "ar_best_update": 1, "ar_sched_load": 1, "ar_iter_advance": 1, "ar_gather_rows": 1,
                     "ar_pack_int": 3, "ar_unpack_int": 1, "ar_pack_awq": 2, "ar_unpack_awq": 1,
                     "ar_pack_fp4_nv": 1, "ar_pack_fp4_mx": 1, "ar_unpack_fp4": 1}


def _check(rc, what):
    LAUNCHES[0] += _KERNELS_PER_CALL.get(what, 1)
    _lib.check(rc, what)


DTYPE_IDS = {"int_sym": DT_INT_SYM, "int_asym": DT_INT_ASYM, "mx_fp4": DT_MX_FP4, "nv_fp4": DT_NV_FP4}


@dataclass(frozen=True)
class Spec:
    """Quantisation spec of one linear layer (mirror of struct ar_qspec)."""
    dtype: int
    bits: int
    group_size: int
    n: int
    k: int
    q_scale_thresh: float = 1e-5
    scale_bound_hi: float = 1.0

    @property
    def kpad(self) -> int:
        g = self.group_size
        return (self.k + g - 1) // g * g

    @property
    def groups(self) -> int:
        return self.n * (self.kpad // self.group_size)

    @property
    def is_int(self) -> bool:
        return self.dtype in (DT_INT_SYM, DT_INT_ASYM)

    def c(self) -> QSpec:
        return QSpec(self.dtype, self.bits, self.group_size, self.n, self.k, self.q_scale_thresh, self.scale_bound_hi)


def make_spec(name: str, bits: int, group_size: int, n: int, k: int, q_scale_thresh: float = 1e-5,
              scale_bound_hi: float = 1.0) -> Spec:
    """group_size -1, or a weight narrower than the group (K < group_size), means one group per ROW in the reference
    (reshape_pad_tensor_by_group_size, data_type/utils.py:57-61): encoded as group_size == K (int types only)."""
    if group_size == 0:
        raise NotImplementedError("group_size = 0 (one group per tensor) is outside the H100 hot path")
    if group_size == -1 or k < group_size:
        if name not in ("int_sym", "int_asym"):
            raise NotImplementedError(f"{name}: per-row groups (group_size=-1 / K < group_size) exist for the int types only")
        if k % 8:
            raise NotImplementedError("per-row groups need K % 8 == 0")
        group_size = k
    return Spec(DTYPE_IDS[name], bits, group_size, n, k, q_scale_thresh, scale_bound_hi)


def _cspec(spec: "Spec", init_scale=None) -> QSpec:
    """struct ar_qspec for a call; `init_scale` (fp32 [G], enable_alg_ext) rides in the spec (include/ar_b200.h)."""
    cs = spec.c()
    if init_scale is not None:
        _want(init_scale, torch.float32, "init_scale")
        if init_scale.numel() != spec.groups:
            raise ValueError(f"init_scale has {init_scale.numel()} entries, the layer has {spec.groups} groups")
        cs.init_scale = _p(init_scale)
    return cs


def _p(t):
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError("auto_round_b200 kernels take CUDA tensors only (no CPU fallback)")
    if not t.is_contiguous():
        raise RuntimeError("tensor must be contiguous")
    return C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _want(t, dtype, what):
    if t is not None and t.dtype != dtype:
        raise TypeError(f"{what}: expected {dtype}, got {t.dtype}")


def group_minmax(spec: Spec, w: torch.Tensor):
    """weight_min / weight_max per group, bf16 [G] (auto_round/wrapper.py:154-167)."""
    _want(w, torch.bfloat16, "w")
    wmin = torch.empty(spec.groups, dtype=torch.bfloat16, device=w.device)
    wmax = torch.empty_like(wmin)
    cs = spec.c()
    _check(_lib.load().ar_group_minmax(C.byref(cs), _p(w), _p(wmin), _p(wmax), _stream()), "ar_group_minmax")
    return wmin, wmax


def nv_global_scale(w: torch.Tensor) -> torch.Tensor:
    """448*6/amax(|W|) as a device fp32 scalar (auto_round/data_type/nvfp.py:56-64)."""
    _want(w, torch.bfloat16, "w")
    amax = torch.zeros(1, dtype=torch.float32, device=w.device)
    gs = torch.empty(1, dtype=torch.float32, device=w.device)
    lib = _lib.load()
    _check(lib.ar_absmax(_p(w), w.numel(), _p(amax), _stream()), "ar_absmax")
    _check(lib.ar_nv_global_scale(_p(amax), _p(gs), _stream()), "ar_nv_global_scale")
    return gs


def scale_dtype_of(spec: Spec):
    return {DT_INT_SYM: torch.float16, DT_INT_ASYM: torch.float16, DT_MX_FP4: torch.bfloat16,
            DT_NV_FP4: torch.float32}[spec.dtype]


def qdq_fwd(spec: Spec, w, v=None, min_scale=None, max_scale=None, wmin=None, wmax=None, gscale=None,
            out_wq=None, want_wq=True, want_scale=False, init_scale=None):
    """Fake-quant forward.  Returns (wq bf16 [N,K] | None, scale [G] | None, zp fp32 [G] | None)."""
    _want(w, torch.bfloat16, "w")
    for t, nm in ((v, "v"), (min_scale, "min_scale"), (max_scale, "max_scale"), (gscale, "gscale")):
        _want(t, torch.float32, nm)
    wq = (out_wq if out_wq is not None else torch.empty_like(w)) if want_wq else None
    scale = torch.empty(spec.groups, dtype=scale_dtype_of(spec), device=w.device) if want_scale else None
    zp = torch.empty(spec.groups, dtype=torch.float32, device=w.device) if (want_scale and spec.dtype == DT_INT_ASYM) else None
    cs = _cspec(spec, init_scale)
    _check(_lib.load().ar_qdq_fwd(C.byref(cs), _p(w), _p(v), _p(min_scale), _p(max_scale), _p(wmin), _p(wmax),
                                      _p(gscale), _p(wq), _p(scale), _p(zp), _stream()), "ar_qdq_fwd")
    return wq, scale, zp


def qdq_bwd(spec: Spec, w, gq, v=None, min_scale=None, max_scale=None, wmin=None, wmax=None, gscale=None,
            dv=None, dmin=None, dmax=None, accumulate=False, init_scale=None):
    """Fake-quant backward: Gq fp32 [N,K] -> (dv fp32 [N,Kpad], dmin [G] | None, dmax [G])."""
    _want(w, torch.bfloat16, "w")
    _want(gq, torch.float32, "gq")
    dev = w.device
    if dv is None:
        dv = torch.empty(spec.n, spec.kpad, dtype=torch.float32, device=dev)
    if dmax is None:
        dmax = torch.empty(spec.groups, dtype=torch.float32, device=dev)
    if dmin is None and spec.is_int:
        dmin = torch.empty(spec.groups, dtype=torch.float32, device=dev)
    cs = _cspec(spec, init_scale)
    _check(_lib.load().ar_qdq_bwd(C.byref(cs), _p(w), _p(v), _p(min_scale), _p(max_scale), _p(wmin), _p(wmax),
                                      _p(gscale), _p(gq), _p(dv), _p(dmin), _p(dmax), int(accumulate), _stream()),
               "ar_qdq_bwd")
    return dv, dmin, dmax


def gemm(a, b, a_mn_major=False, b_mn_major=False, bias=None, out=None):
    """D[M,N] = A·Bᵀ on wgmma.  A is [M,K] (or stored [K,M] if a_mn_major), B is [N,K] (or stored [K,N])."""
    _want(a, torch.bfloat16, "a")
    _want(b, torch.bfloat16, "b")
    if a_mn_major:
        k, m = a.shape
    else:
        m, k = a.shape
    if b_mn_major:
        kb, n = b.shape
    else:
        n, kb = b.shape
    if kb != k:
        raise ValueError(f"reduction dims differ: {k} vs {kb}")
    d = out if out is not None else torch.empty(m, n, dtype=torch.bfloat16, device=a.device)
    _check(_lib.load().ar_gemm_bf16(_p(a), _p(b), _p(d), m, n, k, int(a_mn_major), int(b_mn_major),
                                        a.stride(0), b.stride(0), d.stride(0), _p(bias), _stream()), "ar_gemm_bf16")
    return d


def fq_linear_bwd_dx(spec: Spec, dy2d, wq, out=None):
    _want(dy2d, torch.bfloat16, "dy")
    t = dy2d.shape[0]
    dx = out if out is not None else torch.empty(t, spec.k, dtype=torch.bfloat16, device=dy2d.device)
    cs = spec.c()
    _check(_lib.load().ar_fq_linear_bwd_dx(C.byref(cs), _p(dy2d), t, _p(wq), _p(dx), _stream()), "ar_fq_linear_bwd_dx")
    return dx


def fq_update(spec: Spec, w, v, min_scale, max_scale, wmin, wmax, gscale, gq, wq_out, lr_table, best_v=None, best_min=None,
              best_max=None, flag=None, it=0, it_dev=None, clamp_hi=1.0, row0=0, row1=None, gq_row0=0, init_scale=None,
              dbg=None, has_grad=None, wire=None):
    """Fused per-layer update (include/ar_b200.h ar_fq_update): qdq backward from the bf16 dWq `gq`, snapshot, sign-SGD
    step, next iteration's fake-quant weight into `wq_out` -- rows [row0, row1).  `dbg` = (dv, dmin, dmax) fp32 outputs."""
    _want(w, torch.bfloat16, "w")
    _want(gq, torch.bfloat16, "gq")
    if wq_out is not None:
        _want(wq_out, torch.bfloat16, "wq_out")
    for t, nm in ((v, "v"), (min_scale, "min_scale"), (max_scale, "max_scale"), (best_v, "best_v"), (lr_table, "lr_table")):
        _want(t, torch.float32, nm)
    row1 = spec.n if row1 is None else row1
    if gq.numel() < (row1 - gq_row0) * spec.k:
        raise ValueError("gq does not cover rows [gq_row0, row1)")
    cs = _cspec(spec, init_scale)
    dv, dmn, dmx = dbg if dbg is not None else (None, None, None)
    codes = gpar = None
    if wire is not None:                      # uint8 segment of this rank: [codes | group params] (wire_segment_bytes)
        rows = row1 - row0
        nb = rows * (spec.kpad // 8) * 4
        if wire.dtype != torch.uint8 or wire.numel() < wire_segment_bytes(spec, rows):
            raise ValueError("wire segment too small")
        codes, gpar = wire[:nb], wire[nb:]
    _check(_lib.load().ar_fq_update(C.byref(cs), _p(w), _p(v), _p(min_scale), _p(max_scale), _p(wmin), _p(wmax), _p(gscale),
                                    _p(gq), int(gq_row0), int(row0), int(row1), _p(best_v), _p(best_min), _p(best_max),
                                    _p(flag), _p(lr_table), int(it), _p(it_dev), float(clamp_hi),
                                    _p(wq_out) if wire is None else None, _p(dv), _p(dmn),
                                    _p(dmx), _p(has_grad), _p(codes), _p(gpar), _stream()), "ar_fq_update")


def wire_supported(spec: Spec) -> bool:
    """The 4-bit wire form of the next fake-quant weight (data-parallel all-gather): bits <= 4, grouped (not per-row)."""
    return spec.bits <= 4 and spec.group_size in (16, 32, 64, 128, 256)


def wire_segment_bytes(spec: Spec, rows: int) -> int:
    """One rank's segment: u32 per 8 elements + {a, off} fp32 per group, rounded up to 16 bytes."""
    nb = rows * (spec.kpad // 8) * 4 + rows * (spec.kpad // spec.group_size) * 8
    return (nb + 15) // 16 * 16


def wq_decode(spec: Spec, segments, world, wq_out):
    """wq_out[N,K] <- the all-gathered wire segments (uint8 [world * seg_bytes]); the values fq_update's wq_out would hold."""
    _want(wq_out, torch.bfloat16, "wq_out")
    if segments.dtype != torch.uint8 or segments.numel() % world:
        raise ValueError("segments: uint8, world equal parts")
    cs = spec.c()
    _check(_lib.load().ar_wq_decode(C.byref(cs), _p(segments), segments.numel() // world, int(world), _p(wq_out), _stream()),
           "ar_wq_decode")
    return wq_out


def mse_fwd_bwd(pred2d, ref2d, row_mask, inv_numel, upstream, loss_sum, dpred=None, want_grad=True):
    """loss_sum (double [1]) += sum(((pred-ref)*m)^2); returns dpred bf16 (see include/ar_b200.h)."""
    _want(pred2d, torch.bfloat16, "pred")
    _want(ref2d, torch.bfloat16, "ref")
    _want(loss_sum, torch.float64, "loss_sum")
    _want(row_mask, torch.uint8, "row_mask")
    rows, cols = pred2d.shape
    if want_grad and dpred is None:
        dpred = torch.empty_like(pred2d)
    _check(_lib.load().ar_mse_fwd_bwd(_p(pred2d), _p(ref2d), _p(row_mask), rows, cols, float(inv_numel), float(upstream),
                                          _p(loss_sum), _p(dpred) if want_grad else None, _stream()), "ar_mse_fwd_bwd")
    return dpred


def best_update(loss_sum, inv_numel, inv_num_elm, it, state, flag, loss_hist, inv_num_elm_dev=None, it_dev=None):
    """`inv_num_elm_dev` (double [1]) / `it_dev` (int32 [1]) override the host values (CUDA-graph replay)."""
    _check(_lib.load().ar_best_update(_p(loss_sum), float(inv_numel), float(inv_num_elm), int(it), _p(inv_num_elm_dev),
                                      _p(it_dev), _p(state), _p(flag), _p(loss_hist), _stream()), "ar_best_update")


def sched_load(idx_table, inv_num_elm_table, it_dev, count, cur32, cur64, cur_inv):
    _want(idx_table, torch.int32, "idx_table")
    _want(it_dev, torch.int32, "it")
    _check(_lib.load().ar_sched_load(_p(idx_table), _p(inv_num_elm_table), _p(it_dev), int(count), _p(cur32), _p(cur64),
                                     _p(cur_inv), _stream()), "ar_sched_load")


def iter_advance(it_dev):
    _check(_lib.load().ar_iter_advance(_p(it_dev), _stream()), "ar_iter_advance")


def gather_rows(src, idx_i32, out=None):
    """out[i] = src[idx[i]] for a [S, ...] bf16 tensor of cached samples."""
    _want(src, torch.bfloat16, "src")
    _want(idx_i32, torch.int32, "idx")
    count = idx_i32.numel()
    row = src[0].numel()
    if out is None:
        out = torch.empty((count,) + tuple(src.shape[1:]), dtype=src.dtype, device=src.device)
    _check(_lib.load().ar_gather_rows(_p(src), _p(idx_i32), count, row, _p(out), _stream()), "ar_gather_rows")
    return out


def pack_int(wq, scale_f16, zp, bits, group_size, zp_minus_one, zp_const=0):
    """-> qweight i32 [K*bits/32,N], qzeros i32 [G',N*bits/32], scales fp16 [G',N], g_idx i32 [K]."""
    _want(wq, torch.bfloat16, "wq")
    _want(scale_f16, torch.float16, "scale")
    _want(zp, torch.float32, "zp")
    n, k = wq.shape
    g = k if group_size in (-1, 0) else group_size
    ng = (k + g - 1) // g
    dev = wq.device
    qweight = torch.empty(k * bits // 32, n, dtype=torch.int32, device=dev)
    qzeros = torch.empty(ng, n * bits // 32, dtype=torch.int32, device=dev)
    scales_t = torch.empty(ng, n, dtype=torch.float16, device=dev)
    g_idx = torch.empty(k, dtype=torch.int32, device=dev)
    _check(_lib.load().ar_pack_int(_p(wq), _p(scale_f16), _p(zp), int(zp_const), n, k, bits, g, int(zp_minus_one),
                                       _p(qweight), _p(qzeros), _p(scales_t), _p(g_idx), _stream()), "ar_pack_int")
    return qweight, qzeros, scales_t, g_idx


def unpack_int(qweight, qzeros, scales_t, n, k, bits, group_size, zp_minus_one, want_codes=False):
    g = k if group_size in (-1, 0) else group_size
    w = torch.empty(n, k, dtype=torch.bfloat16, device=qweight.device)
    codes = torch.empty(n, k, dtype=torch.int32, device=qweight.device) if want_codes else None
    _check(_lib.load().ar_unpack_int(_p(qweight), _p(qzeros), _p(scales_t), n, k, bits, g, int(zp_minus_one), _p(w),
                                         _p(codes), _stream()), "ar_unpack_int")
    return w, codes


def pack_awq(wq, scale_f16, zp, group_size, zp_const=0):
    """AWQ GEMM layout, 4 bit -> qweight i32 [K,N/8], qzeros i32 [G,N/8], scales fp16 [G,N].  `zp` fp32 [N,G], or None
    for a symmetric layer (`zp_const` fills every nibble).  Shapes the layout cannot hold raise the reference's
    ValueError (export_to_awq/utils.py:153-158)."""
    _want(wq, torch.bfloat16, "wq")
    _want(scale_f16, torch.float16, "scale")
    _want(zp, torch.float32, "zp")
    n, k = wq.shape
    g = k if group_size == -1 else group_size
    if g <= 0 or k % g != 0:
        raise ValueError(f"in_features ({k}) shape mismatch")
    if n % 8 != 0:
        raise ValueError(f"out_features ({n}) shape mismatch")
    dev = wq.device
    qweight = torch.empty(k, n // 8, dtype=torch.int32, device=dev)
    qzeros = torch.empty(k // g, n // 8, dtype=torch.int32, device=dev)
    scales_t = torch.empty(k // g, n, dtype=torch.float16, device=dev)
    _check(_lib.load().ar_pack_awq(_p(wq), _p(scale_f16), _p(zp), int(zp_const), n, k, g, _p(qweight), _p(qzeros),
                                   _p(scales_t), _stream()), "ar_pack_awq")
    return qweight, qzeros, scales_t


def unpack_awq(qweight, qzeros, scales_t, n, k, group_size, want_codes=False):
    w = torch.empty(n, k, dtype=torch.bfloat16, device=qweight.device)
    codes = torch.empty(n, k, dtype=torch.int32, device=qweight.device) if want_codes else None
    _check(_lib.load().ar_unpack_awq(_p(qweight), _p(qzeros), _p(scales_t), n, k, group_size, _p(w), _p(codes), _stream()),
           "ar_unpack_awq")
    return w, codes


def pack_fp4_nv(wq, scale_f32, gscale):
    _want(wq, torch.bfloat16, "wq")
    _want(scale_f32, torch.float32, "scale")
    n, k = wq.shape
    packed = torch.empty(n, k // 2, dtype=torch.uint8, device=wq.device)
    sc = torch.empty(n, k // 16, dtype=torch.uint8, device=wq.device)
    _check(_lib.load().ar_pack_fp4_nv(_p(wq), _p(scale_f32), _p(gscale), n, k, _p(packed), _p(sc), _stream()),
               "ar_pack_fp4_nv")
    return packed, sc


def pack_fp4_mx(wq, exp_bf16):
    _want(wq, torch.bfloat16, "wq")
    _want(exp_bf16, torch.bfloat16, "exp")
    n, k = wq.shape
    packed = torch.empty(n, k // 2, dtype=torch.uint8, device=wq.device)
    sc = torch.empty(n, k // 32, dtype=torch.uint8, device=wq.device)
    _check(_lib.load().ar_pack_fp4_mx(_p(wq), _p(exp_bf16), n, k, _p(packed), _p(sc), _stream()), "ar_pack_fp4_mx")
    return packed, sc


def unpack_fp4(packed, n, k):
    out = torch.empty(n, k, dtype=torch.bfloat16, device=packed.device)
    _check(_lib.load().ar_unpack_fp4(_p(packed), n, k, _p(out), _stream()), "ar_unpack_fp4")
    return out


# ------------------------------------------------------------------------- MoE: routing + grouped GEMMs (csrc/ar_moe.cu)
class MoeRoute:
    """Device-side routing tables of one iteration (ar_moe_route): static shapes, filled in the stream."""

    def __init__(self, pairs: int, e_local: int, device):
        self.pairs, self.e_local = pairs, e_local
        self.max_rows = (pairs + 255 * e_local + 255) // 256 * 256
        i32 = dict(dtype=torch.int32, device=device)
        self.counts = torch.zeros(e_local, **i32)
        self.offsets = torch.zeros(e_local + 1, **i32)
        self.row_of_pair = torch.zeros(pairs, **i32)
        self.pair_of_row = torch.zeros(self.max_rows, **i32)
        self.mtab = torch.zeros(2 * (self.max_rows // 256), **i32)
        self.num_mt = torch.zeros(1, **i32)
        self.ktab = torch.zeros(3 * e_local, **i32)
        self.num_active = torch.zeros(1, **i32)


def moe_route(route: MoeRoute, expert_ids, e_begin=0):
    _want(expert_ids, torch.int64, "expert_ids")
    if expert_ids.numel() != route.pairs:
        raise ValueError("expert_ids does not match the route's pair count")
    _check(_lib.load().ar_moe_route(_p(expert_ids), route.pairs, int(e_begin), route.e_local, route.max_rows, _p(route.counts),
                                    _p(route.offsets), _p(route.row_of_pair), _p(route.pair_of_row), _p(route.mtab),
                                    _p(route.num_mt), _p(route.ktab), _p(route.num_active), _stream()), "ar_moe_route")
    return route


def moe_gather(x2d, route: MoeRoute, topk, pair_w=None, out=None):
    _want(x2d, torch.bfloat16, "x")
    _want(pair_w, torch.bfloat16, "pair_w")
    cols = x2d.shape[1]
    if out is None:
        out = torch.empty(route.max_rows, cols, dtype=torch.bfloat16, device=x2d.device)
    _check(_lib.load().ar_moe_gather(_p(x2d), _p(route.pair_of_row), _p(pair_w), int(topk), route.max_rows, cols, _p(out),
                                     _stream()), "ar_moe_gather")
    return out


def moe_combine(d, route: MoeRoute, tokens, topk, pair_w=None, d2=None, out=None):
    _want(d, torch.bfloat16, "d")
    _want(d2, torch.bfloat16, "d2")
    _want(pair_w, torch.bfloat16, "pair_w")
    cols = d.shape[1]
    if out is None:
        out = torch.empty(tokens, cols, dtype=torch.bfloat16, device=d.device)
    _check(_lib.load().ar_moe_combine(_p(d), _p(d2), _p(route.row_of_pair), _p(pair_w), int(tokens), int(topk), cols, _p(out),
                                      _stream()), "ar_moe_combine")
    return out


def moe_rowdot(g2d, d, route: MoeRoute, topk):
    _want(g2d, torch.bfloat16, "g")
    _want(d, torch.bfloat16, "d")
    dw = torch.empty(route.pairs, dtype=torch.bfloat16, device=d.device)
    _check(_lib.load().ar_moe_rowdot(_p(g2d), _p(d), _p(route.row_of_pair), route.pairs, int(topk), d.shape[1], _p(dw), _stream()),
           "ar_moe_rowdot")
    return dw


def gemm_grouped_m(a, b_stack, route: MoeRoute, n, k, b_mn_major=False, out=None):
    """GROUP_M: out[rows, n] = a[rows, k] · B_eᵀ per 256-row tile.  b_stack: [E, n, k] (forward) or, with b_mn_major,
    [E, k, n] read as the MN-major operand (grad-in: reduction over the expert's k rows)."""
    _want(a, torch.bfloat16, "a")
    _want(b_stack, torch.bfloat16, "b")
    rows = route.max_rows
    e = b_stack.shape[0]
    if out is None:
        out = torch.empty(rows, n, dtype=torch.bfloat16, device=a.device)
    group_rows = k if b_mn_major else n
    _check(_lib.load().ar_gemm_bf16_grouped(_p(a), _p(b_stack), _p(out), 1, rows, n, k, 0, int(b_mn_major), a.stride(0),
                                            b_stack.stride(1), out.stride(0), group_rows, e, _p(route.mtab), _p(route.num_mt),
                                            rows // 256, 0, _stream()), "ar_gemm_bf16_grouped")
    return out


def gemm_grouped_k(dy, x, route: MoeRoute, out_stack):
    """GROUP_K: out_stack[e, :n_out] = dy[rows_e, :n_out]ᵀ · x[rows_e, :k_out] for every expert with tokens.  out_stack is
    [E, pitch, k_out] with pitch = n_out rounded up to 256 (rows n_out.. of a slab are scratch)."""
    _want(dy, torch.bfloat16, "dy")
    _want(x, torch.bfloat16, "x")
    _want(out_stack, torch.bfloat16, "out")
    e, pitch, k_out = out_stack.shape
    n_out = dy.shape[1]
    if pitch % 256 or pitch < n_out or not out_stack.is_contiguous():
        raise ValueError("out_stack must be contiguous [E, pitch, k_out] with pitch a multiple of 256 >= dy.shape[1]")
    _check(_lib.load().ar_gemm_bf16_grouped(_p(dy), _p(x), _p(out_stack), 2, route.max_rows, k_out, route.max_rows, 1, 1,
                                            dy.stride(0), x.stride(0), k_out, pitch, e, _p(route.ktab),
                                            _p(route.num_active), route.e_local, n_out, _stream()), "ar_gemm_bf16_grouped")
    return out_stack


# ------------------------------------------------------------------- fused block glue (csrc/ar_block.cu)
def rmsnorm_fwd(x2d, w, eps):
    _want(x2d, torch.bfloat16, "x")
    _want(w, torch.bfloat16, "w")
    rows, hidden = x2d.shape
    y = torch.empty_like(x2d)
    rstd = torch.empty(rows, dtype=torch.float32, device=x2d.device)
    _check(_lib.load().ar_rmsnorm_fwd(_p(x2d), _p(w), float(eps), rows, hidden, _p(y), _p(rstd), _stream()), "ar_rmsnorm_fwd")
    return y, rstd


def rmsnorm_bwd(dy2d, x2d, w, rstd):
    rows, hidden = x2d.shape
    dx = torch.empty_like(x2d)
    _check(_lib.load().ar_rmsnorm_bwd(_p(dy2d), _p(x2d), _p(w), _p(rstd), rows, hidden, _p(dx), 0, _stream()), "ar_rmsnorm_bwd")
    return dx


def rope(x_bshd, cos, sin, backward=False):
    """x [B,S,H,D] contiguous bf16; cos/sin [1|B, S, D] bf16 contiguous."""
    _want(x_bshd, torch.bfloat16, "x")
    _want(cos, torch.bfloat16, "cos")
    b, s, h, d = x_bshd.shape
    out = torch.empty_like(x_bshd)
    _check(_lib.load().ar_rope(_p(x_bshd), _p(cos), _p(sin), b, s, h, d, cos.shape[0], int(backward), _p(out), _stream()), "ar_rope")
    return out


def swiglu_fwd(gate, up):
    _want(gate, torch.bfloat16, "gate")
    h = torch.empty_like(gate)
    _check(_lib.load().ar_swiglu_fwd(_p(gate), _p(up), gate.numel(), _p(h), _stream()), "ar_swiglu_fwd")
    return h


def swiglu_bwd(dh, gate, up):
    dg, du = torch.empty_like(gate), torch.empty_like(up)
    _check(_lib.load().ar_swiglu_bwd(_p(dh), _p(gate), _p(up), gate.numel(), _p(dg), _p(du), _stream()), "ar_swiglu_bwd")
    return dg, du


# ------------------------------------------------------------------------------- optimized RTN / alg_ext searches
def int_search_table(bits: int, search_ratio: float = 0.75):
    """Candidate numerators of search_scales (auto_round/data_type/int.py:49-64), base candidate -2^(bits-1) first.
    Python double arithmetic as in the reference; the kernel multiplies the fp32 cast by the bf16 reciprocal."""
    nmax = int(2.0 ** (bits - 1))
    if bits == 2:
        half, step = 18 * 5, 0.01
    else:
        span = nmax * search_ratio
        step = span / 200 * 2
        half = int(span / step)
    return [float(-nmax)] + [-(nmax - step * i) for i in range(-half, half + 1) if i != 0]


NV_SEARCH_TABLE = [1.0] + [sv / 100.0 for sv in range(50, 152) if sv / 100.0 != 1.0]   # nvfp.py:359-364
MX_SEARCH_TABLE = [1.0, 0.5, 2.0]                                                        # mxfp.py:147


_TABLES = {}


def _table(key, values, device):
    k = (key, str(device))
    if k not in _TABLES:
        _TABLES[k] = torch.tensor(values, dtype=torch.float64).to(torch.float32).to(device)
    return _TABLES[k]


def _qw_args(qw, spec: Spec):
    if qw is None:
        return None, 0
    _want(qw, torch.float32, "qw")
    if qw.dim() == 1:
        if qw.numel() != spec.k:
            raise ValueError(f"importance vector has {qw.numel()} entries, weight has K={spec.k}")
        return qw, 0
    if qw.dim() != 2 or qw.shape[0] != spec.n or qw.shape[1] < spec.kpad:
        raise ValueError("importance matrix must be [N, >=Kpad]")
    return qw, qw.shape[1]


def search_scale_int(spec: Spec, w, qw=None, want_wq=True):
    """opt_rtn_int_sym (auto_round/data_type/int.py:89-122): returns (scale fp32 [G] holding bf16 values, wq bf16 | None)."""
    _want(w, torch.bfloat16, "w")
    qw, stride = _qw_args(qw, spec)
    coef = _table(("int", spec.bits), int_search_table(spec.bits), w.device)
    scale = torch.empty(spec.groups, dtype=torch.float32, device=w.device)
    wq = torch.empty_like(w) if want_wq else None
    cs = spec.c()
    _check(_lib.load().ar_search_scale_int(_p(w), _p(qw), stride, _p(coef), coef.numel(), C.byref(cs), _p(scale), _p(wq),
                                           _stream()), "ar_search_scale_int")
    return scale, wq


def search_scale_nv(spec: Spec, w, qw=None):
    """search_nvfp4_scale (auto_round/data_type/nvfp.py:331-385): per-group coefficient, fp32 [G]."""
    _want(w, torch.bfloat16, "w")
    qw, stride = _qw_args(qw, spec)
    coef = _table("nv", NV_SEARCH_TABLE, w.device)
    own_gs = nv_global_scale(w)                       # the search uses the tensor's own global scale
    out = torch.empty(spec.groups, dtype=torch.float32, device=w.device)
    cs = spec.c()
    _check(_lib.load().ar_search_scale_nv(_p(w), _p(qw), stride, _p(own_gs), _p(coef), coef.numel(), C.byref(cs), _p(out),
                                          _stream()), "ar_search_scale_nv")
    return out


def search_scale_mx(spec: Spec, w, qw=None):
    """search_mx_scale (auto_round/data_type/mxfp.py:103-169): per-group coefficient in {1, 0.5, 2}, fp32 [G]."""
    _want(w, torch.bfloat16, "w")
    qw, stride = _qw_args(qw, spec)
    coef = _table("mx", MX_SEARCH_TABLE, w.device)
    out = torch.empty(spec.groups, dtype=torch.float32, device=w.device)
    cs = spec.c()
    _check(_lib.load().ar_search_scale_mx(_p(w), _p(qw), stride, _p(coef), coef.numel(), C.byref(cs), _p(out), _stream()),
           "ar_search_scale_mx")
    return out


def imatrix_accum(x2d, imatrix):
    """imatrix[k] += sum_rows x^2 (algorithms/quantization/rtn/quantizer.py:86-105), in place."""
    _want(x2d, torch.bfloat16, "x")
    _want(imatrix, torch.float32, "imatrix")
    if x2d.dim() != 2 or imatrix.numel() != x2d.shape[1]:
        raise ValueError("imatrix_accum: x [rows, K], imatrix [K]")
    _check(_lib.load().ar_imatrix_accum(_p(x2d), x2d.shape[0], x2d.shape[1], _p(imatrix), _stream()), "ar_imatrix_accum")
    return imatrix


# ----------------------------------------------------------------------- enable_alg_ext: outlier-suppressed block loss
class OutlierSelect:
    """Device scratch of the top-k selection (sign_roundv2/quantizer.py:371-378): the 32768-bin histogram of the bf16
    pattern of |pred - ref| and sel = [threshold pattern, ties to drop, tie counter]."""

    def __init__(self, device):
        self.hist = torch.zeros(32768, dtype=torch.int32, device=device)
        self.sel = torch.zeros(4, dtype=torch.int32, device=device)
        self.hist_all = None                  # [world, 32768] under data parallelism


def mse_outlier_fwd_bwd(pred2d, ref2d, row_mask, upstream, loss_sum, scratch: OutlierSelect, dpred=None, want_grad=True,
                        numel_global=None, all_gather=None, rank=0, world=1):
    """SignRoundV2Quantizer._get_loss with its backward: drops the numel // 1000 largest |pred - ref| (selection on the
    bf16 difference, token mask ignored there), loss_sum (double [1]) += sum((|d| * mask * keep)^2); returns dpred bf16.
    Data parallel (world > 1): `pred2d` holds this rank's samples; the top-k and the mean run over the GLOBAL batch of
    `numel_global` elements -- `all_gather(out [world, 32768], local [32768])` exchanges the ranks' histograms."""
    _want(pred2d, torch.bfloat16, "pred")
    _want(ref2d, torch.bfloat16, "ref")
    _want(loss_sum, torch.float64, "loss_sum")
    if row_mask is not None:
        _want(row_mask, torch.uint8, "row_mask")
    rows, cols = pred2d.shape
    numel = rows * cols
    total = numel if numel_global is None else int(numel_global)
    k = max(1, int(total / 1000))
    if want_grad and dpred is None:
        dpred = torch.empty_like(pred2d)
    lib = _lib.load()
    _check(lib.ar_absdiff_hist(_p(pred2d), _p(ref2d), numel, _p(scratch.hist), _stream()), "ar_absdiff_hist")
    if world > 1:
        if scratch.hist_all is None or scratch.hist_all.shape[0] != world:
            scratch.hist_all = torch.zeros(world, scratch.hist.numel(), dtype=torch.int32, device=scratch.hist.device)
        all_gather(scratch.hist_all, scratch.hist)
        _check(lib.ar_topk_threshold_ranks(_p(scratch.hist_all), world, rank, _p(scratch.hist), k, _p(scratch.sel), _stream()),
               "ar_topk_threshold_ranks")
    else:
        _check(lib.ar_topk_threshold(_p(scratch.hist), k, _p(scratch.sel), _stream()), "ar_topk_threshold")
    _check(lib.ar_mse_outlier_fwd_bwd(_p(pred2d), _p(ref2d), _p(row_mask), rows, cols, 0 if numel_global is None else total,
                                      float(upstream), _p(scratch.sel), _p(loss_sum), _p(dpred if want_grad else None),
                                      _stream()), "ar_mse_outlier_fwd_bwd")
    return dpred
