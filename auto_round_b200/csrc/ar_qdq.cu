// Standalone fake-quant kernels: forward (Wq, scale, zp), backward (dV, d min/max_scale), group min/max,
// tensor amax.  HBM-bound elementwise work: 8 consecutive K-elements per lane (16 B bf16 loads, 2x16 B fp32
// loads), a quantisation group spans g/8 adjacent lanes of one warp, group reductions are shuffles.
//   algorithmic bytes / weight:  fwd 2 (W) + 4 (V) + 2 (Wq) = 8 B;  bwd 2 + 4 + 4 (Gq) + 4 (dV) = 14 B
#include "ar_qdq_math.cuh"

namespace ar {

constexpr int kThreads = 256;

struct QArgs {
  const uint16_t* w;
  const float* v;
  const float* mn;
  const float* mx;
  const uint16_t* wmin;
  const uint16_t* wmax;
  const float* gscale;
  int n, k, kpad, bits;
  float thr;
  const float* init;   // ar_qspec::init_scale (alg_ext) or null
};

template <int LPG>
__device__ __forceinline__ float group_max(float x) {
#pragma unroll
  for (int o = LPG / 2; o > 0; o >>= 1) x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, o));
  return x;
}
template <int LPG>
__device__ __forceinline__ float group_min(float x) {
#pragma unroll
  for (int o = LPG / 2; o > 0; o >>= 1) x = fminf(x, __shfl_xor_sync(0xffffffffu, x, o));
  return x;
}
template <int LPG>
__device__ __forceinline__ float group_sum(float x) {
#pragma unroll
  for (int o = LPG / 2; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}

// load 8 consecutive elements of row n starting at k0 (zero beyond K: the reference zero-pads K to a group multiple)
__device__ __forceinline__ void load_w8(const uint16_t* w, int64_t row_off, int k0, int k, bool vec, float (&out)[8]) {
  if (vec && k0 + 8 <= k) {
    const U4 r = *reinterpret_cast<const U4*>(w + row_off + k0);
    const uint32_t u[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      out[2 * i] = bf16_bits_to_f32((uint16_t)(u[i] & 0xffffu));
      out[2 * i + 1] = bf16_bits_to_f32((uint16_t)(u[i] >> 16));
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) out[i] = (k0 + i < k) ? bf16_bits_to_f32(w[row_off + k0 + i]) : 0.f;
  }
}
__device__ __forceinline__ void load_f8(const float* p, int64_t off, float (&out)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p + off);
  const float4 b = *reinterpret_cast<const float4*>(p + off + 4);
  out[0] = a.x; out[1] = a.y; out[2] = a.z; out[3] = a.w;
  out[4] = b.x; out[5] = b.y; out[6] = b.z; out[7] = b.w;
}

template <class Ctx, int G, bool IS_FP4>
__device__ __forceinline__ void make_group(const QArgs& a, int64_t gidx, const float (&w)[8], bool valid, Ctx& ctx,
                                           GroupIn& gi) {
  constexpr int LPG = G / 8;
  gi.thr = a.thr;
  gi.plain = (a.mn == nullptr) && (a.mx == nullptr);
  ctx.init(a.bits);
  gi.gscale = (IS_FP4 && a.gscale) ? *a.gscale : 0.f;
  gi.mn = (valid && a.mn) ? a.mn[gidx] : 1.f;
  gi.mx = (valid && a.mx) ? a.mx[gidx] : 1.f;
  gi.has_init = (a.init != nullptr);
  gi.init = (valid && a.init) ? a.init[gidx] : 1.f;
  if (IS_FP4) {
    float m = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) m = fmaxf(m, fabsf(w[i]));
    gi.wmax = group_max<LPG>(m);
    gi.wmin = 0.f;
  } else if (a.wmin != nullptr) {
    gi.wmin = valid ? bf16_bits_to_f32(a.wmin[gidx]) : 0.f;
    gi.wmax = valid ? bf16_bits_to_f32(a.wmax[gidx]) : 0.f;
  } else {
    float lo = 0.f, hi = 0.f;   // clamp(min, max=0) / clamp(max, min=0)
#pragma unroll
    for (int i = 0; i < 8; ++i) { lo = fminf(lo, w[i]); hi = fmaxf(hi, w[i]); }
    gi.wmin = group_min<LPG>(lo);
    gi.wmax = group_max<LPG>(hi);
  }
  ctx.setup(gi);
}

enum ScaleKind { SCALE_F16 = 0, SCALE_BF16 = 1, SCALE_F32 = 2 };

template <class Ctx, int G, bool IS_FP4, int SKIND>
__global__ void __launch_bounds__(kThreads) qdq_fwd_kernel(QArgs a, uint16_t* wq, void* scale_out, float* zp_out) {
  constexpr int LPG = G / 8;
  const int cpr = a.kpad / 8;                                  // 8-element chunks per (padded) row
  const int64_t total = (int64_t)a.n * cpr;
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  const bool valid = c < total;
  const int64_t cc = valid ? c : 0;
  const int n = (int)(cc / cpr);
  const int k0 = (int)(cc % cpr) * 8;
  const int64_t gidx = (int64_t)n * (a.kpad / G) + k0 / G;
  const bool vec = (a.k % 8) == 0;
  float w[8], v[8];
  load_w8(a.w, (int64_t)n * a.k, k0, a.k, vec, w);
  if (a.v) load_f8(a.v, (int64_t)n * a.kpad + k0, v);
  else {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = 0.f;
  }
  Ctx ctx;
  GroupIn gi;
  make_group<Ctx, G, IS_FP4>(a, gidx, w, valid, ctx, gi);
  if (!valid) return;
  if (wq != nullptr) {
    uint32_t packed[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint32_t lo = f32_to_bf16_bits(ctx.fwd(w[2 * i], v[2 * i]));
      const uint32_t hi = f32_to_bf16_bits(ctx.fwd(w[2 * i + 1], v[2 * i + 1]));
      packed[i] = lo | (hi << 16);
    }
    if (vec && k0 + 8 <= a.k) {
      *reinterpret_cast<U4*>(wq + (int64_t)n * a.k + k0) = U4{packed[0], packed[1], packed[2], packed[3]};
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if (k0 + i < a.k) wq[(int64_t)n * a.k + k0 + i] = (uint16_t)((packed[i / 2] >> (16 * (i & 1))) & 0xffffu);
    }
  }
  if ((k0 % G) == 0) {
    if (scale_out != nullptr) {
      const float s = ctx.scale_out();
      if (SKIND == SCALE_F16) reinterpret_cast<__half*>(scale_out)[gidx] = __float2half_rn(s);
      else if (SKIND == SCALE_BF16) reinterpret_cast<__nv_bfloat16*>(scale_out)[gidx] = __float2bfloat16_rn(s);
      else reinterpret_cast<float*>(scale_out)[gidx] = s;
    }
    if (zp_out != nullptr) zp_out[gidx] = ctx.zp_out();
  }
}

template <class Ctx, int G, bool IS_FP4>
__global__ void __launch_bounds__(kThreads) qdq_bwd_kernel(QArgs a, const float* gq, float* dv, float* dmin,
                                                           float* dmax, int accumulate) {
  constexpr int LPG = G / 8;
  const int cpr = a.kpad / 8;
  const int64_t total = (int64_t)a.n * cpr;
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  const bool valid = c < total;
  const int64_t cc = valid ? c : 0;
  const int n = (int)(cc / cpr);
  const int k0 = (int)(cc % cpr) * 8;
  const int64_t gidx = (int64_t)n * (a.kpad / G) + k0 / G;
  const bool vec = (a.k % 8) == 0;
  float w[8], v[8], g[8];
  load_w8(a.w, (int64_t)n * a.k, k0, a.k, vec, w);
  if (a.v) load_f8(a.v, (int64_t)n * a.kpad + k0, v);
  else {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = 0.f;
  }
  if (vec && k0 + 8 <= a.k) load_f8(gq, (int64_t)n * a.k + k0, g);
  else {
#pragma unroll
    for (int i = 0; i < 8; ++i) g[i] = (k0 + i < a.k) ? gq[(int64_t)n * a.k + k0 + i] : 0.f;
  }
  Ctx ctx;
  GroupIn gi;
  make_group<Ctx, G, IS_FP4>(a, gidx, w, valid, ctx, gi);
  GroupAcc acc;
  float d[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) ctx.bwd(w[i], v[i], g[i], d[i], acc);
  acc.a = group_sum<LPG>(acc.a);
  acc.b = group_sum<LPG>(acc.b);
  if (!valid) return;
  float* o = dv + (int64_t)n * a.kpad + k0;
  if (accumulate) {
    float old[8];
    load_f8(dv, (int64_t)n * a.kpad + k0, old);
#pragma unroll
    for (int i = 0; i < 8; ++i) d[i] += old[i];
  }
  *reinterpret_cast<float4*>(o) = make_float4(d[0], d[1], d[2], d[3]);
  *reinterpret_cast<float4*>(o + 4) = make_float4(d[4], d[5], d[6], d[7]);
  if ((k0 % G) == 0) {
    float gmn, gmx;
    ctx.finish(acc, gi, gmn, gmx);
    if (dmax) dmax[gidx] = accumulate ? dmax[gidx] + gmx : gmx;
    if (dmin) dmin[gidx] = accumulate ? dmin[gidx] + gmn : gmn;
  }
}

template <int G>
__global__ void __launch_bounds__(kThreads) group_minmax_kernel(QArgs a, uint16_t* omin, uint16_t* omax) {
  constexpr int LPG = G / 8;
  const int cpr = a.kpad / 8;
  const int64_t total = (int64_t)a.n * cpr;
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  const bool valid = c < total;
  const int64_t cc = valid ? c : 0;
  const int n = (int)(cc / cpr);
  const int k0 = (int)(cc % cpr) * 8;
  float w[8];
  load_w8(a.w, (int64_t)n * a.k, k0, a.k, (a.k % 8) == 0, w);
  float lo = 0.f, hi = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) { lo = fminf(lo, w[i]); hi = fmaxf(hi, w[i]); }
  lo = group_min<LPG>(lo);
  hi = group_max<LPG>(hi);
  if (valid && (k0 % G) == 0) {
    const int64_t gidx = (int64_t)n * (a.kpad / G) + k0 / G;
    omin[gidx] = f32_to_bf16_bits(lo);
    omax[gidx] = f32_to_bf16_bits(hi);
  }
}

__global__ void absmax_kernel(const uint16_t* w, int64_t numel, float* out) {
  float m = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < numel; i += (int64_t)gridDim.x * blockDim.x)
    m = fmaxf(m, fabsf(bf16_bits_to_f32(w[i])));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int*>(out), __float_as_int(m));  // m >= 0: int order == float order
}
__global__ void nv_gscale_kernel(const float* amax, float* gs) {
  const float a = fabsf(*amax);
  *gs = 448.f * 6.f * ((a == 0.f) ? 0.f : 1.f / a);   // FLOAT8_E4M3_MAX * FLOAT4_E2M1_MAX * get_reciprocal(amax)
}

// --------------------------------------------------------------------------------------------- dispatch
static int check_spec(const ar_qspec* q) {
  AR_REQUIRE(q != nullptr, AR_E_BADARG, "qspec is null");
  AR_REQUIRE(q->n > 0 && q->k > 0, AR_E_BADARG, "bad shape n=%d k=%d", q->n, q->k);
  const int g = q->group_size;
  const bool is_int_t = (q->dtype == AR_DT_INT_SYM || q->dtype == AR_DT_INT_ASYM);
  AR_REQUIRE(g == 16 || g == 32 || g == 64 || g == 128 || g == 256 || (is_int_t && g == q->k && q->k % 8 == 0), AR_E_UNSUPPORTED,
             "group_size %d not supported (16/32/64/128/256, or == K (per-row groups, int types, K %% 8 == 0))", g);
  if (q->dtype == AR_DT_INT_SYM || q->dtype == AR_DT_INT_ASYM)
    AR_REQUIRE(q->bits == 2 || q->bits == 3 || q->bits == 4 || q->bits == 8, AR_E_UNSUPPORTED, "int bits %d", q->bits);
  else if (q->dtype == AR_DT_MX_FP4 || q->dtype == AR_DT_NV_FP4)
    AR_REQUIRE(q->bits == 4, AR_E_UNSUPPORTED, "fp4 requires bits=4");
  else
    AR_REQUIRE(false, AR_E_BADARG, "unknown dtype %d", q->dtype);
  return AR_OK;
}

static bool row_mode(const ar_qspec* q) {
  const int g = q->group_size;
  return !(g == 16 || g == 32 || g == 64 || g == 128 || g == 256);
}

static QArgs make_args(const ar_qspec* q, const void* w, const float* v, const float* mn, const float* mx,
                       const void* wmin, const void* wmax, const float* gscale) {
  QArgs a;
  a.w = (const uint16_t*)w; a.v = v; a.mn = mn; a.mx = mx;
  a.wmin = (const uint16_t*)wmin; a.wmax = (const uint16_t*)wmax; a.gscale = gscale;
  a.n = q->n; a.k = q->k;
  a.kpad = (q->k + q->group_size - 1) / q->group_size * q->group_size;
  a.thr = q->q_scale_thresh;
  a.bits = q->bits;
  a.init = q->init_scale;
  return a;
}

template <class Ctx, bool FP4, int SK>
static void launch_fwd_g(int g, dim3 grid, cudaStream_t st, const QArgs& a, uint16_t* wq, void* so, float* zo) {
  switch (g) {
    case 16: qdq_fwd_kernel<Ctx, 16, FP4, SK><<<grid, kThreads, 0, st>>>(a, wq, so, zo); break;
    case 32: qdq_fwd_kernel<Ctx, 32, FP4, SK><<<grid, kThreads, 0, st>>>(a, wq, so, zo); break;
    case 64: qdq_fwd_kernel<Ctx, 64, FP4, SK><<<grid, kThreads, 0, st>>>(a, wq, so, zo); break;
    case 128: qdq_fwd_kernel<Ctx, 128, FP4, SK><<<grid, kThreads, 0, st>>>(a, wq, so, zo); break;
    default: qdq_fwd_kernel<Ctx, 256, FP4, SK><<<grid, kThreads, 0, st>>>(a, wq, so, zo); break;
  }
}
template <class Ctx, bool FP4>
static void launch_bwd_g(int g, dim3 grid, cudaStream_t st, const QArgs& a, const float* gq, float* dv, float* dmn,
                         float* dmx, int acc) {
  switch (g) {
    case 16: qdq_bwd_kernel<Ctx, 16, FP4><<<grid, kThreads, 0, st>>>(a, gq, dv, dmn, dmx, acc); break;
    case 32: qdq_bwd_kernel<Ctx, 32, FP4><<<grid, kThreads, 0, st>>>(a, gq, dv, dmn, dmx, acc); break;
    case 64: qdq_bwd_kernel<Ctx, 64, FP4><<<grid, kThreads, 0, st>>>(a, gq, dv, dmn, dmx, acc); break;
    case 128: qdq_bwd_kernel<Ctx, 128, FP4><<<grid, kThreads, 0, st>>>(a, gq, dv, dmn, dmx, acc); break;
    default: qdq_bwd_kernel<Ctx, 256, FP4><<<grid, kThreads, 0, st>>>(a, gq, dv, dmn, dmx, acc); break;
  }
}

// ------------------------------------------------------------------------------------ fused per-layer update
// One pass over a layer's weights per sign-SGD iteration (replaces: fused grad-w epilogue -> sign-SGD kernel -> next
// iteration's qdq forward, 30-34 B/weight in three launches):
//   Gq = dL/dWq (bf16, the plain grad-w GEMM's output; under data parallelism the reduce-scattered SUM over ranks)
//   fake-quant backward in registers (dV = Gq*s*mask, group sums -> d min/max_scale)            wrapper.py:273-290 autograd
//   best-param snapshot of the PRE-update parameters when *flag                                   quantizer.py:511-515
//   p <- p - lr_t * sign(grad), min/max_scale clamped to [0, clamp_hi]                            sign_sgd.py:369-389
//   Wq' = qdq(W; V', scales') for the NEXT iteration's forward / grad-in GEMMs                    wrapper.py:244-293
// Algorithmic bytes / weight: read 2 (W) + 4 (V) + 2 (Gq), write 4 (V') + 2 (Wq') = 14 B (+4 B when the snapshot fires).
// Rows [row0, row1) only: a data-parallel rank owns a row shard; `gq` is indexed from row `gq_row0`.
struct UpdArgs {
  const uint16_t* gq;      // bf16 [rows, K]
  int gq_row0, row0, row1;
  float* v;                // in/out [N, kpad]
  float* mn;               // in/out [G] or null
  float* mx;               // in/out [G]
  float* best_v;           // snapshot targets (null: no snapshot)
  float* best_mn;
  float* best_mx;
  const int32_t* flag;
  const float* lr_table;
  int iter;
  const int32_t* it_ptr;
  float clamp_hi;
  uint16_t* wq;            // out bf16 [N, K]
  // data-parallel wire form of the shard's new Wq (instead of `wq`): one u32 of eight 4-bit codes per chunk, indexed from row
  // row0, and {a, off} per group -- ar_wq_decode rebuilds bf16(a * (code - off)) (fp4: a * e2m1(code)) on every rank
  uint32_t* codes;
  float2* gparams;
  float* dv_dbg;           // optional pre-sign gradients (tests): [N, kpad], [G], [G]
  float* dmn_dbg;
  float* dmx_dbg;
  const int32_t* has_grad; // optional: *has_grad == 0 -> the layer received no gradient this iteration: leave it untouched
};

// p - lr * sign(g), with sign(0) = sign(NaN) = 0
__device__ __forceinline__ float sign_step(float p, float lr, float g) {
  return (g > 0.f || g < 0.f) ? p - copysignf(lr, g) : p;
}

template <class Ctx, int G, bool IS_FP4>
__global__ void __launch_bounds__(kThreads) fq_update_kernel(QArgs a, UpdArgs u) {
  constexpr int LPG = G / 8;
  // a layer without a gradient this iteration (an expert no token was routed to) is not stepped, but it still takes part
  // in the best-parameter snapshot: collect_best_params clones EVERY parameter (compressors/utils.py:205-217)
  const bool no_grad = (u.has_grad != nullptr) && (*u.has_grad == 0);
  const bool snap_any = (u.flag != nullptr) && (*u.flag != 0) && (u.best_v != nullptr);
  if (no_grad && !snap_any) return;
  const int cpr = a.kpad / 8;
  const int64_t total = (int64_t)(u.row1 - u.row0) * cpr;
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  const bool valid = c < total;
  const int64_t cc = valid ? c : 0;
  const int n = u.row0 + (int)(cc / cpr);
  const int k0 = (int)(cc % cpr) * 8;
  const int64_t gidx = (int64_t)n * (a.kpad / G) + k0 / G;
  const bool vec = (a.k % 8) == 0;
  const int iter = u.it_ptr ? *u.it_ptr : u.iter;
  const float lr_v = u.lr_table[2 * iter], lr_s = u.lr_table[2 * iter + 1];
  const bool snap = snap_any;
  if (no_grad) {                                     // snapshot only
    if (!valid) return;
    const int64_t vo = (int64_t)n * a.kpad + k0;
    *reinterpret_cast<float4*>(u.best_v + vo) = *reinterpret_cast<const float4*>(u.v + vo);
    *reinterpret_cast<float4*>(u.best_v + vo + 4) = *reinterpret_cast<const float4*>(u.v + vo + 4);
    if ((k0 % G) == 0) {
      if (u.best_mx) u.best_mx[gidx] = u.mx[gidx];
      if (u.best_mn && u.mn) u.best_mn[gidx] = u.mn[gidx];
    }
    return;
  }
  float w[8], v[8], g[8];
  load_w8(a.w, (int64_t)n * a.k, k0, a.k, vec, w);
  load_w8(u.gq, (int64_t)(n - u.gq_row0) * a.k, k0, a.k, vec, g);
  const int64_t voff = (int64_t)n * a.kpad + k0;
  load_f8(u.v, voff, v);
  a.v = u.v; a.mn = u.mn; a.mx = u.mx;
  Ctx ctx;
  GroupIn gi;
  make_group<Ctx, G, IS_FP4>(a, gidx, w, valid, ctx, gi);
  GroupAcc acc;
  float d[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) ctx.bwd(w[i], v[i], g[i], d[i], acc);
  acc.a = group_sum<LPG>(acc.a);
  acc.b = group_sum<LPG>(acc.b);
  if (!valid) return;
  float gmn, gmx;
  ctx.finish(acc, gi, gmn, gmx);
  const bool lead = (k0 % G) == 0;
  if (u.dv_dbg) {
    *reinterpret_cast<float4*>(u.dv_dbg + voff) = make_float4(d[0], d[1], d[2], d[3]);
    *reinterpret_cast<float4*>(u.dv_dbg + voff + 4) = make_float4(d[4], d[5], d[6], d[7]);
    if (lead && u.dmx_dbg) u.dmx_dbg[gidx] = gmx;
    if (lead && u.dmn_dbg) u.dmn_dbg[gidx] = gmn;
  }
  if (snap) {
    *reinterpret_cast<float4*>(u.best_v + voff) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(u.best_v + voff + 4) = make_float4(v[4], v[5], v[6], v[7]);
    if (lead) {
      if (u.best_mx) u.best_mx[gidx] = gi.mx;
      if (u.best_mn && u.mn) u.best_mn[gidx] = gi.mn;
    }
  }
  // sign-SGD step (every lane of a group derives the same new scales from the shuffled group sums)
#pragma unroll
  for (int i = 0; i < 8; ++i) v[i] = sign_step(v[i], lr_v, d[i]);
  *reinterpret_cast<float4*>(u.v + voff) = make_float4(v[0], v[1], v[2], v[3]);
  *reinterpret_cast<float4*>(u.v + voff + 4) = make_float4(v[4], v[5], v[6], v[7]);
  gi.mx = clampf(sign_step(gi.mx, lr_s, gmx), 0.f, u.clamp_hi);
  if (u.mn) gi.mn = clampf(sign_step(gi.mn, lr_s, gmn), 0.f, u.clamp_hi);
  if (lead) {
    u.mx[gidx] = gi.mx;
    if (u.mn) u.mn[gidx] = gi.mn;
  }
  // next iteration's fake-quant weight
  ctx.setup(gi);
  if (u.codes != nullptr) {                          // 4-bit wire codes + group parameters; the decode kernel writes Wq
    uint32_t word = 0u;
#pragma unroll
    for (int i = 0; i < 8; ++i) word |= (ctx.enc(w[i], v[i]) & 15u) << (4 * i);
    u.codes[(int64_t)(n - u.row0) * cpr + k0 / 8] = word;
    if (lead) {
      float pa, po;
      ctx.dec_params(pa, po);
      u.gparams[(int64_t)(n - u.row0) * (a.kpad / G) + k0 / G] = make_float2(pa, po);
    }
    return;
  }
  uint32_t packed[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t lo = f32_to_bf16_bits(ctx.fwd(w[2 * i], v[2 * i]));
    const uint32_t hi = f32_to_bf16_bits(ctx.fwd(w[2 * i + 1], v[2 * i + 1]));
    packed[i] = lo | (hi << 16);
  }
  if (vec && k0 + 8 <= a.k) {
    *reinterpret_cast<U4*>(u.wq + (int64_t)n * a.k + k0) = U4{packed[0], packed[1], packed[2], packed[3]};
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if (k0 + i < a.k) u.wq[(int64_t)n * a.k + k0 + i] = (uint16_t)((packed[i / 2] >> (16 * (i & 1))) & 0xffffu);
  }
}

// Rebuild the bf16 fake-quant weight of a whole layer from the all-gathered wire segments: rank r's segment holds the codes
// (u32 per 8 elements) and then the {a, off} pairs of its rows [r * rows_per_rank, (r + 1) * rows_per_rank).
__global__ void __launch_bounds__(kThreads) wq_decode_kernel(const uint8_t* __restrict__ seg_all, int64_t seg_bytes,
                                                            int rows_per_rank, int n, int k, int kpad, int g, int is_fp4,
                                                            uint16_t* __restrict__ wq) {
  const int cpr = kpad / 8, gpr = kpad / g;
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (c >= (int64_t)n * cpr) return;
  const int row = (int)(c / cpr), k0 = (int)(c % cpr) * 8;
  const int r = row / rows_per_rank, lrow = row - r * rows_per_rank;
  const uint8_t* seg = seg_all + (int64_t)r * seg_bytes;
  const uint32_t word = reinterpret_cast<const uint32_t*>(seg)[(int64_t)lrow * cpr + k0 / 8];
  const float2 pr = reinterpret_cast<const float2*>(seg + (int64_t)rows_per_rank * cpr * 4)[(int64_t)lrow * gpr + k0 / g];
  uint32_t packed[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t n0 = (word >> (8 * i)) & 15u, n1 = (word >> (8 * i + 4)) & 15u;
    const float f0 = is_fp4 ? e2m1_dec(n0) * pr.x : pr.x * ((float)n0 - pr.y);
    const float f1 = is_fp4 ? e2m1_dec(n1) * pr.x : pr.x * ((float)n1 - pr.y);
    packed[i] = (uint32_t)f32_to_bf16_bits(f0) | ((uint32_t)f32_to_bf16_bits(f1) << 16);
  }
  if ((k % 8) == 0 && k0 + 8 <= k) {
    *reinterpret_cast<U4*>(wq + (int64_t)row * k + k0) = U4{packed[0], packed[1], packed[2], packed[3]};
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if (k0 + i < k) wq[(int64_t)row * k + k0 + i] = (uint16_t)((packed[i / 2] >> (16 * (i & 1))) & 0xffffu);
  }
}

template <class Ctx, bool FP4>
static void launch_upd_g(int g, dim3 grid, cudaStream_t st, const QArgs& a, const UpdArgs& u) {
  switch (g) {
    case 16: fq_update_kernel<Ctx, 16, FP4><<<grid, kThreads, 0, st>>>(a, u); break;
    case 32: fq_update_kernel<Ctx, 32, FP4><<<grid, kThreads, 0, st>>>(a, u); break;
    case 64: fq_update_kernel<Ctx, 64, FP4><<<grid, kThreads, 0, st>>>(a, u); break;
    case 128: fq_update_kernel<Ctx, 128, FP4><<<grid, kThreads, 0, st>>>(a, u); break;
    default: fq_update_kernel<Ctx, 256, FP4><<<grid, kThreads, 0, st>>>(a, u); break;
  }
}

// ------------------------------------------------------------------------------------------ per-row groups
// group_size = -1 (per output channel) or K < group_size: the reference keeps the weight as [N, K] and every ROW is one
// group (reshape_pad_tensor_by_group_size, data_type/utils.py:57-61).  One warp per row, lanes stride over 8-element chunks;
// int types only (the fp4 formats fix their group size).  K % 8 == 0.
constexpr int kRowWarps = kThreads / 32;

template <class Ctx>
__device__ __forceinline__ void row_group_in(const QArgs& a, int row, int lane, GroupIn& gi, Ctx& ctx) {
  gi.thr = a.thr;
  gi.plain = (a.mn == nullptr) && (a.mx == nullptr);
  gi.gscale = 0.f;
  gi.mn = a.mn ? a.mn[row] : 1.f;
  gi.mx = a.mx ? a.mx[row] : 1.f;
  gi.has_init = (a.init != nullptr);
  gi.init = a.init ? a.init[row] : 1.f;
  ctx.init(a.bits);
  if (a.wmin != nullptr) {
    gi.wmin = bf16_bits_to_f32(a.wmin[row]);
    gi.wmax = bf16_bits_to_f32(a.wmax[row]);
  } else {
    float lo = 0.f, hi = 0.f;
    for (int c = lane; c < a.k / 8; c += 32) {
      float w[8];
      load_w8(a.w, (int64_t)row * a.k, c * 8, a.k, true, w);
#pragma unroll
      for (int i = 0; i < 8; ++i) { lo = fminf(lo, w[i]); hi = fmaxf(hi, w[i]); }
    }
    gi.wmin = group_min<32>(lo);
    gi.wmax = group_max<32>(hi);
  }
  ctx.setup(gi);
}

__global__ void __launch_bounds__(kThreads) group_minmax_row_kernel(QArgs a, uint16_t* omin, uint16_t* omax) {
  const int row = blockIdx.x * kRowWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= a.n) return;
  float lo = 0.f, hi = 0.f;
  for (int c = lane; c < a.k / 8; c += 32) {
    float w[8];
    load_w8(a.w, (int64_t)row * a.k, c * 8, a.k, true, w);
#pragma unroll
    for (int i = 0; i < 8; ++i) { lo = fminf(lo, w[i]); hi = fmaxf(hi, w[i]); }
  }
  lo = group_min<32>(lo);
  hi = group_max<32>(hi);
  if (lane == 0) { omin[row] = f32_to_bf16_bits(lo); omax[row] = f32_to_bf16_bits(hi); }
}

template <class Ctx>
__global__ void __launch_bounds__(kThreads) qdq_fwd_row_kernel(QArgs a, uint16_t* wq, __half* scale_out, float* zp_out) {
  const int row = blockIdx.x * kRowWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= a.n) return;
  Ctx ctx;
  GroupIn gi;
  row_group_in<Ctx>(a, row, lane, gi, ctx);
  if (wq != nullptr) {
    for (int c = lane; c < a.k / 8; c += 32) {
      float w[8], v[8];
      load_w8(a.w, (int64_t)row * a.k, c * 8, a.k, true, w);
      if (a.v) load_f8(a.v, (int64_t)row * a.k + c * 8, v);
      uint32_t packed[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint32_t lo = f32_to_bf16_bits(ctx.fwd(w[2 * i], a.v ? v[2 * i] : 0.f));
        const uint32_t hi = f32_to_bf16_bits(ctx.fwd(w[2 * i + 1], a.v ? v[2 * i + 1] : 0.f));
        packed[i] = lo | (hi << 16);
      }
      *reinterpret_cast<U4*>(wq + (int64_t)row * a.k + c * 8) = U4{packed[0], packed[1], packed[2], packed[3]};
    }
  }
  if (lane == 0) {
    if (scale_out) scale_out[row] = __float2half_rn(ctx.scale_out());
    if (zp_out) zp_out[row] = ctx.zp_out();
  }
}

template <class Ctx>
__global__ void __launch_bounds__(kThreads) fq_update_row_kernel(QArgs a, UpdArgs u) {
  const int row = u.row0 + blockIdx.x * kRowWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= u.row1) return;
  const bool no_grad = (u.has_grad != nullptr) && (*u.has_grad == 0);
  const bool snap = (u.flag != nullptr) && (*u.flag != 0) && (u.best_v != nullptr);
  if (no_grad && !snap) return;
  const int iter = u.it_ptr ? *u.it_ptr : u.iter;
  const float lr_v = u.lr_table[2 * iter], lr_s = u.lr_table[2 * iter + 1];
  a.v = u.v; a.mn = u.mn; a.mx = u.mx;
  Ctx ctx;
  GroupIn gi;
  row_group_in<Ctx>(a, row, lane, gi, ctx);
  const int64_t wrow = (int64_t)row * a.k, grow = (int64_t)(row - u.gq_row0) * a.k;
  if (no_grad) {                                     // snapshot only (see fq_update_kernel)
    for (int c = lane; c < a.k / 8; c += 32) {
      *reinterpret_cast<float4*>(u.best_v + wrow + c * 8) = *reinterpret_cast<const float4*>(u.v + wrow + c * 8);
      *reinterpret_cast<float4*>(u.best_v + wrow + c * 8 + 4) = *reinterpret_cast<const float4*>(u.v + wrow + c * 8 + 4);
    }
    if (lane == 0) { if (u.best_mx) u.best_mx[row] = gi.mx; if (u.best_mn && u.mn) u.best_mn[row] = gi.mn; }
    return;
  }
  // pass 1: the group sums of the scale gradients
  GroupAcc acc;
  for (int c = lane; c < a.k / 8; c += 32) {
    float w[8], v[8], g[8], d;
    load_w8(a.w, wrow, c * 8, a.k, true, w);
    load_w8(u.gq, grow, c * 8, a.k, true, g);
    load_f8(u.v, wrow + c * 8, v);
#pragma unroll
    for (int i = 0; i < 8; ++i) ctx.bwd(w[i], v[i], g[i], d, acc);
  }
  acc.a = group_sum<32>(acc.a);
  acc.b = group_sum<32>(acc.b);
  float gmn, gmx;
  ctx.finish(acc, gi, gmn, gmx);
  const float old_mn = gi.mn, old_mx = gi.mx;
  Ctx next = ctx;
  GroupIn gn = gi;
  gn.mx = clampf(sign_step(gi.mx, lr_s, gmx), 0.f, u.clamp_hi);
  if (u.mn) gn.mn = clampf(sign_step(gi.mn, lr_s, gmn), 0.f, u.clamp_hi);
  next.setup(gn);
  // pass 2: dV again (same parameters), snapshot, step, next iteration's fake-quant weight
  for (int c = lane; c < a.k / 8; c += 32) {
    float w[8], v[8], g[8], d[8];
    GroupAcc dummy;
    load_w8(a.w, wrow, c * 8, a.k, true, w);
    load_w8(u.gq, grow, c * 8, a.k, true, g);
    load_f8(u.v, wrow + c * 8, v);
#pragma unroll
    for (int i = 0; i < 8; ++i) ctx.bwd(w[i], v[i], g[i], d[i], dummy);
    if (u.dv_dbg) {
      *reinterpret_cast<float4*>(u.dv_dbg + wrow + c * 8) = make_float4(d[0], d[1], d[2], d[3]);
      *reinterpret_cast<float4*>(u.dv_dbg + wrow + c * 8 + 4) = make_float4(d[4], d[5], d[6], d[7]);
    }
    if (snap) {
      *reinterpret_cast<float4*>(u.best_v + wrow + c * 8) = make_float4(v[0], v[1], v[2], v[3]);
      *reinterpret_cast<float4*>(u.best_v + wrow + c * 8 + 4) = make_float4(v[4], v[5], v[6], v[7]);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = sign_step(v[i], lr_v, d[i]);
    *reinterpret_cast<float4*>(u.v + wrow + c * 8) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(u.v + wrow + c * 8 + 4) = make_float4(v[4], v[5], v[6], v[7]);
    uint32_t packed[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint32_t lo = f32_to_bf16_bits(next.fwd(w[2 * i], v[2 * i]));
      const uint32_t hi = f32_to_bf16_bits(next.fwd(w[2 * i + 1], v[2 * i + 1]));
      packed[i] = lo | (hi << 16);
    }
    *reinterpret_cast<U4*>(u.wq + wrow + c * 8) = U4{packed[0], packed[1], packed[2], packed[3]};
  }
  if (lane == 0) {
    if (u.dmx_dbg) u.dmx_dbg[row] = gmx;
    if (u.dmn_dbg) u.dmn_dbg[row] = gmn;
    if (snap) { if (u.best_mx) u.best_mx[row] = old_mx; if (u.best_mn && u.mn) u.best_mn[row] = old_mn; }
    u.mx[row] = gn.mx;
    if (u.mn) u.mn[row] = gn.mn;
  }
}

}  // namespace ar

using namespace ar;

extern "C" int ar_qdq_fwd(const ar_qspec* q, const void* w, const float* v, const float* mn, const float* mx,
                          const void* wmin, const void* wmax, const float* gscale, void* wq, void* scale_out,
                          float* zp_out, void* stream) {
  if (int rc = check_spec(q)) return rc;
  AR_REQUIRE(w != nullptr, AR_E_BADARG, "w is null");
  AR_REQUIRE((wmin == nullptr) == (wmax == nullptr), AR_E_BADARG, "wmin/wmax must both be given or both null");
  AR_REQUIRE(q->dtype != AR_DT_NV_FP4 || gscale != nullptr, AR_E_BADARG, "nv_fp4 needs gscale");
  const QArgs a = make_args(q, w, v, mn, mx, wmin, wmax, gscale);
  cudaStream_t st = (cudaStream_t)stream;
  if (row_mode(q)) {
    const dim3 rgrid((unsigned)((a.n + kRowWarps - 1) / kRowWarps));
    if (q->dtype == AR_DT_INT_SYM) qdq_fwd_row_kernel<IntSym><<<rgrid, kThreads, 0, st>>>(a, (uint16_t*)wq, (__half*)scale_out, nullptr);
    else qdq_fwd_row_kernel<IntAsym><<<rgrid, kThreads, 0, st>>>(a, (uint16_t*)wq, (__half*)scale_out, zp_out);
    AR_CHECK_LAUNCH();
    return AR_OK;
  }
  const int64_t chunks = (int64_t)a.n * (a.kpad / 8);
  const dim3 grid((unsigned)((chunks + kThreads - 1) / kThreads));
  const int g = q->group_size;
  if (q->dtype == AR_DT_INT_SYM) {
    launch_fwd_g<IntSym, false, SCALE_F16>(g, grid, st, a, (uint16_t*)wq, scale_out, nullptr);
  } else if (q->dtype == AR_DT_INT_ASYM) {
    launch_fwd_g<IntAsym, false, SCALE_F16>(g, grid, st, a, (uint16_t*)wq, scale_out, zp_out);
  } else if (q->dtype == AR_DT_MX_FP4) {
    launch_fwd_g<MxFp4, true, SCALE_BF16>(g, grid, st, a, (uint16_t*)wq, scale_out, nullptr);
  } else {
    launch_fwd_g<NvFp4, true, SCALE_F32>(g, grid, st, a, (uint16_t*)wq, scale_out, nullptr);
  }
  AR_CHECK_LAUNCH();
  return AR_OK;
}

extern "C" int ar_qdq_bwd(const ar_qspec* q, const void* w, const float* v, const float* mn, const float* mx,
                          const void* wmin, const void* wmax, const float* gscale, const float* gq, float* dv,
                          float* dmin, float* dmax, int accumulate, void* stream) {
  if (int rc = check_spec(q)) return rc;
  AR_REQUIRE(w && gq && dv, AR_E_BADARG, "w/gq/dv must be non-null");
  AR_REQUIRE(!row_mode(q), AR_E_UNSUPPORTED, "ar_qdq_bwd: per-row groups are served by ar_fq_update only");
  AR_REQUIRE((wmin == nullptr) == (wmax == nullptr), AR_E_BADARG, "wmin/wmax must both be given or both null");
  AR_REQUIRE(q->dtype != AR_DT_NV_FP4 || gscale != nullptr, AR_E_BADARG, "nv_fp4 needs gscale");
  const QArgs a = make_args(q, w, v, mn, mx, wmin, wmax, gscale);
  const int64_t chunks = (int64_t)a.n * (a.kpad / 8);
  const dim3 grid((unsigned)((chunks + kThreads - 1) / kThreads));
  cudaStream_t st = (cudaStream_t)stream;
  const int g = q->group_size;
  if (q->dtype == AR_DT_INT_SYM) {
    launch_bwd_g<IntSym, false>(g, grid, st, a, gq, dv, dmin, dmax, accumulate);
  } else if (q->dtype == AR_DT_INT_ASYM) {
    launch_bwd_g<IntAsym, false>(g, grid, st, a, gq, dv, dmin, dmax, accumulate);
  } else if (q->dtype == AR_DT_MX_FP4) {
    launch_bwd_g<MxFp4, true>(g, grid, st, a, gq, dv, dmin, dmax, accumulate);
  } else {
    launch_bwd_g<NvFp4, true>(g, grid, st, a, gq, dv, dmin, dmax, accumulate);
  }
  AR_CHECK_LAUNCH();
  return AR_OK;
}

extern "C" int ar_group_minmax(const ar_qspec* q, const void* w, void* wmin, void* wmax, void* stream) {
  if (int rc = check_spec(q)) return rc;
  AR_REQUIRE(w && wmin && wmax, AR_E_BADARG, "null pointer");
  const QArgs a = make_args(q, w, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
  cudaStream_t st = (cudaStream_t)stream;
  if (row_mode(q)) {
    group_minmax_row_kernel<<<(unsigned)((a.n + kRowWarps - 1) / kRowWarps), kThreads, 0, st>>>(a, (uint16_t*)wmin, (uint16_t*)wmax);
    AR_CHECK_LAUNCH();
    return AR_OK;
  }
  const int64_t chunks = (int64_t)a.n * (a.kpad / 8);
  const dim3 grid((unsigned)((chunks + kThreads - 1) / kThreads));
  switch (q->group_size) {
    case 16: group_minmax_kernel<16><<<grid, kThreads, 0, st>>>(a, (uint16_t*)wmin, (uint16_t*)wmax); break;
    case 32: group_minmax_kernel<32><<<grid, kThreads, 0, st>>>(a, (uint16_t*)wmin, (uint16_t*)wmax); break;
    case 64: group_minmax_kernel<64><<<grid, kThreads, 0, st>>>(a, (uint16_t*)wmin, (uint16_t*)wmax); break;
    case 128: group_minmax_kernel<128><<<grid, kThreads, 0, st>>>(a, (uint16_t*)wmin, (uint16_t*)wmax); break;
    default: group_minmax_kernel<256><<<grid, kThreads, 0, st>>>(a, (uint16_t*)wmin, (uint16_t*)wmax); break;
  }
  AR_CHECK_LAUNCH();
  return AR_OK;
}

extern "C" int ar_absmax(const void* w, int64_t numel, float* amax, void* stream) {
  AR_REQUIRE(w && amax && numel > 0, AR_E_BADARG, "bad args");
  const int blocks = (int)((numel + 256 * 16 - 1) / (256 * 16));
  absmax_kernel<<<blocks < 2048 ? (blocks > 0 ? blocks : 1) : 2048, 256, 0, (cudaStream_t)stream>>>(
      (const uint16_t*)w, numel, amax);
  AR_CHECK_LAUNCH();
  return AR_OK;
}
extern "C" int ar_nv_global_scale(const float* amax, float* gs, void* stream) {
  AR_REQUIRE(amax && gs, AR_E_BADARG, "bad args");
  nv_gscale_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(amax, gs);
  AR_CHECK_LAUNCH();
  return AR_OK;
}

extern "C" int ar_fq_update(const ar_qspec* q, const void* w, float* v, float* mn, float* mx, const void* wmin,
                            const void* wmax, const float* gscale, const void* gq, int gq_row0, int row0, int row1,
                            float* best_v, float* best_mn, float* best_mx, const int32_t* flag, const float* lr_table,
                            int iter, const int32_t* it_ptr, float clamp_hi, void* wq_out, float* dv_dbg, float* dmn_dbg,
                            float* dmx_dbg, const int32_t* has_grad, void* codes_out, void* gparams_out, void* stream) {
  if (int rc = check_spec(q)) return rc;
  AR_REQUIRE(w && v && mx && gq && lr_table && (wq_out || codes_out), AR_E_BADARG,
             "w/v/max_scale/gq/lr_table and wq_out (or codes_out) must be non-null");
  AR_REQUIRE((codes_out == nullptr) == (gparams_out == nullptr), AR_E_BADARG, "codes_out and gparams_out go together");
  AR_REQUIRE(codes_out == nullptr || (q->bits <= 4 && !row_mode(q)), AR_E_UNSUPPORTED,
             "the 4-bit wire form exists for bits <= 4 and grouped (not per-row) layouts");
  AR_REQUIRE((wmin == nullptr) == (wmax == nullptr), AR_E_BADARG, "wmin/wmax must both be given or both null");
  AR_REQUIRE(q->dtype != AR_DT_NV_FP4 || gscale != nullptr, AR_E_BADARG, "nv_fp4 needs gscale");
  AR_REQUIRE(0 <= row0 && row0 <= row1 && row1 <= q->n && gq_row0 <= row0 && iter >= 0, AR_E_BADARG,
             "bad row range [%d,%d) of %d (gq from row %d)", row0, row1, q->n, gq_row0);
  if (row0 == row1) return AR_OK;
  const QArgs a = make_args(q, w, v, mn, mx, wmin, wmax, gscale);
  UpdArgs u;
  u.gq = (const uint16_t*)gq; u.gq_row0 = gq_row0; u.row0 = row0; u.row1 = row1;
  u.v = v; u.mn = mn; u.mx = mx; u.best_v = best_v; u.best_mn = best_mn; u.best_mx = best_mx; u.flag = flag;
  u.lr_table = lr_table; u.iter = iter; u.it_ptr = it_ptr; u.clamp_hi = clamp_hi; u.wq = (uint16_t*)wq_out;
  u.dv_dbg = dv_dbg; u.dmn_dbg = dmn_dbg; u.dmx_dbg = dmx_dbg; u.has_grad = has_grad;
  u.codes = (uint32_t*)codes_out; u.gparams = (float2*)gparams_out;
  cudaStream_t st = (cudaStream_t)stream;
  if (row_mode(q)) {
    const dim3 rgrid((unsigned)((row1 - row0 + kRowWarps - 1) / kRowWarps));
    if (q->dtype == AR_DT_INT_SYM) fq_update_row_kernel<IntSym><<<rgrid, kThreads, 0, st>>>(a, u);
    else fq_update_row_kernel<IntAsym><<<rgrid, kThreads, 0, st>>>(a, u);
    AR_CHECK_LAUNCH();
    return AR_OK;
  }
  const int64_t chunks = (int64_t)(row1 - row0) * (a.kpad / 8);
  const dim3 grid((unsigned)((chunks + kThreads - 1) / kThreads));
  const int g = q->group_size;
  if (q->dtype == AR_DT_INT_SYM) launch_upd_g<IntSym, false>(g, grid, st, a, u);
  else if (q->dtype == AR_DT_INT_ASYM) launch_upd_g<IntAsym, false>(g, grid, st, a, u);
  else if (q->dtype == AR_DT_MX_FP4) launch_upd_g<MxFp4, true>(g, grid, st, a, u);
  else launch_upd_g<NvFp4, true>(g, grid, st, a, u);
  AR_CHECK_LAUNCH();
  return AR_OK;
}

extern "C" int ar_wq_decode(const ar_qspec* q, const void* segments, int64_t seg_bytes, int world, void* wq_out, void* stream) {
  if (int rc = check_spec(q)) return rc;
  AR_REQUIRE(segments && wq_out && world >= 1 && q->n % world == 0, AR_E_BADARG, "ar_wq_decode: bad arguments (rows must split evenly)");
  AR_REQUIRE(q->bits <= 4 && !row_mode(q), AR_E_UNSUPPORTED, "ar_wq_decode: bits <= 4, grouped layouts");
  const int g = q->group_size;
  const int kpad = (q->k + g - 1) / g * g;
  const int rows = q->n / world;
  AR_REQUIRE(seg_bytes >= (int64_t)rows * (kpad / 8) * 4 + (int64_t)rows * (kpad / g) * 8, AR_E_BADARG, "ar_wq_decode: segment too small");
  const int64_t chunks = (int64_t)q->n * (kpad / 8);
  const int fp4 = (q->dtype == AR_DT_MX_FP4 || q->dtype == AR_DT_NV_FP4) ? 1 : 0;
  wq_decode_kernel<<<(unsigned)((chunks + kThreads - 1) / kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      (const uint8_t*)segments, seg_bytes, rows, q->n, q->k, kpad, g, fp4, (uint16_t*)wq_out);
  AR_CHECK_LAUNCH();
  return AR_OK;
}
