// Fused elementwise ops of a Llama-family decoder block (the glue between the fake-quant linears inside the
// sign-SGD iteration): RMSNorm, rotary embedding, SwiGLU -- forward and backward, one HBM pass each.
// They replace ~40 ATen elementwise launches per iteration with 10.  Forward values reproduce the HF eager op order bit-for-bit
// (fp32 math, bf16 rounding at the same points):
//   LlamaRMSNorm.forward      transformers/models/llama/modeling_llama.py  (x.float() -> *rsqrt(mean(x^2)+eps) -> bf16 -> *w)
//   apply_rotary_pos_emb      (q*cos) + (rotate_half(q)*sin), each product and the sum rounded to bf16
//   LlamaMLP.forward          act_fn(gate) * up  with silu rounded to bf16 before the product
// Algorithmic bytes/element: rmsnorm fwd 4 (2 in, 2 out), bwd 6; rope 4 + tables; swiglu fwd 6, bwd 10.
#include "ar_common.cuh"

namespace ar {

__device__ __forceinline__ void unpack8f(const U4& r, float (&o)[8]) {
  const uint32_t u[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    o[2 * i] = bf16_bits_to_f32((uint16_t)(u[i] & 0xffffu));
    o[2 * i + 1] = bf16_bits_to_f32((uint16_t)(u[i] >> 16));
  }
}
__device__ __forceinline__ U4 pack8f(const float (&v)[8]) {
  uint32_t p[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) p[i] = (uint32_t)f32_to_bf16_bits(v[2 * i]) | ((uint32_t)f32_to_bf16_bits(v[2 * i + 1]) << 16);
  return U4{p[0], p[1], p[2], p[3]};
}

__device__ __forceinline__ float block_sum(float v, float* smem) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if ((threadIdx.x & 31) == 0) smem[w] = v;
  __syncthreads();
  float t = 0.f;
  for (int i = 0; i < nw; ++i) t += smem[i];
  __syncthreads();
  return t;
}

// ---------------------------------------------------------------------------------------------- RMSNorm
// one block per row; VPT vectors of 8 elements per thread are kept in registers (H = blockDim * 8 * VPT)
template <int VPT>
__global__ void __launch_bounds__(256) rmsnorm_fwd_kernel(const U4* __restrict__ x, const U4* __restrict__ w, float eps, int h8,
                                                          U4* __restrict__ y, float* __restrict__ rstd) {
  __shared__ float red[8];
  const int64_t row = blockIdx.x;
  float v[VPT][8];
  float ss = 0.f;
#pragma unroll
  for (int j = 0; j < VPT; ++j) {
    const int c = threadIdx.x + j * blockDim.x;
    if (c < h8) {
      unpack8f(x[row * h8 + c], v[j]);
#pragma unroll
      for (int i = 0; i < 8; ++i) ss += v[j][i] * v[j][i];
    }
  }
  ss = block_sum(ss, red);
  const float r = rsqrtf(ss / (float)(h8 * 8) + eps);
  if (threadIdx.x == 0 && rstd) rstd[row] = r;
#pragma unroll
  for (int j = 0; j < VPT; ++j) {
    const int c = threadIdx.x + j * blockDim.x;
    if (c < h8) {
      float wv[8], o[8];
      unpack8f(w[c], wv);
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = wv[i] * bf16_round(v[j][i] * r);      // weight * hidden.to(bf16)
      y[row * h8 + c] = pack8f(o);
    }
  }
}

// dx = r * (dn - n * mean(dn * n)),  n = x*r,  dn = bf16(dy * w)   (autograd of the HF graph, fp32 inside)
template <int VPT>
__global__ void __launch_bounds__(256) rmsnorm_bwd_kernel(const U4* __restrict__ dy, const U4* __restrict__ x,
                                                          const U4* __restrict__ w, const float* __restrict__ rstd, int h8,
                                                          U4* __restrict__ dx, int accumulate) {
  __shared__ float red[8];
  const int64_t row = blockIdx.x;
  const float r = rstd[row];
  float n[VPT][8], dn[VPT][8];
  float dot = 0.f;
#pragma unroll
  for (int j = 0; j < VPT; ++j) {
    const int c = threadIdx.x + j * blockDim.x;
    if (c < h8) {
      float xv[8], gv[8], wv[8];
      unpack8f(x[row * h8 + c], xv);
      unpack8f(dy[row * h8 + c], gv);
      unpack8f(w[c], wv);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        n[j][i] = xv[i] * r;
        dn[j][i] = bf16_round(gv[i] * wv[i]);
        dot += dn[j][i] * n[j][i];
      }
    }
  }
  dot = block_sum(dot, red) / (float)(h8 * 8);
#pragma unroll
  for (int j = 0; j < VPT; ++j) {
    const int c = threadIdx.x + j * blockDim.x;
    if (c < h8) {
      float o[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = r * (dn[j][i] - n[j][i] * dot);
      if (accumulate) {                      // residual stream: dx += (gradient arriving through the skip path)
        float old[8];
        unpack8f(dx[row * h8 + c], old);
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] = bf16_round(o[i]) + old[i];
      }
      dx[row * h8 + c] = pack8f(o);
    }
  }
}

// ------------------------------------------------------------------------------------------------- RoPE
// x laid out [B, S, H, D] (the projection output viewed per head), cos/sin [Bc, S, D] (Bc = 1 or B).
// One thread = 8 elements of the first half + the matching 8 of the second half of one head vector.
// fwd: out = x*cos + rotate_half(x)*sin ; bwd (transpose): dx = g*cos - rotate_half(g*sin)  (rotate_half(v) = [-v2, v1])
template <bool BWD>
__global__ void __launch_bounds__(256) rope_kernel(const uint16_t* __restrict__ x, const uint16_t* __restrict__ cs,
                                                   const uint16_t* __restrict__ sn, int64_t total, int s, int h, int d,
                                                   int bc_is_one, uint16_t* __restrict__ out) {
  const int half8 = d / 16;                               // vectors of 8 in one half
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int v = (int)(i % half8);
  const int64_t vec = i / half8;                          // (b, s, h) index
  const int64_t bs = vec / h;                             // b*S + s
  const int64_t tab = (bc_is_one ? (bs % s) : bs) * d;
  const uint16_t* px = x + vec * d;
  float a[8], b[8], c1[8], c2[8], s1[8], s2[8], o1[8], o2[8];
  unpack8f(*reinterpret_cast<const U4*>(px + v * 8), a);
  unpack8f(*reinterpret_cast<const U4*>(px + d / 2 + v * 8), b);
  unpack8f(*reinterpret_cast<const U4*>(cs + tab + v * 8), c1);
  unpack8f(*reinterpret_cast<const U4*>(cs + tab + d / 2 + v * 8), c2);
  unpack8f(*reinterpret_cast<const U4*>(sn + tab + v * 8), s1);
  unpack8f(*reinterpret_cast<const U4*>(sn + tab + d / 2 + v * 8), s2);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    if (!BWD) {
      // (x*cos) + (rotate_half(x)*sin): bf16 rounding of each product, of the negation (exact) and of the sum
      o1[j] = bf16_round(a[j] * c1[j]) + bf16_round((-b[j]) * s1[j]);
      o2[j] = bf16_round(b[j] * c2[j]) + bf16_round(a[j] * s2[j]);
    } else {
      // dx1 = g1*cos1 + g2*sin2 ; dx2 = g2*cos2 - g1*sin1
      o1[j] = a[j] * c1[j] + b[j] * s2[j];
      o2[j] = b[j] * c2[j] - a[j] * s1[j];
    }
  }
  uint16_t* po = out + vec * d;
  *reinterpret_cast<U4*>(po + v * 8) = pack8f(o1);
  *reinterpret_cast<U4*>(po + d / 2 + v * 8) = pack8f(o2);
}

// ----------------------------------------------------------------------------------------------- SwiGLU
__device__ __forceinline__ float silu_f(float x) { return x / (1.f + expf(-x)); }

__global__ void __launch_bounds__(256) swiglu_fwd_kernel(const U4* __restrict__ g, const U4* __restrict__ u, int64_t n8,
                                                         U4* __restrict__ h) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (int64_t)gridDim.x * blockDim.x) {
    float a[8], b[8], o[8];
    unpack8f(g[i], a);
    unpack8f(u[i], b);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = bf16_round(silu_f(a[j])) * b[j];
    h[i] = pack8f(o);
  }
}
// dg = dh*u * silu'(g), du = dh*silu(g);  silu'(x) = s(x) * (1 + x*(1 - s(x)))
__global__ void __launch_bounds__(256) swiglu_bwd_kernel(const U4* __restrict__ dh, const U4* __restrict__ g,
                                                         const U4* __restrict__ u, int64_t n8, U4* __restrict__ dg,
                                                         U4* __restrict__ du) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (int64_t)gridDim.x * blockDim.x) {
    float a[8], b[8], d[8], og[8], ou[8];
    unpack8f(g[i], a);
    unpack8f(u[i], b);
    unpack8f(dh[i], d);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float sg = 1.f / (1.f + expf(-a[j]));
      const float act = bf16_round(a[j] * sg);
      ou[j] = d[j] * act;
      og[j] = bf16_round(d[j] * b[j]) * (sg * (1.f + a[j] * (1.f - sg)));
    }
    dg[i] = pack8f(og);
    du[i] = pack8f(ou);
  }
}

static unsigned grid_for(int64_t work, int threads) {
  int64_t b = (work + threads - 1) / threads;
  const int64_t cap = (int64_t)sm_count() * 16;
  if (b > cap) b = cap;
  return (unsigned)(b < 1 ? 1 : b);
}

}  // namespace ar

using namespace ar;

extern "C" int ar_rmsnorm_fwd(const void* x, const void* w, float eps, int64_t rows, int hidden, void* y, float* rstd,
                              void* stream) {
  AR_REQUIRE(x && w && y && rows > 0, AR_E_BADARG, "null pointer");
  AR_REQUIRE(hidden % 8 == 0 && hidden <= 8 * 256 * 4, AR_E_UNSUPPORTED, "hidden %d: need a multiple of 8, <= 8192", hidden);
  const int h8 = hidden / 8;
  cudaStream_t st = (cudaStream_t)stream;
  int threads = h8 >= 256 ? 256 : ((h8 + 31) / 32 * 32);
  const int vpt = (h8 + threads - 1) / threads;
  if (vpt == 1) rmsnorm_fwd_kernel<1><<<(unsigned)rows, threads, 0, st>>>((const U4*)x, (const U4*)w, eps, h8, (U4*)y, rstd);
  else if (vpt == 2) rmsnorm_fwd_kernel<2><<<(unsigned)rows, threads, 0, st>>>((const U4*)x, (const U4*)w, eps, h8, (U4*)y, rstd);
  else rmsnorm_fwd_kernel<4><<<(unsigned)rows, threads, 0, st>>>((const U4*)x, (const U4*)w, eps, h8, (U4*)y, rstd);
  AR_CHECK_LAUNCH();
  return AR_OK;
}

extern "C" int ar_rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd, int64_t rows, int hidden,
                              void* dx, int accumulate, void* stream) {
  AR_REQUIRE(dy && x && w && rstd && dx && rows > 0, AR_E_BADARG, "null pointer");
  AR_REQUIRE(hidden % 8 == 0 && hidden <= 8 * 256 * 4, AR_E_UNSUPPORTED, "hidden %d: need a multiple of 8, <= 8192", hidden);
  const int h8 = hidden / 8;
  cudaStream_t st = (cudaStream_t)stream;
  int threads = h8 >= 256 ? 256 : ((h8 + 31) / 32 * 32);
  const int vpt = (h8 + threads - 1) / threads;
  if (vpt == 1) rmsnorm_bwd_kernel<1><<<(unsigned)rows, threads, 0, st>>>((const U4*)dy, (const U4*)x, (const U4*)w, rstd, h8, (U4*)dx, accumulate);
  else if (vpt == 2) rmsnorm_bwd_kernel<2><<<(unsigned)rows, threads, 0, st>>>((const U4*)dy, (const U4*)x, (const U4*)w, rstd, h8, (U4*)dx, accumulate);
  else rmsnorm_bwd_kernel<4><<<(unsigned)rows, threads, 0, st>>>((const U4*)dy, (const U4*)x, (const U4*)w, rstd, h8, (U4*)dx, accumulate);
  AR_CHECK_LAUNCH();
  return AR_OK;
}

extern "C" int ar_rope(const void* x, const void* cos_t, const void* sin_t, int64_t b, int s, int h, int d, int table_batch,
                       int backward, void* out, void* stream) {
  AR_REQUIRE(x && cos_t && sin_t && out && b > 0 && s > 0 && h > 0, AR_E_BADARG, "null pointer / bad shape");
  AR_REQUIRE(d % 16 == 0, AR_E_UNSUPPORTED, "head_dim %d must be a multiple of 16", d);
  AR_REQUIRE(table_batch == 1 || table_batch == b, AR_E_BADARG, "cos/sin batch must be 1 or B");
  const int64_t total = b * s * h * (d / 16);
  const unsigned grid = (unsigned)((total + 255) / 256);
  cudaStream_t st = (cudaStream_t)stream;
  if (backward) rope_kernel<true><<<grid, 256, 0, st>>>((const uint16_t*)x, (const uint16_t*)cos_t, (const uint16_t*)sin_t, total, s, h, d, table_batch == 1, (uint16_t*)out);
  else rope_kernel<false><<<grid, 256, 0, st>>>((const uint16_t*)x, (const uint16_t*)cos_t, (const uint16_t*)sin_t, total, s, h, d, table_batch == 1, (uint16_t*)out);
  AR_CHECK_LAUNCH();
  return AR_OK;
}

extern "C" int ar_swiglu_fwd(const void* gate, const void* up, int64_t numel, void* h, void* stream) {
  AR_REQUIRE(gate && up && h && numel > 0 && numel % 8 == 0, AR_E_BADARG, "bad args");
  swiglu_fwd_kernel<<<grid_for(numel / 8, 256), 256, 0, (cudaStream_t)stream>>>((const U4*)gate, (const U4*)up, numel / 8, (U4*)h);
  AR_CHECK_LAUNCH();
  return AR_OK;
}

extern "C" int ar_swiglu_bwd(const void* dh, const void* gate, const void* up, int64_t numel, void* dgate, void* dup,
                             void* stream) {
  AR_REQUIRE(dh && gate && up && dgate && dup && numel > 0 && numel % 8 == 0, AR_E_BADARG, "bad args");
  swiglu_bwd_kernel<<<grid_for(numel / 8, 256), 256, 0, (cudaStream_t)stream>>>((const U4*)dh, (const U4*)gate, (const U4*)up,
                                                                                 numel / 8, (U4*)dgate, (U4*)dup);
  AR_CHECK_LAUNCH();
  return AR_OK;
}
