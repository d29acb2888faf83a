// Low-bit weight packers (export hot path) -- HBM-bound byte/integer kernels, bit-exact to the reference.
//   INT:  auto_round_extension/torch/qlinear_torch_zp.py:93-150, qlinear_torch.py:110-168 (2/4/8 bit),
//         qlinear_torch.py:170-281 (3 bit).  codes = round(Wq/s + zp) along K, 32/bits per int32, LSB first,
//         stored transposed [K*bits/32, N].  Algorithmic bytes/weight: 2 (bf16 in) + bits/8 (out) + scales.
//   FP4:  auto_round/export/export_to_autoround/qlinear_fp.py:141-193, :235-265.
// Reads are coalesced along K (a warp reads 32 consecutive words' worth of one row), the word tile is
// transposed through shared memory, writes are coalesced along N.
#include "ar_qdq_math.cuh"

namespace ar {

// code of one element: torch.round(W / s + zp).to(int32)   (fp32 division after bf16/fp16 promotion)
__device__ __forceinline__ int32_t int_code(float w, float s, float zp) { return (int32_t)rintf(w / s + zp); }

// ---- 2/4/8-bit: tile = 32 rows (n) x 32 words (kw).  blockDim = (32, 8).  A thread builds one output word from PER = 32 / BITS
// consecutive K-elements of one row: ONE vector load (8 / 16 / 32 B), one scale / zero-point load when the word lies inside
// a group (every supported group size), and the quotient without div.rn (div_exact: bit-identical to w / s for a bf16 w
// and an fp16 s with |s| >= 1e-5, tests/test_div_exact.py; any other scale takes the IEEE division).
template <int BITS>
__global__ void __launch_bounds__(256) pack_pow2_kernel(const uint16_t* __restrict__ wq, const __half* __restrict__ scale,
                                                        const float* __restrict__ zp, float zp_const, int n, int k,
                                                        int group_size, int32_t* __restrict__ qweight) {
  constexpr int PER = 32 / BITS;
  __shared__ int32_t tile[32][33];
  const int kw_total = k / PER;
  const int ngroups = (k + group_size - 1) / group_size;
  const int kw = blockIdx.x * 32 + threadIdx.x;
  const bool one_group = (group_size % PER) == 0;
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int row = blockIdx.y * 32 + r;
    int32_t word = 0;
    if (row < n && kw < kw_total) {
      const int k0 = kw * PER;
      const uint16_t* src = wq + (int64_t)row * k + k0;
      uint16_t e[PER];
      if (BITS == 8) {
        const U2 v = *reinterpret_cast<const U2*>(src);
        e[0] = (uint16_t)(v.x & 0xffffu); e[1] = (uint16_t)(v.x >> 16); e[2] = (uint16_t)(v.y & 0xffffu); e[3] = (uint16_t)(v.y >> 16);
      } else {
#pragma unroll
        for (int q = 0; q < PER / 8; ++q) {
          const U4 v = reinterpret_cast<const U4*>(src)[q];
          const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int i = 0; i < 4; ++i) { e[q * 8 + 2 * i] = (uint16_t)(u[i] & 0xffffu); e[q * 8 + 2 * i + 1] = (uint16_t)(u[i] >> 16); }
        }
      }
      uint32_t acc = 0;
      if (one_group) {
        const int64_t gidx = (int64_t)row * ngroups + k0 / group_size;
        const float s = __half2float(scale[gidx]);
        const float z = zp ? zp[gidx] : zp_const;
        if (fabsf(s) >= 1e-5f) {
          const float rs = 1.f / s;
#pragma unroll
          for (int j = 0; j < PER; ++j)
            acc += ((uint32_t)(int32_t)rintf(div_exact(bf16_bits_to_f32(e[j]), s, rs) + z)) << (BITS * j);
        } else {
#pragma unroll
          for (int j = 0; j < PER; ++j) acc += ((uint32_t)int_code(bf16_bits_to_f32(e[j]), s, z)) << (BITS * j);
        }
      } else {
#pragma unroll
        for (int j = 0; j < PER; ++j) {
          const int gi = (k0 + j) / group_size;
          const float s = __half2float(scale[(int64_t)row * ngroups + gi]);
          const float z = zp ? zp[(int64_t)row * ngroups + gi] : zp_const;
          acc += ((uint32_t)int_code(bf16_bits_to_f32(e[j]), s, z)) << (BITS * j);   // sum of shifted lanes, wraps like int32
        }
      }
      word = (int32_t)acc;
    }
    tile[r][threadIdx.x] = word;
  }
  __syncthreads();
  for (int c = threadIdx.y; c < 32; c += 8) {
    const int okw = blockIdx.x * 32 + c;
    const int orow = blockIdx.y * 32 + threadIdx.x;
    if (okw < kw_total && orow < n) qweight[(int64_t)okw * n + orow] = tile[threadIdx.x][c];
  }
}

__device__ __forceinline__ void pack3_words(const uint32_t (&v)[32], uint32_t (&o)[3]) {
  o[0] = o[1] = o[2] = 0;
#pragma unroll
  for (int j = 0; j < 10; ++j) o[0] |= v[j] << (3 * j);
  o[0] |= v[10] << 30;
  o[1] |= (v[10] >> 2) & 1u;
#pragma unroll
  for (int j = 0; j < 10; ++j) o[1] |= v[11 + j] << (3 * j + 1);
  o[1] |= v[21] << 31;
  o[2] |= (v[21] >> 1) & 3u;
#pragma unroll
  for (int j = 0; j < 10; ++j) o[2] |= v[22 + j] << (3 * j + 2);
}

// ---- 3-bit: one thread packs 32 values of one row into 3 words.  blockDim = 128, thread -> (row fastest) for coalesced stores
__global__ void pack_3bit_kernel(const uint16_t* __restrict__ wq, const __half* __restrict__ scale,
                                 const float* __restrict__ zp, float zp_const, int n, int k, int group_size,
                                 int32_t* __restrict__ qweight) {
  const int ngroups = (k + group_size - 1) / group_size;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t total = (int64_t)n * (k / 32);
  if (idx >= total) return;
  const int row = (int)(idx % n);
  const int blk = (int)(idx / n);
  uint32_t v[32], o[3];
  for (int j = 0; j < 32; ++j) {
    const int kk = blk * 32 + j;
    const int gi = kk / group_size;
    const float s = __half2float(scale[(int64_t)row * ngroups + gi]);
    const float z = zp ? zp[(int64_t)row * ngroups + gi] : zp_const;
    v[j] = (uint32_t)int_code(bf16_bits_to_f32(wq[(int64_t)row * k + kk]), s, z);
  }
  pack3_words(v, o);
  for (int t = 0; t < 3; ++t) qweight[(int64_t)(blk * 3 + t) * n + row] = (int32_t)o[t];
}

// qzeros [G', N*bits/32]: packs zp (or the constant) along N; scales_t [G', N] = scale^T; g_idx [K]
template <int BITS>
__global__ void pack_zeros_kernel(const float* __restrict__ zp, int zp_const, int zp_minus_one, int n, int ngroups,
                                  int32_t* __restrict__ qzeros) {
  constexpr int PER = 32 / BITS;
  const int cols = n / 32 * BITS;                       // words per group row
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)ngroups * cols) return;
  const int gi = (int)(idx / cols), c = (int)(idx % cols);
  uint32_t acc = 0;
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    const int row = c * PER + j;
    int32_t z = zp ? (int32_t)zp[(int64_t)row * ngroups + gi] : zp_const;
    if (zp_minus_one) z -= 1;
    acc += ((uint32_t)z) << (BITS * j);
  }
  qzeros[idx] = (int32_t)acc;
}
__global__ void pack_zeros3_kernel(const float* __restrict__ zp, int zp_const, int zp_minus_one, int n, int ngroups,
                                   int32_t* __restrict__ qzeros) {
  const int blocks = n / 32;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)ngroups * blocks) return;
  const int gi = (int)(idx / blocks), b = (int)(idx % blocks);
  uint32_t v[32], o[3];
  for (int j = 0; j < 32; ++j) {
    int32_t z = zp ? (int32_t)zp[(int64_t)(b * 32 + j) * ngroups + gi] : zp_const;
    if (zp_minus_one) z -= 1;
    v[j] = (uint32_t)z;
  }
  pack3_words(v, o);
  for (int t = 0; t < 3; ++t) qzeros[(int64_t)gi * (blocks * 3) + b * 3 + t] = (int32_t)o[t];
}
__global__ void scales_t_gidx_kernel(const __half* __restrict__ scale, int n, int k, int ngroups, int group_size,
                                     __half* __restrict__ scales_t, int32_t* __restrict__ g_idx) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (scales_t && idx < (int64_t)n * ngroups) {
    const int gi = (int)(idx / n), row = (int)(idx % n);
    scales_t[idx] = scale[(int64_t)row * ngroups + gi];
  }
  if (g_idx && idx < k) g_idx[idx] = (int32_t)(idx / group_size);
}

// ---- unpack / dequant (round-trip tests; mirrors triton_utils/dequant.py:54-117)
__global__ void unpack_int_kernel(const int32_t* __restrict__ qweight, const int32_t* __restrict__ qzeros,
                                  const __half* __restrict__ scales_t, int n, int k, int bits, int group_size,
                                  int zp_minus_one, uint16_t* __restrict__ w_out, int32_t* __restrict__ codes) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)n * k) return;
  const int row = (int)(idx % n), kk = (int)(idx / n);
  const uint32_t mask = (1u << bits) - 1u;
  uint32_t code, z;
  if (bits == 3) {
    const int blk = kk / 32, j = kk % 32;
    const uint32_t w0 = (uint32_t)qweight[(int64_t)(blk * 3 + 0) * n + row];
    const uint32_t w1 = (uint32_t)qweight[(int64_t)(blk * 3 + 1) * n + row];
    const uint32_t w2 = (uint32_t)qweight[(int64_t)(blk * 3 + 2) * n + row];
    const uint64_t lo = (uint64_t)w0 | ((uint64_t)w1 << 32);
    if (j < 21) code = (uint32_t)((lo >> (3 * j)) & 7u);
    else if (j == 21) code = ((w1 >> 31) & 1u) | ((w2 & 3u) << 1);
    else code = (w2 >> (3 * (j - 22) + 2)) & 7u;
  } else {
    const int per = 32 / bits;
    code = (((uint32_t)qweight[(int64_t)(kk / per) * n + row]) >> (bits * (kk % per))) & mask;
  }
  const int gi = kk / group_size;
  if (bits == 3) {
    const int blk = row / 32, j = row % 32, cols = n / 32 * 3;
    const uint32_t w0 = (uint32_t)qzeros[(int64_t)gi * cols + blk * 3 + 0];
    const uint32_t w1 = (uint32_t)qzeros[(int64_t)gi * cols + blk * 3 + 1];
    const uint32_t w2 = (uint32_t)qzeros[(int64_t)gi * cols + blk * 3 + 2];
    const uint64_t lo = (uint64_t)w0 | ((uint64_t)w1 << 32);
    if (j < 21) z = (uint32_t)((lo >> (3 * j)) & 7u);
    else if (j == 21) z = ((w1 >> 31) & 1u) | ((w2 & 3u) << 1);
    else z = (w2 >> (3 * (j - 22) + 2)) & 7u;
  } else {
    const int per = 32 / bits;
    z = (((uint32_t)qzeros[(int64_t)gi * (n / per) + row / per]) >> (bits * (row % per))) & mask;
  }
  if (zp_minus_one) z = (z + 1u) & 0xffffffffu;
  if (codes) codes[(int64_t)row * k + kk] = (int32_t)code;
  if (w_out) {
    const float s = __half2float(scales_t[(int64_t)gi * n + row]);
    w_out[(int64_t)row * k + kk] = f32_to_bf16_bits(((float)(int32_t)code - (float)(int32_t)z) * s);
  }
}

// ---- AWQ "GEMM" layout, 4 bit (auto_round/export/export_to_awq/utils.py:197-273): the eight codes of output columns
// 8j .. 8j+7 of one k go into word j of row k, column 8j+i at bit 4 * order[i].  The words run along N while the weight is
// row-major in K, so a tile of 128 rows x 64 k is turned through shared memory: a thread loads 16 B (8 k of one row, a
// warp covers 128 B of each of 4 rows), codes them against one scale / zero-point (a group is a multiple of 8 k) and
// parks them as 8 bytes; then a thread gathers the 8 rows of one word column for those 8 k and writes 8 words, a warp
// covering 64 B of each of 2 output rows per store.  Bytes per weight: 2 read + 0.5 written.
__device__ __constant__ int kAwqShift[8] = {0, 16, 4, 20, 8, 24, 12, 28};            // 4 * [0, 4, 1, 5, 2, 6, 3, 7]
constexpr int AWQ_TN = 128, AWQ_TK = 64;

__global__ void __launch_bounds__(256) pack_awq_kernel(const uint16_t* __restrict__ wq, const __half* __restrict__ scale,
                                                       const float* __restrict__ zp, float zp_const, int n, int k,
                                                       int group_size, int32_t* __restrict__ qweight) {
  __shared__ U2 tile[AWQ_TN][AWQ_TK / 8 + 1];         // [row][k chunk] -> 8 int8 codes
  const int ngroups = k / group_size;
  const int row0 = blockIdx.y * AWQ_TN, k0 = blockIdx.x * AWQ_TK;
  for (int t = threadIdx.x; t < AWQ_TN * (AWQ_TK / 8); t += 256) {
    const int r = t / (AWQ_TK / 8), c = t % (AWQ_TK / 8);
    const int row = row0 + r, kk = k0 + c * 8;
    uint32_t lo = 0, hi = 0;
    if (row < n && kk < k) {
      const U4 v = *reinterpret_cast<const U4*>(wq + (int64_t)row * k + kk);
      const uint32_t u[4] = {v.x, v.y, v.z, v.w};
      const int64_t gidx = (int64_t)row * ngroups + kk / group_size;
      const float s = __half2float(scale[gidx]);
      const float z = zp ? zp[gidx] : zp_const;
      const bool exact = fabsf(s) >= 1e-5f;           // div_exact's domain; any other scale takes the IEEE division
      const float rs = 1.f / s;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float w = bf16_bits_to_f32((uint16_t)((e & 1) ? (u[e / 2] >> 16) : (u[e / 2] & 0xffffu)));
        const uint32_t code = (uint32_t)(exact ? (int32_t)rintf(div_exact(w, s, rs) + z) : int_code(w, s, z)) & 0xffu;
        if (e < 4) lo |= code << (8 * e); else hi |= code << (8 * (e - 4));
      }
    }
    tile[r][c] = U2{lo, hi};
  }
  __syncthreads();
  const int words = n / 8;
  for (int t = threadIdx.x; t < (AWQ_TN / 8) * (AWQ_TK / 8); t += 256) {
    const int j = t % (AWQ_TN / 8), c = t / (AWQ_TN / 8);
    const int oj = row0 / 8 + j, kk = k0 + c * 8;
    if (oj >= words || kk >= k) continue;
    uint32_t acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const U2 v = tile[j * 8 + i][c];
#pragma unroll
      for (int e = 0; e < 8; ++e) {                   // sum of shifted int32 lanes, wraps as the reference's does
        const int32_t code = (int32_t)(int8_t)(((e < 4) ? (v.x >> (8 * e)) : (v.y >> (8 * (e - 4)))) & 0xffu);
        acc[e] += ((uint32_t)code) << kAwqShift[i];
      }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) qweight[(int64_t)(kk + e) * words + oj] = (int32_t)acc[e];
  }
}

// qzeros [G, N/8]: the zero-points of columns 8j .. 8j+7 in the same nibble order (a constant fills every nibble);
// scales [G, N] = scale^T
__global__ void awq_zeros_scales_kernel(const __half* __restrict__ scale, const float* __restrict__ zp, int zp_const, int n,
                                        int ngroups, int32_t* __restrict__ qzeros, __half* __restrict__ scales_t) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)n * ngroups) return;
  const int gi = (int)(idx / n), row = (int)(idx % n);
  scales_t[idx] = scale[(int64_t)row * ngroups + gi];
  if (row % 8 == 0) {
    uint32_t acc = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (zp) acc += ((uint32_t)(int32_t)zp[(int64_t)(row + i) * ngroups + gi]) << kAwqShift[i];
      else acc |= ((uint32_t)zp_const) << (4 * i);
    }
    qzeros[(int64_t)gi * (n / 8) + row / 8] = (int32_t)acc;
  }
}

// inverse (dequantize_gemm, export_to_awq/utils.py:45-101): W'[N,K] = (code - zero) * scale
__global__ void unpack_awq_kernel(const int32_t* __restrict__ qweight, const int32_t* __restrict__ qzeros,
                                  const __half* __restrict__ scales_t, int n, int k, int group_size,
                                  uint16_t* __restrict__ w_out, int32_t* __restrict__ codes) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)n * k) return;
  const int row = (int)(idx % n), kk = (int)(idx / n), gi = kk / group_size;
  const int sh = kAwqShift[row % 8];
  const int32_t code = (int32_t)((((uint32_t)qweight[(int64_t)kk * (n / 8) + row / 8]) >> sh) & 15u);
  const int32_t z = (int32_t)((((uint32_t)qzeros[(int64_t)gi * (n / 8) + row / 8]) >> sh) & 15u);
  if (codes) codes[(int64_t)row * k + kk] = code;
  if (w_out) w_out[(int64_t)row * k + kk] = f32_to_bf16_bits((float)(code - z) * __half2float(scales_t[(int64_t)gi * n + row]));
}

// ---- FP4: nibble = first-argmin over {0,.5,1,1.5,2,3,4,6} | signbit<<3 ; low nibble = even k
template <bool IN_BF16_MATH>
__device__ __forceinline__ uint32_t e2m1_nibble(float x) {
  // a value that already IS an E2M1 number (every weight that comes out of the fake-quant functions) has distance 0 to exactly
  // one table entry: that index is the first argmin -- no search needed
  const uint32_t direct = e2m1_enc(x);
  if (e2m1_dec(direct) == x) return direct;
  const float lut[8] = {0.f, 0.5f, 1.f, 1.5f, 2.f, 3.f, 4.f, 6.f};
  const float a = fabsf(x);
  float best = 0.f;
  uint32_t bi = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float d = fabsf(a - lut[i]);
    if (IN_BF16_MATH) d = bf16_round(d);            // the MX path runs in the weight dtype (bf16)
    if (i == 0 || d < best) { best = d; bi = i; }
  }
  return bi | ((__float_as_uint(x) >> 31) << 3);
}

// one thread: 16 consecutive k of one row -> 8 bytes.  G = 16 (nv)
__global__ void pack_fp4_nv_kernel(const uint16_t* __restrict__ wq, const float* __restrict__ scale,
                                   const float* __restrict__ gscale, int n, int k, uint8_t* __restrict__ packed,
                                   uint8_t* __restrict__ scale_e4m3) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int gpr = k / 16;
  if (idx >= (int64_t)n * gpr) return;
  const int row = (int)(idx / gpr), gi = (int)(idx % gpr);
  const float gs = *gscale;
  const float sc = scale[idx];
  const float rg = (gs == 0.f) ? 0.f : 1.f / gs;
  const float prod = sc * rg;
  const float inv = (prod == 0.f) ? 0.f : 1.f / prod;
  uint16_t src[16];
  {
    const U4* v = reinterpret_cast<const U4*>(wq + (int64_t)row * k + gi * 16);        // 2 x 16 B (k % 16 == 0)
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const U4 t = v[q];
      const uint32_t u[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) { src[q * 8 + 2 * i] = (uint16_t)(u[i] & 0xffffu); src[q * 8 + 2 * i + 1] = (uint16_t)(u[i] >> 16); }
    }
  }
  uint32_t lo = 0, hi = 0;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    float x = bf16_bits_to_f32(src[j]) * inv;
    x = nv_cast_to_fp4(clampf(x, -6.f, 6.f));
    const uint32_t nib = e2m1_nibble<false>(x);
    if (j < 8) lo |= nib << (4 * j); else hi |= nib << (4 * (j - 8));
  }
  *reinterpret_cast<U2*>(packed + (int64_t)row * (k / 2) + gi * 8) = U2{lo, hi};
  if (scale_e4m3) scale_e4m3[idx] = f32_to_e4m3_bits(sc);
}

// G = 32 (mx): x = bf16(W / 2^e) in bf16 arithmetic
__global__ void pack_fp4_mx_kernel(const uint16_t* __restrict__ wq, const uint16_t* __restrict__ exp_bf16, int n, int k,
                                   uint8_t* __restrict__ packed, uint8_t* __restrict__ scale_e8m0) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int gpr = k / 32;
  if (idx >= (int64_t)n * gpr) return;
  const int row = (int)(idx / gpr), gi = (int)(idx % gpr);
  const float e = bf16_bits_to_f32(exp_bf16[idx]);
  const float p = bf16_round(exp2f(e));                        // 2 ** scales, bf16 tensor
  // p is a power of two for every exponent the quantiser stores: W / p == W * (1 / p) exactly; anything else divides
  const bool pow2 = (__float_as_uint(p) & 0x007fffffu) == 0u && p != 0.f;
  const float rp = pow2 ? 1.f / p : 0.f;
  const U4* v = reinterpret_cast<const U4*>(wq + (int64_t)row * k + gi * 32);          // 4 x 16 B (k % 32 == 0)
  uint32_t o[4] = {0, 0, 0, 0};
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const U4 t = v[q];
    const uint32_t u[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float w = bf16_bits_to_f32((uint16_t)((i & 1) ? (u[i / 2] >> 16) : (u[i / 2] & 0xffffu)));
      const float x = bf16_round(pow2 ? w * rp : w / p);
      o[q] |= e2m1_nibble<true>(x) << (4 * i);
    }
  }
  *reinterpret_cast<U4*>(packed + (int64_t)row * (k / 2) + gi * 16) = U4{o[0], o[1], o[2], o[3]};
  if (scale_e8m0) scale_e8m0[idx] = (uint8_t)clampf(bf16_round(e + 127.f), 0.f, 255.f);
}

__global__ void unpack_fp4_kernel(const uint8_t* __restrict__ packed, int64_t nbytes, uint16_t* __restrict__ out) {
  const float lut[8] = {0.f, 0.5f, 1.f, 1.5f, 2.f, 3.f, 4.f, 6.f};
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nbytes) return;
  const uint8_t b = packed[idx];
  const float a = lut[b & 7u] * ((b & 8u) ? -1.f : 1.f);
  const float c = lut[(b >> 4) & 7u] * ((b & 0x80u) ? -1.f : 1.f);
  out[2 * idx] = f32_to_bf16_bits(a);
  out[2 * idx + 1] = f32_to_bf16_bits(c);
}

}  // namespace ar

using namespace ar;

extern "C" int ar_pack_int(const void* wq, const void* scale, const float* zp, int zp_const, int n, int k, int bits,
                           int group_size, int zp_minus_one, int32_t* qweight, int32_t* qzeros, void* scales_t,
                           int32_t* g_idx, void* stream) {
  AR_REQUIRE(wq && scale && qweight, AR_E_BADARG, "null pointer");
  AR_REQUIRE(bits == 2 || bits == 3 || bits == 4 || bits == 8, AR_E_UNSUPPORTED, "bits %d", bits);
  AR_REQUIRE(k % 32 == 0 && n % 32 == 0, AR_E_UNSUPPORTED, "pack needs n,k multiples of 32 (n=%d k=%d)", n, k);
  if (group_size <= 0) group_size = k;
  cudaStream_t st = (cudaStream_t)stream;
  const int ngroups = (k + group_size - 1) / group_size;
  const float zc = (float)zp_const;
  if (bits == 3) {
    const int64_t total = (int64_t)n * (k / 32);
    pack_3bit_kernel<<<(unsigned)((total + 127) / 128), 128, 0, st>>>((const uint16_t*)wq, (const __half*)scale, zp, zc,
                                                                     n, k, group_size, qweight);
  } else {
    const int per = 32 / bits;
    const dim3 grid((k / per + 31) / 32, (n + 31) / 32), block(32, 8);
    if (bits == 2) pack_pow2_kernel<2><<<grid, block, 0, st>>>((const uint16_t*)wq, (const __half*)scale, zp, zc, n, k, group_size, qweight);
    else if (bits == 4) pack_pow2_kernel<4><<<grid, block, 0, st>>>((const uint16_t*)wq, (const __half*)scale, zp, zc, n, k, group_size, qweight);
    else pack_pow2_kernel<8><<<grid, block, 0, st>>>((const uint16_t*)wq, (const __half*)scale, zp, zc, n, k, group_size, qweight);
  }
  AR_CHECK_LAUNCH();
  if (qzeros) {
    if (bits == 3) {
      const int64_t total = (int64_t)ngroups * (n / 32);
      pack_zeros3_kernel<<<(unsigned)((total + 127) / 128), 128, 0, st>>>(zp, zp_const, zp_minus_one, n, ngroups, qzeros);
    } else {
      const int64_t total = (int64_t)ngroups * (n / 32 * bits);
      const unsigned g = (unsigned)((total + 255) / 256);
      if (bits == 2) pack_zeros_kernel<2><<<g, 256, 0, st>>>(zp, zp_const, zp_minus_one, n, ngroups, qzeros);
      else if (bits == 4) pack_zeros_kernel<4><<<g, 256, 0, st>>>(zp, zp_const, zp_minus_one, n, ngroups, qzeros);
      else pack_zeros_kernel<8><<<g, 256, 0, st>>>(zp, zp_const, zp_minus_one, n, ngroups, qzeros);
    }
    AR_CHECK_LAUNCH();
  }
  if (scales_t || g_idx) {
    int64_t total = (int64_t)n * ngroups;
    if (k > total) total = k;
    scales_t_gidx_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>((const __half*)scale, n, k, ngroups, group_size,
                                                                         (__half*)scales_t, g_idx);
    AR_CHECK_LAUNCH();
  }
  return AR_OK;
}

extern "C" int ar_unpack_int(const int32_t* qweight, const int32_t* qzeros, const void* scales_t, int n, int k, int bits,
                             int group_size, int zp_minus_one, void* w_out, int32_t* codes, void* stream) {
  AR_REQUIRE(qweight && qzeros && scales_t, AR_E_BADARG, "null pointer");
  AR_REQUIRE(bits == 2 || bits == 3 || bits == 4 || bits == 8, AR_E_UNSUPPORTED, "bits %d", bits);
  if (group_size <= 0) group_size = k;
  const int64_t total = (int64_t)n * k;
  unpack_int_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      qweight, qzeros, (const __half*)scales_t, n, k, bits, group_size, zp_minus_one, (uint16_t*)w_out, codes);
  AR_CHECK_LAUNCH();
  return AR_OK;
}

extern "C" int ar_pack_awq(const void* wq, const void* scale, const float* zp, int zp_const, int n, int k, int group_size,
                           int32_t* qweight, int32_t* qzeros, void* scales_t, void* stream) {
  AR_REQUIRE(wq && scale && qweight && qzeros && scales_t, AR_E_BADARG, "null pointer");
  AR_REQUIRE(n > 0 && k > 0, AR_E_BADARG, "empty weight (n=%d k=%d)", n, k);
  if (group_size == -1) group_size = k;
  AR_REQUIRE(group_size > 0 && k % group_size == 0, AR_E_BADARG, "in_features (%d) shape mismatch", k);
  AR_REQUIRE(n % 8 == 0, AR_E_BADARG, "out_features (%d) shape mismatch", n);
  AR_REQUIRE(group_size % 8 == 0, AR_E_UNSUPPORTED, "awq pack needs group_size %% 8 == 0 (group_size=%d)", group_size);
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid((k + AWQ_TK - 1) / AWQ_TK, (n + AWQ_TN - 1) / AWQ_TN);
  AR_REQUIRE(grid.y <= 65535u, AR_E_UNSUPPORTED, "awq pack: n=%d too large", n);
  pack_awq_kernel<<<grid, 256, 0, st>>>((const uint16_t*)wq, (const __half*)scale, zp, (float)zp_const, n, k, group_size, qweight);
  AR_CHECK_LAUNCH();
  const int ngroups = k / group_size;
  const int64_t total = (int64_t)n * ngroups;
  awq_zeros_scales_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>((const __half*)scale, zp, zp_const, n, ngroups,
                                                                          qzeros, (__half*)scales_t);
  AR_CHECK_LAUNCH();
  return AR_OK;
}

extern "C" int ar_unpack_awq(const int32_t* qweight, const int32_t* qzeros, const void* scales_t, int n, int k,
                             int group_size, void* w_out, int32_t* codes, void* stream) {
  AR_REQUIRE(qweight && qzeros && scales_t && (w_out || codes), AR_E_BADARG, "null pointer");
  if (group_size == -1) group_size = k;
  AR_REQUIRE(n > 0 && k > 0 && group_size > 0 && k % group_size == 0 && n % 8 == 0, AR_E_BADARG,
             "awq unpack: n=%d k=%d group_size=%d", n, k, group_size);
  const int64_t total = (int64_t)n * k;
  unpack_awq_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      qweight, qzeros, (const __half*)scales_t, n, k, group_size, (uint16_t*)w_out, codes);
  AR_CHECK_LAUNCH();
  return AR_OK;
}

extern "C" int ar_pack_fp4_nv(const void* wq, const float* scale, const float* gscale, int n, int k, uint8_t* packed,
                              uint8_t* scale_e4m3, void* stream) {
  AR_REQUIRE(wq && scale && gscale && packed, AR_E_BADARG, "null pointer");
  AR_REQUIRE(k % 16 == 0, AR_E_UNSUPPORTED, "nv_fp4 pack needs k %% 16 == 0");
  const int64_t total = (int64_t)n * (k / 16);
  pack_fp4_nv_kernel<<<(unsigned)((total + 127) / 128), 128, 0, (cudaStream_t)stream>>>((const uint16_t*)wq, scale, gscale,
                                                                                         n, k, packed, scale_e4m3);
  AR_CHECK_LAUNCH();
  return AR_OK;
}
extern "C" int ar_pack_fp4_mx(const void* wq, const void* exp_bf16, int n, int k, uint8_t* packed, uint8_t* scale_e8m0,
                              void* stream) {
  AR_REQUIRE(wq && exp_bf16 && packed, AR_E_BADARG, "null pointer");
  AR_REQUIRE(k % 32 == 0, AR_E_UNSUPPORTED, "mx_fp4 pack needs k %% 32 == 0");
  const int64_t total = (int64_t)n * (k / 32);
  pack_fp4_mx_kernel<<<(unsigned)((total + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
      (const uint16_t*)wq, (const uint16_t*)exp_bf16, n, k, packed, scale_e8m0);
  AR_CHECK_LAUNCH();
  return AR_OK;
}
extern "C" int ar_unpack_fp4(const uint8_t* packed, int n, int k, void* values, void* stream) {
  AR_REQUIRE(packed && values && k % 2 == 0, AR_E_BADARG, "bad args");
  const int64_t nbytes = (int64_t)n * (k / 2);
  unpack_fp4_kernel<<<(unsigned)((nbytes + 255) / 256), 256, 0, (cudaStream_t)stream>>>(packed, nbytes, (uint16_t*)values);
  AR_CHECK_LAUNCH();
  return AR_OK;
}
