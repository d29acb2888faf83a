// MoE expert routing on the device (no host synchronisation, static launch shapes, CUDA-graph capturable) -- replaces the
// per-expert python loop of the reference (auto_round/modeling/fused_moe/moe_experts_interface.py:173-260:
// nonzero / index_select / index_copy_ per expert) with
//
//   ar_moe_route     top-k expert ids [T, k]  ->  a layout of the (token, slot) pairs SORTED BY EXPERT, every expert's segment
//                    padded to the 256-row GEMM tile, plus the tile tables the grouped wgmma GEMMs walk
//   ar_moe_gather    Xp[row] = X[token(row)] (optionally * the routing weight of that pair), pad rows = 0
//   ar_moe_combine   out[token] = sum over its k slots of (D[row(token, slot)] * w[token, slot])   (gather form: deterministic,
//                    no atomics -- the reference's `.view(ntok, k, -1).sum(dim=1)`)
//   ar_moe_rowdot    d w[token, slot] = <dOut[token], D[row]>                                       (gradient of the routing weights)
//
// Expert-parallel ownership: only pairs whose expert lies in [e_begin, e_end) get a row; the others have row = -1 and
// contribute nothing (their owner rank handles them), so the same kernels serve one GPU (all experts) and an EP rank.
#include "ar_common.cuh"

namespace ar {

constexpr int kRouteThreads = 1024;
constexpr int kMaxLocalExperts = 32;
constexpr int kTile = 256;

// One block.  pairs = T * k entries, thread i owns the contiguous chunk [i * per, (i + 1) * per).
//   counts[e]           pairs routed to local expert e (e relative to e_begin)
//   offsets[e]          first row of the expert's segment (multiple of 256); offsets[E] = rows in use
//   row_of_pair[p]      row of pair p in the sorted layout, -1 if its expert is not local
//   pair_of_row[r]      pair index of row r, -1 for padding rows (r < max_rows)
//   mtab                {m0, expert} per 256-row tile (GROUP_M table), *num_mt entries
//   ktab                {expert, k_off, k_len} per expert with tokens (GROUP_K table), *num_active entries
__global__ void __launch_bounds__(kRouteThreads) moe_route_kernel(const int64_t* __restrict__ expert_ids, int pairs, int e_begin,
                                                                  int e_local, int max_rows, int32_t* __restrict__ counts,
                                                                  int32_t* __restrict__ offsets, int32_t* __restrict__ row_of_pair,
                                                                  int32_t* __restrict__ pair_of_row, int32_t* __restrict__ mtab,
                                                                  int32_t* __restrict__ num_mt, int32_t* __restrict__ ktab,
                                                                  int32_t* __restrict__ num_active) {
  extern __shared__ int32_t sh[];                       // [e_local][kRouteThreads] per-thread counts -> exclusive prefix
  __shared__ int32_t s_off[kMaxLocalExperts + 1];
  __shared__ int32_t s_warp[kRouteThreads / 32];
  const int tid = threadIdx.x;
  const int per = (pairs + kRouteThreads - 1) / kRouteThreads;
  const int lo = tid * per, hi = min(pairs, lo + per);
  for (int e = 0; e < e_local; ++e) sh[e * kRouteThreads + tid] = 0;
  for (int r = tid; r < max_rows; r += kRouteThreads) pair_of_row[r] = -1;
  for (int p = lo; p < hi; ++p) {
    const int e = (int)expert_ids[p] - e_begin;
    if (e >= 0 && e < e_local) sh[e * kRouteThreads + tid] += 1;
  }
  __syncthreads();
  // exclusive scan over the threads, one expert at a time (warp shuffles + one pass over the 32 warp totals)
  for (int e = 0; e < e_local; ++e) {
    const int v = sh[e * kRouteThreads + tid];
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if ((tid & 31) >= o) x += y;
    }
    if ((tid & 31) == 31) s_warp[tid >> 5] = x;
    __syncthreads();
    if (tid < 32) {
      int w = s_warp[tid];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, w, o);
        if (tid >= o) w += y;
      }
      s_warp[tid] = w;                                  // inclusive over warps
    }
    __syncthreads();
    const int base = (tid >> 5) ? s_warp[(tid >> 5) - 1] : 0;
    sh[e * kRouteThreads + tid] = base + x - v;         // exclusive prefix of this thread
    if (tid == kRouteThreads - 1) counts[e] = base + x;
    __syncthreads();
  }
  if (tid == 0) {
    int off = 0, nmt = 0, nact = 0;
    for (int e = 0; e < e_local; ++e) {
      const int c = counts[e];
      const int padded = (c + kTile - 1) / kTile * kTile;
      s_off[e] = off;
      offsets[e] = off;
      for (int m0 = off; m0 < off + padded; m0 += kTile) { mtab[2 * nmt] = m0; mtab[2 * nmt + 1] = e; ++nmt; }
      if (c > 0) { ktab[3 * nact] = e; ktab[3 * nact + 1] = off; ktab[3 * nact + 2] = padded; ++nact; }
      off += padded;
    }
    s_off[e_local] = off;
    offsets[e_local] = off;
    *num_mt = nmt;
    *num_active = nact;
  }
  __syncthreads();
  int local[kMaxLocalExperts];
#pragma unroll
  for (int e = 0; e < kMaxLocalExperts; ++e) local[e] = 0;
  for (int p = lo; p < hi; ++p) {
    const int e = (int)expert_ids[p] - e_begin;
    int row = -1;
    if (e >= 0 && e < e_local) {
      int c = 0;
#pragma unroll
      for (int j = 0; j < kMaxLocalExperts; ++j)        // (register array: no dynamic indexing)
        if (j == e) { c = local[j]; local[j] = c + 1; }
      row = s_off[e] + sh[e * kRouteThreads + tid] + c;
      pair_of_row[row] = p;
    }
    row_of_pair[p] = row;
  }
}

// Xp[row, :] = scale(row) * X[pair_of_row[row] / topk, :]   (pad rows -> 0).  cols % 8 == 0.
__global__ void __launch_bounds__(256) moe_gather_kernel(const U4* __restrict__ x, const int32_t* __restrict__ pair_of_row,
                                                         const uint16_t* __restrict__ pair_w, int topk, int cols8,
                                                         U4* __restrict__ out) {
  const int row = blockIdx.x;
  const int p = pair_of_row[row];
  const float w = (p >= 0 && pair_w) ? bf16_bits_to_f32(pair_w[p]) : 1.f;
  const U4* src = x + (int64_t)(p >= 0 ? p / topk : 0) * cols8;
  U4* dst = out + (int64_t)row * cols8;
  for (int c = threadIdx.x; c < cols8; c += blockDim.x) {
    U4 v = U4{0u, 0u, 0u, 0u};
    if (p >= 0) {
      v = src[c];
      if (pair_w) {                                     // bf16 * bf16 -> bf16, like `grad * weights.unsqueeze(-1)`
        uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float a = bf16_bits_to_f32((uint16_t)(u[i] & 0xffffu)) * w, b = bf16_bits_to_f32((uint16_t)(u[i] >> 16)) * w;
          u[i] = (uint32_t)f32_to_bf16_bits(a) | ((uint32_t)f32_to_bf16_bits(b) << 16);
        }
        v = U4{u[0], u[1], u[2], u[3]};
      }
    }
    dst[c] = v;
  }
}

// out[token, :] = bf16( sum_slot float(bf16(D[row(token, slot), :] * w[token, slot])) (+ the same over D2) ), rows < 0 skipped
__global__ void __launch_bounds__(256) moe_combine_kernel(const U4* __restrict__ d, const U4* __restrict__ d2,
                                                          const int32_t* __restrict__ row_of_pair,
                                                          const uint16_t* __restrict__ pair_w, int topk, int cols8,
                                                          U4* __restrict__ out) {
  const int token = blockIdx.x;
  for (int c = threadIdx.x; c < cols8; c += blockDim.x) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int s = 0; s < topk; ++s) {
      const int p = token * topk + s;
      const int row = row_of_pair[p];
      if (row < 0) continue;
      const float w = pair_w ? bf16_bits_to_f32(pair_w[p]) : 1.f;
      for (int src = 0; src < 2; ++src) {
        const U4* base = src == 0 ? d : d2;
        if (base == nullptr) continue;
        const U4 v = base[(int64_t)row * cols8 + c];
        const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          float a = bf16_bits_to_f32((uint16_t)(u[i] & 0xffffu)), b = bf16_bits_to_f32((uint16_t)(u[i] >> 16));
          if (pair_w) {                                 // the product is a bf16 tensor in the reference
            a = bf16_bits_to_f32(f32_to_bf16_bits(a * w));
            b = bf16_bits_to_f32(f32_to_bf16_bits(b * w));
          }
          acc[2 * i] += a;
          acc[2 * i + 1] += b;
        }
      }
    }
    uint32_t o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) o[i] = (uint32_t)f32_to_bf16_bits(acc[2 * i]) | ((uint32_t)f32_to_bf16_bits(acc[2 * i + 1]) << 16);
    out[(int64_t)token * cols8 + c] = U4{o[0], o[1], o[2], o[3]};
  }
}

// dw[pair] = bf16( <g[token(pair), :], D[row(pair), :]> ), 0 for pairs without a row.  One warp per pair.
__global__ void __launch_bounds__(256) moe_rowdot_kernel(const U4* __restrict__ g, const U4* __restrict__ d,
                                                         const int32_t* __restrict__ row_of_pair, int pairs, int topk, int cols8,
                                                         uint16_t* __restrict__ dw) {
  const int p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (p >= pairs) return;
  const int lane = threadIdx.x & 31;
  const int row = row_of_pair[p];
  float acc = 0.f;
  if (row >= 0) {
    const U4* a = g + (int64_t)(p / topk) * cols8;
    const U4* b = d + (int64_t)row * cols8;
    for (int c = lane; c < cols8; c += 32) {
      const U4 x = a[c], y = b[c];
      const uint32_t ux[4] = {x.x, x.y, x.z, x.w}, uy[4] = {y.x, y.y, y.z, y.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        acc += bf16_bits_to_f32((uint16_t)(ux[i] & 0xffffu)) * bf16_bits_to_f32((uint16_t)(uy[i] & 0xffffu));
        acc += bf16_bits_to_f32((uint16_t)(ux[i] >> 16)) * bf16_bits_to_f32((uint16_t)(uy[i] >> 16));
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) dw[p] = f32_to_bf16_bits(acc);
}

}  // namespace ar

using namespace ar;

extern "C" int ar_moe_route(const int64_t* expert_ids, int pairs, int e_begin, int e_local, int max_rows, int32_t* counts,
                            int32_t* offsets, int32_t* row_of_pair, int32_t* pair_of_row, int32_t* mtab, int32_t* num_mt,
                            int32_t* ktab, int32_t* num_active, void* stream) {
  AR_REQUIRE(expert_ids && counts && offsets && row_of_pair && pair_of_row && mtab && num_mt && ktab && num_active, AR_E_BADARG,
             "ar_moe_route: null pointer");
  AR_REQUIRE(pairs > 0 && e_local > 0 && e_local <= kMaxLocalExperts, AR_E_UNSUPPORTED,
             "ar_moe_route: 1..%d local experts supported (got %d)", kMaxLocalExperts, e_local);
  AR_REQUIRE(max_rows >= pairs + e_local * (kTile - 1) && max_rows % kTile == 0, AR_E_BADARG,
             "ar_moe_route: max_rows must be a multiple of 256 and >= pairs + experts * 255");
  const size_t smem = (size_t)e_local * kRouteThreads * sizeof(int32_t);
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(moe_route_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         kMaxLocalExperts * kRouteThreads * (int)sizeof(int32_t));
    AR_REQUIRE(e == cudaSuccess, (int)e, "ar_moe_route: shared memory opt-in failed: %s", cudaGetErrorString(e));
    configured = true;
  }
  moe_route_kernel<<<1, kRouteThreads, smem, (cudaStream_t)stream>>>(expert_ids, pairs, e_begin, e_local, max_rows, counts, offsets,
                                                                   row_of_pair, pair_of_row, mtab, num_mt, ktab, num_active);
  AR_CHECK_LAUNCH();
  return AR_OK;
}

extern "C" int ar_moe_gather(const void* x, const int32_t* pair_of_row, const void* pair_w_bf16, int topk, int rows, int cols,
                             void* out, void* stream) {
  AR_REQUIRE(x && pair_of_row && out && rows > 0 && topk > 0, AR_E_BADARG, "ar_moe_gather: bad arguments");
  AR_REQUIRE(cols % 8 == 0, AR_E_UNSUPPORTED, "ar_moe_gather: cols must be a multiple of 8");
  moe_gather_kernel<<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>((const U4*)x, pair_of_row, (const uint16_t*)pair_w_bf16, topk,
                                                                     cols / 8, (U4*)out);
  AR_CHECK_LAUNCH();
  return AR_OK;
}

extern "C" int ar_moe_combine(const void* d, const void* d2, const int32_t* row_of_pair, const void* pair_w_bf16, int tokens,
                              int topk, int cols, void* out, void* stream) {
  AR_REQUIRE(d && row_of_pair && out && tokens > 0 && topk > 0, AR_E_BADARG, "ar_moe_combine: bad arguments");
  AR_REQUIRE(cols % 8 == 0, AR_E_UNSUPPORTED, "ar_moe_combine: cols must be a multiple of 8");
  moe_combine_kernel<<<(unsigned)tokens, 256, 0, (cudaStream_t)stream>>>((const U4*)d, (const U4*)d2, row_of_pair,
                                                                        (const uint16_t*)pair_w_bf16, topk, cols / 8, (U4*)out);
  AR_CHECK_LAUNCH();
  return AR_OK;
}

extern "C" int ar_moe_rowdot(const void* g, const void* d, const int32_t* row_of_pair, int pairs, int topk, int cols, void* dw_bf16,
                             void* stream) {
  AR_REQUIRE(g && d && row_of_pair && dw_bf16 && pairs > 0 && topk > 0, AR_E_BADARG, "ar_moe_rowdot: bad arguments");
  AR_REQUIRE(cols % 8 == 0, AR_E_UNSUPPORTED, "ar_moe_rowdot: cols must be a multiple of 8");
  const int per_block = 256 / 32;
  moe_rowdot_kernel<<<(unsigned)((pairs + per_block - 1) / per_block), 256, 0, (cudaStream_t)stream>>>(
      (const U4*)g, (const U4*)d, row_of_pair, pairs, topk, cols / 8, (uint16_t*)dw_bf16);
  AR_CHECK_LAUNCH();
  return AR_OK;
}
