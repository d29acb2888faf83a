// Per-iteration glue kernels of the sign-SGD loop: masked MSE + gradient, best-iteration bookkeeping, sample gather,
// device-side schedule (the sign-SGD step itself is part of the per-layer update, ar_fq_update in ar_qdq.cu).  All
// HBM-bound, vectorised 16 B accesses, grid = multiple of the SM count, no host synchronisation (state lives in device
// memory).
#include "ar_common.cuh"

namespace ar {

__device__ __forceinline__ void unpack8(const U4& r, float (&o)[8]) {
  const uint32_t u[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    o[2 * i] = bf16_bits_to_f32((uint16_t)(u[i] & 0xffffu));
    o[2 * i + 1] = bf16_bits_to_f32((uint16_t)(u[i] >> 16));
  }
}

// pred/ref bf16 [rows, cols], cols % 8 == 0.  One thread = 8 elements.
//   loss_sum += sum(diff^2) (double, unnormalised);  dpred = bf16((norm*diff)*upstream) * m
__global__ void __launch_bounds__(256) mse_fwd_bwd_kernel(const uint16_t* __restrict__ pred, const uint16_t* __restrict__ ref,
                                                          const uint8_t* __restrict__ mask, int64_t rows, int cols8,
                                                          float norm, float upstream, double* __restrict__ loss_sum,
                                                          uint16_t* __restrict__ dpred) {
  const int64_t total = rows * (int64_t)cols8;
  float local = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / cols8;
    const bool on = (mask == nullptr) || (mask[row] != 0);
    float p[8], r[8];
    uint32_t out[4] = {0, 0, 0, 0};
    if (on) {
      unpack8(reinterpret_cast<const U4*>(pred)[i], p);
      unpack8(reinterpret_cast<const U4*>(ref)[i], r);
      float g[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = p[j] - r[j];
        local += d * d;
        g[j] = (norm * d) * upstream;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) out[j] = (uint32_t)f32_to_bf16_bits(g[2 * j]) | ((uint32_t)f32_to_bf16_bits(g[2 * j + 1]) << 16);
    }
    if (dpred) reinterpret_cast<U4*>(dpred)[i] = U4{out[0], out[1], out[2], out[3]};
  }
  // block reduction, one double atomic per block
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
  __shared__ float warp_sums[8];
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = local;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < 8; ++w) s += (double)warp_sums[w];
    atomicAdd(loss_sum, s);
  }
}

// state: [0]=best_loss [1]=last_loss [2]=best_iter [3]=spare
__global__ void best_update_kernel(double* loss_sum, double inv_numel, double inv_num_elm, int iter,
                                   const double* inv_num_elm_ptr, const int32_t* it_ptr, double* state, int32_t* flag,
                                   float* loss_hist) {
  if (it_ptr) iter = *it_ptr;                               // device-side schedule (CUDA-graph replay)
  if (inv_num_elm_ptr) inv_num_elm = *inv_num_elm_ptr;
  const float mean = (float)(*loss_sum * inv_numel);       // MSELoss('mean') result is an fp32 scalar
  const double total = (double)mean * inv_num_elm;          // loss.item() / num_elm
  if (iter == 0) state[0] = 3.4028234663852886e38;          // torch.finfo(torch.float).max
  const bool better = total < state[0];
  if (better) { state[0] = total; state[2] = (double)iter; }
  state[1] = total;
  *flag = better ? 1 : 0;
  if (loss_hist) loss_hist[iter] = (float)total;
  *loss_sum = 0.0;
}

__global__ void __launch_bounds__(256) gather_rows_kernel(const U4* __restrict__ src, const int32_t* __restrict__ idx,
                                                          int64_t row_vec, U4* __restrict__ dst) {
  const int64_t s = (int64_t)idx[blockIdx.y] * row_vec, d = (int64_t)blockIdx.y * row_vec;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < row_vec; i += (int64_t)gridDim.x * blockDim.x)
    dst[d + i] = src[s + i];
}

// schedule row of the current iteration -> static buffers read by the rest of the (graph-captured) iteration
__global__ void sched_load_kernel(const int32_t* __restrict__ idx_table, const double* __restrict__ inv_num_elm_table,
                                  const int32_t* __restrict__ it_ptr, int count, int32_t* __restrict__ cur32,
                                  int64_t* __restrict__ cur64, double* __restrict__ cur_inv) {
  const int it = *it_ptr;
  for (int i = threadIdx.x; i < count; i += blockDim.x) {
    const int32_t v = idx_table[(int64_t)it * count + i];
    if (cur32) cur32[i] = v;
    if (cur64) cur64[i] = (int64_t)v;
  }
  if (threadIdx.x == 0 && cur_inv && inv_num_elm_table) *cur_inv = inv_num_elm_table[it];
}
__global__ void iter_advance_kernel(int32_t* it_ptr) { *it_ptr += 1; }

}  // namespace ar

using namespace ar;

extern "C" int ar_mse_fwd_bwd(const void* pred, const void* ref, const uint8_t* row_mask, int64_t rows, int64_t cols,
                              float inv_numel, float upstream, double* loss_sum, void* dpred, void* stream) {
  AR_REQUIRE(pred && ref && loss_sum, AR_E_BADARG, "null pointer");
  AR_REQUIRE(cols % 8 == 0, AR_E_UNSUPPORTED, "cols must be a multiple of 8 (got %lld)", (long long)cols);
  const int64_t total = rows * (cols / 8);
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = (int64_t)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  mse_fwd_bwd_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((const uint16_t*)pred, (const uint16_t*)ref, row_mask,
                                                                         rows, (int)(cols / 8), 2.f * inv_numel, upstream,
                                                                         loss_sum, (uint16_t*)dpred);
  AR_CHECK_LAUNCH();
  return AR_OK;
}

extern "C" int ar_best_update(double* loss_sum, double inv_numel, double inv_num_elm, int iter,
                              const double* inv_num_elm_ptr, const int32_t* it_ptr, double* state, int32_t* flag,
                              float* loss_hist, void* stream) {
  AR_REQUIRE(loss_sum && state && flag && iter >= 0, AR_E_BADARG, "bad args");
  best_update_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(loss_sum, inv_numel, inv_num_elm, iter, inv_num_elm_ptr, it_ptr, state,
                                                        flag, loss_hist);
  AR_CHECK_LAUNCH();
  return AR_OK;
}

extern "C" int ar_gather_rows(const void* src, const int32_t* idx, int count, int64_t row_elems, void* dst, void* stream) {
  AR_REQUIRE(src && idx && dst && count > 0, AR_E_BADARG, "bad args");
  AR_REQUIRE(row_elems % 8 == 0, AR_E_UNSUPPORTED, "row_elems must be a multiple of 8");
  const int64_t row_vec = row_elems / 8;
  int64_t bx = (row_vec + 255) / 256;
  const int64_t cap = ((int64_t)sm_count() * 8 + count - 1) / count;
  if (bx > cap) bx = cap;
  if (bx < 1) bx = 1;
  gather_rows_kernel<<<dim3((unsigned)bx, (unsigned)count), 256, 0, (cudaStream_t)stream>>>((const U4*)src, idx, row_vec, (U4*)dst);
  AR_CHECK_LAUNCH();
  return AR_OK;
}

extern "C" int ar_sched_load(const int32_t* idx_table, const double* inv_num_elm_table, const int32_t* it_ptr, int count,
                             int32_t* cur_idx32, int64_t* cur_idx64, double* cur_inv_num_elm, void* stream) {
  AR_REQUIRE(idx_table && it_ptr && count > 0, AR_E_BADARG, "bad args");
  sched_load_kernel<<<1, 64, 0, (cudaStream_t)stream>>>(idx_table, inv_num_elm_table, it_ptr, count, cur_idx32, cur_idx64,
                                                        cur_inv_num_elm);
  AR_CHECK_LAUNCH();
  return AR_OK;
}

extern "C" int ar_iter_advance(int32_t* it_ptr, void* stream) {
  AR_REQUIRE(it_ptr, AR_E_BADARG, "bad args");
  iter_advance_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(it_ptr);
  AR_CHECK_LAUNCH();
  return AR_OK;
}
