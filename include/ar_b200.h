/*
 * ar_b200.h -- C ABI of the H100-native AutoRound calibration kernels (libar_b200.so).
 *
 * Drop-in boundary for ONE hot path of intel/auto-round: the per-block SignRound tuning loop, its
 * weight quant-dequant numerics and the final low-bit pack.  The reference has no native code on this
 * path (it is eager PyTorch); each entry point below names the reference Python it replaces
 * (paths relative to the reference root, v0.15.0).  INTEGRATION.md shows the ctypes binding a
 * maintainer would add on the reference side.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host; the caller owns all memory;
 *   - no entry point allocates, synchronises with the host, or keeps global state (a small cache of
 *     cuTensorMap descriptors keyed by pointer/shape is the one exception, see ar_gemm_*);
 *   - `stream` is a cudaStream_t passed as void*; work is enqueued on it and the call returns;
 *   - return value: 0 = ok, <0 = argument error (AR_E_*), >0 = a cudaError_t from the launch;
 *     ar_last_error() gives a thread-local message.  No exceptions cross the ABI;
 *   - W is the nn.Linear weight [N, K] (out x in) row-major bf16; quantisation groups run along K
 *     inside a row (group index = n * ceil(K/g) + k / g), exactly as
 *     auto_round/data_type/utils.py:29-71 (reshape_pad_tensor_by_group_size) lays them out;
 *   - V (the learnable rounding offset) is fp32 [N, Kpad], Kpad = ceil(K/g)*g; min_scale/max_scale
 *     are fp32 [G], G = N * Kpad / g  (auto_round/wrapper.py:184-190).
 */
#ifndef AR_B200_H_
#define AR_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AR_B200_VERSION 100

/* data types of the fake-quant functions (auto_round/data_type/register.py names) */
enum {
  AR_DT_INT_SYM = 0,  /* "int_sym"  auto_round/data_type/int.py:165-238  */
  AR_DT_INT_ASYM = 1, /* "int_asym" auto_round/data_type/int.py:241-298  */
  AR_DT_MX_FP4 = 2,   /* "mx_fp4"   auto_round/data_type/mxfp.py:233-291 */
  AR_DT_NV_FP4 = 3    /* "nv_fp4"   auto_round/data_type/nvfp.py:83-98   */
};

enum {
  AR_OK = 0,
  AR_E_BADARG = -1,     /* null pointer / shape not supported */
  AR_E_UNSUPPORTED = -2,/* combination not built (e.g. group size) */
  AR_E_ARCH = -3,       /* wgmma path requested on a device that is not sm_90 */
  AR_E_DRIVER = -4      /* cuTensorMapEncodeTiled unavailable / failed */
};

int ar_version(void);
const char* ar_last_error(void);

/* Quantisation spec of one linear layer.  Plain-old-data, passed by pointer (host memory). */
typedef struct ar_qspec {
  int32_t dtype;          /* AR_DT_* */
  int32_t bits;           /* 2,3,4,8 for int; 4 for fp4 */
  int32_t group_size;     /* 16/32/64/128/256; K is zero-padded to a multiple (reference semantics) */
  int32_t n;              /* rows of W (out features) */
  int32_t k;              /* cols of W (in features) */
  float q_scale_thresh;   /* 1e-5 (fp16 scale) / 1e-8 (fp32 scale): auto_round/wrapper.py:115-118 */
  float scale_bound_hi;   /* upper clamp of min/max_scale: 1.0 (wrapper.py:76) or 2.0 (alg_ext) */
  const float* init_scale; /* NULL, or DEVICE fp32 [N*ceil(K/g)]: enable_alg_ext's searched per-group initial scale
                              (sign_roundv2/quantizer.py:101-125).  int_sym: scale = fp16(init_scale * max_scale), min_scale
                              unused (int.py:201-216); mx/nv: the group amax is multiplied by init_scale * max_scale
                              (mxfp.py:262-266, nvfp.py:93-97).  Honoured by ar_qdq_fwd/_bwd and ar_fq_update. */
} ar_qspec;

/* Per-group min/max of W clamped at 0 (bf16 out, [G]) -- auto_round/wrapper.py:154-167. */
int ar_group_minmax(const ar_qspec* q, const void* w_bf16, void* wmin_bf16, void* wmax_bf16, void* stream);

/* amax(|W|) over the whole tensor into *amax_f32 (atomicMax on the bit pattern; caller zeroes it first),
 * and NVFP4 global scale 448*6/amax -- auto_round/data_type/nvfp.py:56-64 (calculate_gparam). */
int ar_absmax(const void* w_bf16, int64_t numel, float* amax_f32, void* stream);
int ar_nv_global_scale(const float* amax_f32, float* gscale_f32, void* stream);

/*
 * Fake-quant forward: Wq = qdq(W; V, min_scale, max_scale).  Replaces WrapperLinear._qdq_weight
 * (auto_round/wrapper.py:244-293) + the registered data_type function, for all AR_DT_*.
 *   v, min_scale, max_scale may be NULL (=> 0, 1, 1: plain RTN, auto_round/data_type/int.py:125-162).
 *   wmin/wmax: bf16 [G] from ar_group_minmax (int types; ignored for fp4, which use amax|W| per group).
 *   gscale: device fp32 scalar (nv_fp4 only).
 *   wq_bf16 [N,K] may be NULL if only scales are wanted.
 *   scale_out: fp16 [G] (int) | bf16 [G] shared exponent (mx) | fp32 [G] e4m3-valued (nv); may be NULL.
 *   zp_out:    fp32 [G] (int_asym only); may be NULL.
 */
int ar_qdq_fwd(const ar_qspec* q, const void* w_bf16, const float* v, const float* min_scale,
               const float* max_scale, const void* wmin_bf16, const void* wmax_bf16, const float* gscale,
               void* wq_bf16, void* scale_out, float* zp_out, void* stream);

/*
 * Fake-quant backward (what autograd does through the reference's qdq graph, auto_round/wrapper.py:273-290
 * + STE helpers auto_round/data_type/utils.py:314-365): given Gq = dL/dWq fp32 [N,K] produce
 *   dv [N,Kpad] fp32, dmin [G] fp32 (int types; NULL otherwise), dmax [G] fp32.
 *   accumulate != 0 adds into the outputs (gradient accumulation), else overwrites.
 */
int ar_qdq_bwd(const ar_qspec* q, const void* w_bf16, const float* v, const float* min_scale,
               const float* max_scale, const void* wmin_bf16, const void* wmax_bf16, const float* gscale,
               const float* gq_f32, float* dv, float* dmin, float* dmax, int accumulate, void* stream);

/*
 * bf16 GEMM on wgmma/TMA:  D[M,N] = A · Bᵀ  with A logical [M,K], B logical [N,K].
 *   a_mn_major / b_mn_major = 0: operand stored [rows, K] row-major (K contiguous);
 *                            = 1: operand stored [K, rows] row-major (rows contiguous).
 *   lda/ldb/ldd: leading dimension (elements) of the stored matrix.  D is bf16 row-major [M,N].
 *   bias_bf16: optional [N] added in the epilogue.  Replaces F.linear (auto_round/wrapper.py:470-481)
 *   and its two autograd GEMMs.
 */
int ar_gemm_bf16(const void* a, const void* b, void* d, int m, int n, int k, int a_mn_major, int b_mn_major,
                 int64_t lda, int64_t ldb, int64_t ldd, const void* bias_bf16, void* stream);

/*
 * Grouped (ragged per-expert) bf16 GEMM on wgmma for un-fused MoE experts -- replaces the per-expert python loop of
 * auto_round/modeling/fused_moe/moe_experts_interface.py:173-260 (`_run_experts_with_routes`).  Tiles are resolved through the
 * device-side tables written by ar_moe_route in the same stream, so the launch is static (CUDA-graph capturable):
 *   mode 1 (GROUP_M)  D[rows, n] = A[rows, k] · B_eᵀ,  e = expert of each 256-row tile (table: {m0, expert} x *num).
 *                     b_mn_major = 0: B stacked [num_groups * group_rows, k], group_rows = n            (forward)
 *                     b_mn_major = 1: B stored  [num_groups * group_rows, n], group_rows = k: the reduction runs over the
 *                                     expert's rows                                                      (grad-in)
 *   mode 2 (GROUP_K)  for every ACTIVE expert (table: {expert, k_off, k_len} x *num):
 *                     D_e[group_rows, n] = A[k_off : k_off + k_len, :group_rows]ᵀ · B[k_off : k_off + k_len, :n]
 *                     A stored [rows, a_features], B stored [rows, n], D stacked [num_groups * group_rows, n] with
 *                     group_rows = a_features rounded up to 256 (the row pitch of an expert's output slab)   (grad-w)
 * rows = padded row capacity of the sorted token layout (multiple of 256); max_entries bounds *num (grid sizing only);
 * a_features is ignored in mode 1.
 */
int ar_gemm_bf16_grouped(const void* a, const void* b, void* d, int mode, int rows, int n, int k, int a_mn_major, int b_mn_major,
                         int64_t lda, int64_t ldb, int64_t ldd, int group_rows, int num_groups, const int32_t* table,
                         const int32_t* num, int max_entries, int a_features, void* stream);

/*
 * MoE routing on the device (csrc/ar_moe.cu): expert_ids int64 [pairs = tokens * topk] -> the (token, slot) pairs sorted by
 * expert with every expert's segment padded to 256 rows.  Only experts [e_begin, e_begin + e_local) get rows (expert-parallel
 * ownership; e_local <= 32).  Outputs (int32, device): counts[e_local], offsets[e_local + 1], row_of_pair[pairs] (-1 = not
 * local), pair_of_row[max_rows] (-1 = padding), the GROUP_M table mtab[2 * max_rows / 256] + *num_mt and the GROUP_K table
 * ktab[3 * e_local] + *num_active.  max_rows: multiple of 256, >= pairs + 255 * e_local.
 *   ar_moe_gather   out[row, :] = x[pair_of_row[row] / topk, :] (* pair_w[pair], bf16 product) ; padding rows = 0
 *   ar_moe_combine  out[token, :] = bf16(sum_slot bf16(d[row, :] * pair_w[pair]) (+ d2[row, :]))   pair_w NULL: plain sum
 *   ar_moe_rowdot   dw[pair] = bf16(<g[token, :], d[row, :]>)                                      (0 without a row)
 */
int ar_moe_route(const int64_t* expert_ids, int pairs, int e_begin, int e_local, int max_rows, int32_t* counts, int32_t* offsets,
                 int32_t* row_of_pair, int32_t* pair_of_row, int32_t* mtab, int32_t* num_mt, int32_t* ktab, int32_t* num_active,
                 void* stream);
int ar_moe_gather(const void* x_bf16, const int32_t* pair_of_row, const void* pair_w_bf16, int topk, int rows, int cols,
                  void* out_bf16, void* stream);
int ar_moe_combine(const void* d_bf16, const void* d2_bf16, const int32_t* row_of_pair, const void* pair_w_bf16, int tokens,
                   int topk, int cols, void* out_bf16, void* stream);
int ar_moe_rowdot(const void* g_bf16, const void* d_bf16, const int32_t* row_of_pair, int pairs, int topk, int cols,
                  void* dw_bf16, void* stream);

/* Fake-quant linear, grad-in: dX[T,K] = dY[T,N] · Wq[N,K] (ar_gemm_bf16 with Wq read MN-major).  The forward is
 * ar_qdq_fwd + ar_gemm_bf16, the weight gradient the grad-w GEMM + ar_fq_update below. */
int ar_fq_linear_bwd_dx(const ar_qspec* q, const void* dy_bf16, int64_t t, const void* wq_bf16, void* dx_bf16,
                        void* stream);

/*
 * Fused per-layer update of the sign-SGD loop (one pass, 14 B/weight): given Gq = dL/dWq as bf16 [rows, K] -- the plain
 * grad-w GEMM  ar_gemm_bf16(dY, X, a_mn_major=1, b_mn_major=1)  (autograd of F.linear rounds it to the weight dtype,
 * auto_round/wrapper.py:470-481), or under data parallelism the reduce-scattered sum over ranks -- it performs, for rows
 * [row0, row1) of the layer:
 *   fake-quant backward (closed form of autograd through the @register_dtype function, wrapper.py:273-290)
 *   -> if (*flag) best_* = PRE-update parameters (collect_best_params, compressors/utils.py:205-217)
 *   -> p -= lr * sign(grad), min/max_scale clamped to [0, clamp_hi]            (SignSGD.step, sign_sgd.py:356-389)
 *   -> wq_out rows = qdq(W; V', scales') for the next iteration's GEMMs          (WrapperLinear._qdq_weight)
 * v [N,Kpad], min_scale (NULL for mx/nv), max_scale [G] are updated in place; gq is indexed from row gq_row0 (a rank's
 * shard buffer starts at its first row).  dv_dbg/dmn_dbg/dmx_dbg (optional) receive the pre-sign gradients.
 * lr = lr_table[2*it] for V, lr_table[2*it+1] for the scales, it = *it_ptr when it_ptr is given (CUDA-graph replay),
 * else iter.
 * has_grad (optional, device): *has_grad == 0 means the layer received no gradient (an expert no token was routed to):
 * SignSGD skips it (sign_sgd.py:274-276), only the best-parameter snapshot still includes it.
 * codes_out / gparams_out (optional, both or none; bits <= 4, not per-row): instead of wq_out the shard's new fake-quant
 * weight leaves in WIRE form for the data-parallel all-gather -- one u32 of eight 4-bit codes per 8 elements (indexed from
 * row0) and {a, off} fp32 per group -- a quarter of the bf16 bytes; ar_wq_decode rebuilds the identical bf16 weight.
 */
int ar_fq_update(const ar_qspec* q, const void* w_bf16, float* v, float* min_scale, float* max_scale,
                 const void* wmin_bf16, const void* wmax_bf16, const float* gscale, const void* gq_bf16, int gq_row0,
                 int row0, int row1, float* best_v, float* best_min_scale, float* best_max_scale, const int32_t* flag,
                 const float* lr_table, int iter, const int32_t* it_ptr, float clamp_hi, void* wq_out_bf16,
                 float* dv_dbg, float* dmn_dbg, float* dmx_dbg, const int32_t* has_grad, void* codes_out, void* gparams_out,
                 void* stream);
/*
 * wq_out[N,K] (bf16) from `world` all-gathered wire segments of seg_bytes each: segment r = [codes of rows r*N/world ..
 * | {a, off} pairs of those rows]; value = bf16(a * (code - off)) for the int types, bf16(a * e2m1(code)) for MXFP4 / NVFP4 --
 * the same values ar_fq_update would have written to wq_out (int sym: a zero comes back as +0 where s * (-0) gave -0).
 */
int ar_wq_decode(const ar_qspec* q, const void* segments, int64_t seg_bytes, int world, void* wq_out_bf16, void* stream);

/*
 * Masked MSE + its gradient in one pass (auto_round/.../sign_round/quantizer.py:127-158, :789-803):
 *   *loss_sum += sum(((pred*m) - (ref*m))^2)                       (double, UNnormalised, atomically accumulated)
 *   dpred = bf16( ((2*inv_numel) * ((pred*m) - (ref*m))) * upstream ) * m      upstream = 1000 (loss*1000).backward()
 * pred/ref bf16 [rows, cols]; row_mask (uint8 [rows], 1 = valid token) may be NULL; dpred may be NULL.
 */
int ar_mse_fwd_bwd(const void* pred_bf16, const void* ref_bf16, const uint8_t* row_mask, int64_t rows, int64_t cols,
                   float inv_numel, float upstream, double* loss_sum, void* dpred_bf16, void* stream);

/*
 * Best-iteration bookkeeping on the device (no host sync in the loop; quantizer.py:477-515):
 *   mean = fp32(*loss_sum * inv_numel); total = mean * inv_num_elm  (= loss.item()/num_elm)
 *   state[0]=best_loss state[1]=last_loss state[2]=best_iter;  *flag = (total < best_loss);  loss_hist[iter]=total
 *   *loss_sum is reset to 0 for the next iteration.  iter==0 initialises best_loss to FLT_MAX.
 *   inv_num_elm_ptr / it_ptr (device, optional) override the by-value arguments: the loop schedule then lives
 *   entirely on the device and the whole iteration can be replayed as one CUDA graph.
 */
int ar_best_update(double* loss_sum, double inv_numel, double inv_num_elm, int iter, const double* inv_num_elm_ptr,
                   const int32_t* it_ptr, double* state, int32_t* flag, float* loss_hist, void* stream);

/*
 * Device-side loop schedule (replaces the python loop variable so that one iteration = one CUDA graph):
 *   ar_sched_load: cur_idx32/64[0..count) = idx_table[*it_ptr][0..count); *cur_inv_num_elm = inv_num_elm_table[*it_ptr]
 *                  (IndexSampler batches drawn up-front, compressors/utils.py:388-438)
 *   ar_iter_advance: ++*it_ptr
 */
int ar_sched_load(const int32_t* idx_table, const double* inv_num_elm_table, const int32_t* it_ptr, int count,
                  int32_t* cur_idx32, int64_t* cur_idx64, double* cur_inv_num_elm, void* stream);
int ar_iter_advance(int32_t* it_ptr, void* stream);

/* Gather `count` sample rows of `row_elems` bf16 each: dst[i] = src[idx[i]]  (BlockForwardRunner._select_batch). */
int ar_gather_rows(const void* src_bf16, const int32_t* idx, int count, int64_t row_elems, void* dst_bf16,
                   void* stream);

/*
 * Fused elementwise ops of a Llama-family decoder block (the non-GEMM work between the fake-quant linears of the
 * block forward/backward that `quantize_block` drives through the HF layer; they replace ATen eager chains, not a
 * reference kernel).  bf16 in/out, fp32 math, same rounding points as the HF eager code.
 *   rmsnorm: y = w * bf16(x * rsqrt(mean(x^2) + eps));  rstd [rows] saved for backward; bwd gives dx only (w frozen)
 *   rope:    x [B,S,H,D] contiguous, cos/sin [table_batch,S,D]; backward != 0 applies the transposed rotation
 *   swiglu:  h = bf16(silu(gate)) * up ;  bwd: dgate, dup
 */
int ar_rmsnorm_fwd(const void* x_bf16, const void* w_bf16, float eps, int64_t rows, int hidden, void* y_bf16, float* rstd,
                   void* stream);
int ar_rmsnorm_bwd(const void* dy_bf16, const void* x_bf16, const void* w_bf16, const float* rstd, int64_t rows, int hidden,
                   void* dx_bf16, int accumulate, void* stream);
int ar_rope(const void* x_bf16, const void* cos_bf16, const void* sin_bf16, int64_t b, int s, int h, int d, int table_batch,
            int backward, void* out_bf16, void* stream);
int ar_swiglu_fwd(const void* gate_bf16, const void* up_bf16, int64_t numel, void* h_bf16, void* stream);
int ar_swiglu_bwd(const void* dh_bf16, const void* gate_bf16, const void* up_bf16, int64_t numel, void* dgate_bf16,
                  void* dup_bf16, void* stream);

/*
 * INT pack (GPTQ-compatible int32 words along K, stored transposed) -- replaces
 *   auto_round_extension/torch/qlinear_torch_zp.py:93-150 (zp_minus_one=1, sym: zp_const = 2^(bits-1))
 *   auto_round_extension/torch/qlinear_torch.py:110-168, :170-281 (zp_minus_one=0, zp tensor)
 * in:  wq bf16 [N,K] (qdq weight), scale fp16 [N,G'] (G' = ceil(K/g)), zp fp32 [N,G'] or NULL (+zp_const)
 * out: qweight i32 [K*bits/32, N]; qzeros i32 [G', N*bits/32]; scales_t fp16 [G', N]; g_idx i32 [K]
 */
int ar_pack_int(const void* wq_bf16, const void* scale_f16, const float* zp, int zp_const, int n, int k, int bits,
                int group_size, int zp_minus_one, int32_t* qweight, int32_t* qzeros, void* scales_t_f16,
                int32_t* g_idx, void* stream);
/* inverse (tests / round trips): W'[N,K] bf16 = (code - zp) * scale, as triton_utils/dequant.py:54-117 */
int ar_unpack_int(const int32_t* qweight, const int32_t* qzeros, const void* scales_t_f16, int n, int k, int bits,
                  int group_size, int zp_minus_one, void* w_bf16, int32_t* codes_or_null, void* stream);

/*
 * AWQ "GEMM" layout, 4 bit -- WQLinear_GEMM.from_linear, auto_round/export/export_to_awq/utils.py:197-273.  Words run
 * along N (ar_pack_int packs along K): word j of row k holds the codes of output columns 8j .. 8j+7, column 8j+i at bit
 * 4 * [0,4,1,5,2,6,3,7][i]; qzeros packs the zero-points the same way (zp NULL: zp_const fills every nibble).
 * in:  wq bf16 [N,K], scale fp16 [N,G] (G = K / group_size; group_size -1 = K), zp fp32 [N,G] or NULL (+zp_const)
 * out: qweight i32 [K, N/8]; qzeros i32 [G, N/8]; scales fp16 [G, N]
 * AR_E_BADARG when K % group_size != 0 or N % 8 != 0 (the reference's "shape mismatch"); AR_E_UNSUPPORTED when
 * group_size % 8 != 0.
 */
int ar_pack_awq(const void* wq_bf16, const void* scale_f16, const float* zp, int zp_const, int n, int k, int group_size,
                int32_t* qweight, int32_t* qzeros, void* scales_f16, void* stream);
/* inverse (tests / round trips): W'[N,K] bf16 = (code - zero) * scale, as dequantize_gemm (utils.py:45-101); either
 * output may be NULL */
int ar_unpack_awq(const int32_t* qweight, const int32_t* qzeros, const void* scales_f16, int n, int k, int group_size,
                  void* w_bf16_or_null, int32_t* codes_or_null, void* stream);

/*
 * FP4 pack -- auto_round/export/export_to_autoround/qlinear_fp.py:141-193, :235-265
 * nv: weight_packed u8 [N,K/2], weight_scale e4m3 bytes [N,K/16]; scale_f32 = layer.scale, gscale device scalar
 * mx: weight_packed u8 [N,K/2], weight_scale u8 [N,K/32] = clamp(e+127,0,255); exp_bf16 = layer.scale
 */
int ar_pack_fp4_nv(const void* wq_bf16, const float* scale_f32, const float* gscale, int n, int k,
                   uint8_t* weight_packed, uint8_t* weight_scale_e4m3, void* stream);
int ar_pack_fp4_mx(const void* wq_bf16, const void* exp_bf16, int n, int k, uint8_t* weight_packed,
                   uint8_t* weight_scale_e8m0, void* stream);
int ar_unpack_fp4(const uint8_t* weight_packed, int n, int k, void* values_bf16, void* stream);

/*
 * Scale searches of the optimized RTN (iters == 0 default) and of the alg_ext init scale -- replace
 *   auto_round/data_type/int.py:24-86   search_scales  (+ the clip and bf16 qdq of opt_rtn_int_sym, :89-122)
 *   auto_round/data_type/nvfp.py:331-385 search_nvfp4_scale      auto_round/data_type/mxfp.py:103-169 search_mx_scale
 * w bf16 [N,K]; qw = loss weights from the importance matrix: [K] when qw_row_stride == 0 (K padded with 1e-5 as the
 * reference does), [N, qw_row_stride >= Kpad] when the host materialised the zero-handled matrix (gguf.py:437-484),
 * NULL = 1.  coef[ncand] is the candidate table, base candidate first: int: -(2^(bits-1) - step*i) (int.py:59-64),
 * nv: 1.0 then 0.50..1.51, mx: 1.0, 0.5, 2.0.  Outputs are per group, [N * ceil(K/g)] fp32.
 *   ar_search_scale_int: scale (bf16-valued, threshold-clipped); wq (bf16 [N,K], may be NULL) = the opt-RTN qdq weight
 *   ar_search_scale_nv / _mx: the winning coefficient (the `init_scale` / `max_scales` of the reference)
 *   gscale (nv): device scalar 448*6/amax of THIS tensor -- the search ignores the layer's fused global scale
 */
int ar_search_scale_int(const void* w_bf16, const float* qw, long long qw_row_stride, const float* coef, int ncand,
                        const ar_qspec* spec, float* scale, void* wq_bf16, void* stream);
int ar_search_scale_nv(const void* w_bf16, const float* qw, long long qw_row_stride, const float* gscale,
                       const float* coef, int ncand, const ar_qspec* spec, float* coeff_out, void* stream);
int ar_search_scale_mx(const void* w_bf16, const float* qw, long long qw_row_stride, const float* coef, int ncand,
                       const ar_qspec* spec, float* coeff_out, void* stream);
/*
 * Outlier-suppressed block loss of enable_alg_ext -- replaces SignRoundV2Quantizer._get_loss
 * (auto_round/algorithms/quantization/sign_roundv2/quantizer.py:362-399; torch.topk over numel elements per iteration).
 *   ar_absdiff_hist:   hist[32768] (u32, zero before the first call) += histogram of the bf16 bit pattern of |pred - ref|
 *   ar_topk_threshold: from the histogram and k = max(1, numel / 1000): sel[0] = threshold pattern, sel[1] = how many elements
 *                      AT the threshold are dropped, sel[2] = 0 (tie counter); re-zeroes hist
 *   ar_topk_threshold_ranks: data-parallel form.  hist_all = the `world` ranks' histograms [world, 32768] (one all-gather);
 *                      the threshold comes from their sum (the top-k is global over the batch) and the ties at the threshold
 *                      are handed out in rank order so that exactly k elements are dropped over all ranks; re-zeroes
 *                      hist_local (this rank's histogram)
 *   ar_mse_outlier_fwd_bwd: loss_sum (double, unnormalised) += sum((|pred-ref| * row_mask * keep)^2); dpred (bf16, nullable)
 *                      = d(upstream * mean(...)) / d pred.  keep drops patterns > sel[0] and the first sel[1] found at sel[0].
 *                      numel_total > 0: the mean runs over that many elements (the global batch of a data-parallel
 *                      iteration) instead of rows * cols.
 */
int ar_absdiff_hist(const void* pred_bf16, const void* ref_bf16, int64_t numel, uint32_t* hist, void* stream);
int ar_topk_threshold(uint32_t* hist, int64_t k, uint32_t* sel, void* stream);
int ar_topk_threshold_ranks(const uint32_t* hist_all, int world, int rank, uint32_t* hist_local, int64_t k, uint32_t* sel,
                            void* stream);
int ar_mse_outlier_fwd_bwd(const void* pred_bf16, const void* ref_bf16, const uint8_t* row_mask, int64_t rows, int64_t cols,
                           int64_t numel_total, float upstream, uint32_t* sel, double* loss_sum, void* dpred_bf16,
                           void* stream);
/* importance matrix: imatrix[k] += sum over rows of x[row,k]^2 (algorithms/quantization/rtn/quantizer.py:86-105) */
int ar_imatrix_accum(const void* x_bf16, long long rows, int k, float* imatrix, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* AR_B200_H_ */
