// bf16 GEMMs of the fake-quant linear on Hopper tensor cores (wgmma) for sm_90a.
//
//   D[M,N] = A[M,K] · B[N,K]ᵀ ,  fp32 accumulate in registers, operands staged by TMA into 128B-swizzled smem.
//
// One persistent CTA per SM (132 on an H100 SXM), warp-specialised:
//   warps 0..7  two consumer warpgroups: warpgroup w issues wgmma.m64n256k16 for rows [64w, 64w+64) of the 128 x 256
//               tile, then runs the epilogue of its own rows
//   warp 8      TMA producer   (one elected lane; mbarrier full/empty ring; keeps loading the next tile's stages while
//                               the consumers run the epilogue of the current one)
// Tiles are 128 x 256: m64n256k16 reads 17 % fewer smem bytes per FLOP than m64n128k16, and each staged A slab feeds
// twice the output columns.
// Each operand may be K-major (reduction dim contiguous) or MN-major (row dim contiguous), which covers the
// three GEMMs of a linear without any transposed copies (wgmma's transpose bits read MN-major bf16 directly):
//   forward   Y  = X  · Wqᵀ      A = X  [T,K]  K-major      B = Wq [N,K]  K-major
//   grad-in   dX = dY · Wq       A = dY [T,N]  K-major      B = Wq [N,K]  as [K_out, N_red]: MN-major
//   grad-w    dW = dYᵀ· X        A = dY [T,N]  as [N_out, T_red]: MN-major   B = X [T,K] as [K_out, T_red]: MN-major
// Epilogue: fp32 registers -> (+bias) -> bf16 -> global, straight from each warpgroup's accumulators (a quad transpose
// gives 16-byte stores; clipped to the problem); no smem staging and no consumer barrier.  The fake-quant backward of
// the grad-w GEMM's bf16 dWq runs in the per-layer update kernel (ar_fq_update, ar_qdq.cu).
// FLOPs per launch = 2*M*N*K; roofline = dense bf16 tensor peak (MEASURED_PEAKS.json: bf16_tflops).
#include <cuda.h>

#include <stdlib.h>

#include <atomic>
#include <mutex>

#include "ar_common.cuh"

namespace ar {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_N = 256;
constexpr int BLOCK_K = 64;           // 64 bf16 = 128 B = one swizzle atom row
constexpr int WGMMA_K = 16;
constexpr int kStages = 4;
constexpr int kConsumerThreads = 256; // two warpgroups
constexpr int kProducerWarp = 8;
constexpr int kNumThreads = kConsumerThreads + 32;
constexpr int kTableRows = 256;       // row granularity of the MoE routing tables (GROUP_M entries, padded segments)

// ------------------------------------------------------------------------------------------------ PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n"
      ".reg .b32 rx;\n"
      ".reg .pred px;\n"
      "elect.sync rx|px, 0xFFFFFFFF;\n"
      "@px mov.s32 %0, 1;\n"
      "}\n"
      : "+r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE;\n"
      "bra WAIT_LOOP;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(smem_dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// wgmma shared-memory matrix descriptor, SWIZZLE_128B:
//   [0,14) start>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 | [49,52) base offset = 0 (1024-byte aligned atoms) | [62,64) 1 = 128B
// K-major:  SBO = 8 rows * 128 B (next 8-row core-matrix group), LBO unused; K step (16 elem) = +32 B inside the atom
// MN-major: SBO = 8 k-rows * 128 B, LBO = 64 k-rows * 128 B (next 64-wide MN atom); K step (16 rows) = +2048 B
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFFu);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// D(64 x 256, fp32, registers) += A(64 x 16) · B(256 x 16)ᵀ.  Fragment of thread (warp w of the warpgroup, lane l):
// d[4j + 2h + e] = D[16w + l/4 + 8h][8j + 2(l%4) + e], j in [0, 32).
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "{\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
      "}, "
      "%128, %129, 1, 1, 1, %130, %131;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]),
        "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]),
        "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
        "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]),
        "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]),
        "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]),
        "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]),
        "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]),
        "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]),
        "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]),
        "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]),
        "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]),
        "+f"(d[126]), "+f"(d[127])
      : "l"(desc_a), "l"(desc_b), "n"(TA), "n"(TB)
      : "memory");
}

// ---------------------------------------------------------------------------------------- kernel params
// Grouped (ragged per-expert) GEMMs of the MoE path: tiles are resolved through small device-side tables written by the
// routing kernel of the same iteration (ar_moe_route), so launches stay static and graph-capturable.
//   GROUP_M  forward / grad-in of all experts in one launch: A rows are the routed tokens sorted by expert, every expert's
//            segment padded to 256 rows; table[i] = {m0, expert} per 256-row segment tile (two 128-row GEMM tiles); B (the
//            stacked per-expert weights) is offset by expert * b_group_rows (a row offset for a K-major B, a reduction
//            offset for an MN-major B)
//   GROUP_K  grad-w: one [N, K] output per ACTIVE expert, reduction over that expert's token rows;
//            table[i] = {expert, k_off, k_len}; D rows are offset by expert * d_group_rows
enum { GROUP_NONE = 0, GROUP_M = 1, GROUP_K = 2 };
struct GroupDesc {
  int mode;
  const int32_t* table;
  const int32_t* num;             // device scalar: entries in `table`
  int b_group_rows;
  int d_group_rows;
};

struct TileInfo {
  int m0, n0;                     // A-row / B-row coordinate of the tile
  int d_m0, d_n0;                 // output coordinates
  int a_koff, b_koff;             // reduction-coordinate offsets of the A / B loads
  int num_kb;
};

struct GemmParams {
  int m, n, k;                    // logical problem: D[m,n] = A[m,k] B[n,k]^T
  GroupDesc grp;
  // host-only (grouped launches): extents of the tensor maps when they differ from the logical problem, and the tile bound
  int a_rows_map, b_rows_map, b_k_map, d_rows_map, max_tiles;
  int m_tiles, n_tiles;
  uint16_t* d;                    // bf16 output, row pitch ldd, d_rows x n
  int64_t ldd;
  int d_rows;
  const uint16_t* bias;           // optional [n]
  unsigned int* tile_ctr;         // dynamic tile scheduler: ticket counter of this launch (0 at launch, reset to 0 at exit)
  // Unused: keeps the parameter block above 128 bytes.  At 128 bytes or less nvcc reads it through uniform registers and
  // schedules every instantiation differently (155-159 registers instead of 156-158); the rates in DESIGN §4.1 were
  // measured on the code generated for the larger block.
  uint8_t pad[16];
};
static_assert(sizeof(GemmParams) > 128, "see GemmParams::pad");

// Shared memory: the 4 x 48 KB operand ring (192 KB), then the mbarriers and the ticket slots.
struct Smem {
  static constexpr int kABytes = BLOCK_M * BLOCK_K * 2;       // 16 KB
  static constexpr int kBBytes = BLOCK_N * BLOCK_K * 2;       // 32 KB
  static constexpr int kAOff = 0;
  static constexpr int kBOff = kStages * kABytes;
  static constexpr int kBarOff = kBOff + kStages * kBBytes;
  static constexpr int kTotal = kBarOff + 512 + 1024;         // + slack to align the base to 1024 B (SWIZZLE_128B atoms)
  static_assert(kTotal <= 227 * 1024, "GEMM shared memory exceeds the sm_90 per-block limit");
};
constexpr int kSchedSlots = 8;

// tile order: groups of 8 M-tiles sweep all N-tiles, so the concurrent CTAs share A/B tiles in L2
__device__ __forceinline__ void tile_coords(int t, int m_tiles, int n_tiles, int& mt, int& nt) {
  constexpr int GM = 8;
  const int per_group = GM * n_tiles;
  const int grp = t / per_group;
  const int first = grp * GM;
  const int gm = min(GM, m_tiles - first);
  const int in = t - grp * per_group;
  mt = first + in % gm;
  nt = in / gm;
}

template <bool B_MN>
__device__ __forceinline__ TileInfo resolve_tile(const GemmParams& p, int t, int m_tiles, int num_kb_static) {
  TileInfo ti;
  int mt, nt;
  if (p.grp.mode == GROUP_K) {
    const int per = p.m_tiles * p.n_tiles;
    const int ae = t / per;
    tile_coords(t - ae * per, p.m_tiles, p.n_tiles, mt, nt);
    const int e = p.grp.table[3 * ae], koff = p.grp.table[3 * ae + 1], klen = p.grp.table[3 * ae + 2];
    ti.m0 = mt * BLOCK_M;
    ti.n0 = nt * BLOCK_N;
    ti.d_m0 = e * p.grp.d_group_rows + ti.m0;
    ti.d_n0 = ti.n0;
    ti.a_koff = koff;
    ti.b_koff = koff;
    ti.num_kb = klen / BLOCK_K;
    return ti;
  }
  tile_coords(t, m_tiles, p.n_tiles, mt, nt);
  ti.n0 = nt * BLOCK_N;
  ti.d_n0 = ti.n0;
  ti.a_koff = 0;
  ti.b_koff = 0;
  ti.num_kb = num_kb_static;
  if (p.grp.mode == GROUP_M) {
    constexpr int per_entry = kTableRows / BLOCK_M;
    const int en = mt / per_entry;
    const int m0 = p.grp.table[2 * en] + (mt % per_entry) * BLOCK_M, e = p.grp.table[2 * en + 1];
    ti.m0 = m0;
    if (B_MN) ti.b_koff = e * p.grp.b_group_rows; else ti.n0 += e * p.grp.b_group_rows;
  } else {
    ti.m0 = mt * BLOCK_M;
  }
  ti.d_m0 = ti.m0;
  return ti;
}

// bf16 store epilogue straight from one warpgroup's accumulators.  Thread (warp w of the warpgroup, lane l) holds
// D[16w + l/4 + 8h][8j + 2(l%4) + e] in acc[4j + 2h + e]; `row0` is the output row of h = 0.  After the bias and the
// rounding to bf16 pairs, a 4 x 4 transpose inside each quad (two shfl.xor rounds) hands lane q of the quad the 8
// consecutive columns 8(4b + q) .. +7 of its row, so each 16-byte store of a warp writes 8 rows x 64 contiguous bytes.
__device__ __forceinline__ void epilogue_store(const GemmParams& p, const float (&acc)[BLOCK_N / 2], int row0, int n0, int lane) {
  const int q = lane & 3;
  const bool odd = (q & 1) != 0, hi = (q & 2) != 0;
#pragma unroll
  for (int b = 0; b < BLOCK_N / 32; ++b) {
    uint32_t v[2][4];                                      // [h][s]: bf16 pair of columns 8(4b + s) + 2q, +1
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      const int j = 4 * b + s;
      float x[4] = {acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3]};
      if (p.bias) {
        // F.linear under autocast: bf16 GEMM result (+bias in fp32 inside the fused epilogue)
        const int col = n0 + 8 * j + 2 * q;
        const float b0 = col < p.n ? bf16_bits_to_f32(p.bias[col]) : 0.f;
        const float b1 = col + 1 < p.n ? bf16_bits_to_f32(p.bias[col + 1]) : 0.f;
        if (col < p.n) { x[0] += b0; x[2] += b0; }
        if (col + 1 < p.n) { x[1] += b1; x[3] += b1; }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h)
        v[h][s] = (uint32_t)f32_to_bf16_bits(x[2 * h]) | ((uint32_t)f32_to_bf16_bits(x[2 * h + 1]) << 16);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      uint32_t* u = v[h];
      // round 1 (lanes q, q^1): swap the slots whose bit 0 differs from q's; round 2 (q, q^2): the same for bit 1.
      // Afterwards slot s of lane q holds the pair lane s had for j = 4b + q.
      uint32_t t0 = __shfl_xor_sync(0xffffffffu, odd ? u[0] : u[1], 1);
      uint32_t t1 = __shfl_xor_sync(0xffffffffu, odd ? u[2] : u[3], 1);
      if (odd) { u[0] = t0; u[2] = t1; } else { u[1] = t0; u[3] = t1; }
      t0 = __shfl_xor_sync(0xffffffffu, hi ? u[0] : u[2], 2);
      t1 = __shfl_xor_sync(0xffffffffu, hi ? u[1] : u[3], 2);
      if (hi) { u[0] = t0; u[1] = t1; } else { u[2] = t0; u[3] = t1; }
      const int row = row0 + 8 * h, col = n0 + 8 * (4 * b + q);
      if (row >= p.d_rows || col >= p.n) continue;
      uint16_t* o = p.d + (int64_t)row * p.ldd + col;
      if (col + 8 <= p.n) {
        *reinterpret_cast<U4*>(o) = U4{u[0], u[1], u[2], u[3]};
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i)                        // unrolled: constant register indices
          if (col + i < p.n) o[i] = (uint16_t)(u[i >> 1] >> (16 * (i & 1)));
      }
    }
  }
}

// ------------------------------------------------------------------------------------------- the kernel
// Tile scheduling is DYNAMIC: the producer lane draws tile tickets from a global counter (one atomicAdd per tile, issued
// one tile ahead) and publishes each ticket to the eight consumer warps through a small shared-memory ring with full/empty
// mbarriers.  With static striding a CTA that starts late still owns its full share of tiles; that is exactly what happens
// when NCCL kernels of the data-parallel exchange hold a few SMs while a GEMM launches (they cannot co-reside with a 200 KB
// CTA).  With tickets, late CTAs simply find the queue empty.  Ticket order = rasterised tile order, so concurrently
// running CTAs still work on neighbouring tiles (L2 reuse).  The CTA that draws the last terminal ticket resets the counter.
template <bool A_MN, bool B_MN>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const GemmParams p) {
  using L = Smem;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::kBarOff);
  uint64_t* full = bars;                          // [kStages]
  uint64_t* empty = bars + kStages;               // [kStages]
  uint64_t* sfull = bars + 2 * kStages;           // [kSchedSlots] ticket published
  uint64_t* sempty = sfull + kSchedSlots;         // [kSchedSlots] ticket read by all eight consumer warps
  volatile int32_t* stile = reinterpret_cast<volatile int32_t*>(sempty + kSchedSlots);   // [kSchedSlots]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // grouped launches read their tile count from the routing kernel's output
  const int grp_num = (p.grp.mode != GROUP_NONE) ? *p.grp.num : 0;
  const int m_tiles_dyn = (p.grp.mode == GROUP_M) ? grp_num * (kTableRows / BLOCK_M) : p.m_tiles;
  const int num_tiles = (p.grp.mode == GROUP_K) ? grp_num * p.m_tiles * p.n_tiles : m_tiles_dyn * p.n_tiles;
  const int num_kb = (p.k + BLOCK_K - 1) / BLOCK_K;
  constexpr uint32_t kConsumerWarps = kConsumerThreads / 32;

  if (warp == kProducerWarp && lane == 0) {
    prefetch_tmap(&map_a);
    prefetch_tmap(&map_b);
    for (int i = 0; i < kStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], kConsumerWarps); }
    for (int i = 0; i < kSchedSlots; ++i) { mbar_init(&sfull[i], 1); mbar_init(&sempty[i], kConsumerWarps); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == kProducerWarp) {
    // ===================================================================== TMA producer + ticket scheduler
    if (elect_one()) {
      uint32_t it = 0, n = 0;
      int t = (int)atomicAdd(p.tile_ctr, 1u), t_next = 0;
      for (;; ++n) {
        const uint32_t slot = n % kSchedSlots, ph = (n / kSchedSlots) & 1u;
        mbar_wait(&sempty[slot], ph ^ 1u);                 // all consumers are done with the ticket 8 tiles back
        stile[slot] = t;
        mbar_arrive(&sfull[slot]);
        if (t >= num_tiles) break;
        t_next = (int)atomicAdd(p.tile_ctr, 1u);           // next ticket: in flight while this tile's loads are issued
        const TileInfo ti = resolve_tile<B_MN>(p, t, m_tiles_dyn, num_kb);
        for (int kb = 0; kb < ti.num_kb; ++kb, ++it) {
          const uint32_t s = it % kStages, sph = (it / kStages) & 1u;
          mbar_wait(&empty[s], sph ^ 1u);
          mbar_expect_tx(&full[s], L::kABytes + L::kBBytes);
          uint8_t* sa = smem + L::kAOff + s * L::kABytes;
          uint8_t* sb = smem + L::kBOff + s * L::kBBytes;
          const int k0 = kb * BLOCK_K;
          if (!A_MN) {
            tma_load_2d(sa, &map_a, &full[s], ti.a_koff + k0, ti.m0);                 // box {64 k, 128 m}
          } else {
#pragma unroll
            for (int i = 0; i < BLOCK_M / 64; ++i)                                    // box {64 m, 64 k} per 64-wide atom
              tma_load_2d(sa + i * (64 * BLOCK_K * 2), &map_a, &full[s], ti.m0 + i * 64, ti.a_koff + k0);
          }
          if (!B_MN) {
            tma_load_2d(sb, &map_b, &full[s], ti.b_koff + k0, ti.n0);                 // box {64 k, 256 n}
          } else {
#pragma unroll
            for (int i = 0; i < BLOCK_N / 64; ++i)
              tma_load_2d(sb + i * (64 * BLOCK_K * 2), &map_b, &full[s], ti.n0 + i * 64, ti.b_koff + k0);
          }
        }
        t = t_next;
      }
      // every CTA draws exactly one terminal ticket; the holder of the LAST one re-arms the counter for the next launch
      if (t == num_tiles + (int)gridDim.x - 1) atomicExch(p.tile_ctr, 0u);
    }
  } else {
    // ===================================================================== consumer warpgroups: wgmma main loop + epilogue
    const int ctid = threadIdx.x;                          // 0..255
    const int wg = ctid >> 7;                              // rows [64 wg, 64 wg + 64) of the tile
    const int wrow = ((ctid & 127) >> 5) * 16 + (lane >> 2);
    // K-major operands: the second 64 rows start 64 * 128 B further; MN-major: the second 64-wide atom is 8 KB further
    constexpr uint32_t a_lbo = A_MN ? (BLOCK_K * 128) : 16, b_lbo = B_MN ? (BLOCK_K * 128) : 16;
    constexpr uint32_t a_kstep = A_MN ? (WGMMA_K * 128) : (WGMMA_K * 2), b_kstep = B_MN ? (WGMMA_K * 128) : (WGMMA_K * 2);
    uint32_t it = 0;
    for (uint32_t local_tile = 0;; ++local_tile) {
      const uint32_t slot = local_tile % kSchedSlots, ph = (local_tile / kSchedSlots) & 1u;
      mbar_wait(&sfull[slot], ph);
      const int t = stile[slot];
      __syncwarp();
      if (lane == 0) mbar_arrive(&sempty[slot]);
      if (t >= num_tiles) break;
      const TileInfo ti = resolve_tile<B_MN>(p, t, m_tiles_dyn, num_kb);

      float acc[BLOCK_N / 2];
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
      uint32_t prev = 0;
      for (int kb = 0; kb < ti.num_kb; ++kb, ++it) {
        const uint32_t s = it % kStages, sph = (it / kStages) & 1u;
        mbar_wait(&full[s], sph);
        const uint32_t sa = smem_u32(smem + L::kAOff + s * L::kABytes) + wg * (64 * 128);
        const uint32_t sb = smem_u32(smem + L::kBOff + s * L::kBBytes);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / WGMMA_K; ++k)
          wgmma_m64n256k16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, make_smem_desc(sa + k * a_kstep, a_lbo, 1024),
                                                      make_smem_desc(sb + k * b_kstep, b_lbo, 1024));
        wgmma_commit();
        wgmma_wait<1>();                                   // the previous stage's MMAs have retired: hand it back
        if (kb > 0 && lane == 0) mbar_arrive(&empty[prev]);
        prev = s;
      }
      wgmma_wait<0>();
      if (ti.num_kb > 0 && lane == 0) mbar_arrive(&empty[prev]);

      // each warpgroup stores its own 64 rows and moves on to the next ticket: no consumer-wide barrier
      epilogue_store(p, acc, ti.d_m0 + wg * 64 + wrow, ti.d_n0, lane);
    }
  }
}

// ------------------------------------------------------------------------------------------- host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (PFN_encodeTiled)f;
  });
  return fn;
}

// cuTensorMapEncodeTiled is a driver call and fails with CUDA_ERROR_INVALID_CONTEXT in a thread that has no current
// context.  A thread that has made no runtime call yet has none, and PyTorch's autograd device threads start that way
// (they skip cudaSetDevice when the device already matches), so the first GEMM of a backward can come from such a thread.
// cudaSetDevice makes the device's primary context current; once per thread.
static void ensure_context() {
  thread_local bool done = false;
  int dev = 0;
  if (!done && cudaGetDevice(&dev) == cudaSuccess && cudaSetDevice(dev) == cudaSuccess) done = true;
}

// 2-D bf16 tensor map: dim0 = contiguous dimension.  box = {box0, box1}, 128B swizzle (box0 * 2 B == 128 B).
static int make_map(CUtensorMap* map, const void* ptr, uint64_t dim0, uint64_t dim1, uint64_t stride1_elems, uint32_t box0,
                    uint32_t box1) {
  ensure_context();
  PFN_encodeTiled enc = get_encode();
  AR_REQUIRE(enc != nullptr, AR_E_DRIVER, "cuTensorMapEncodeTiled entry point not available");
  AR_REQUIRE(((uintptr_t)ptr & 15u) == 0, AR_E_BADARG, "TMA operand must be 16-byte aligned");
  AR_REQUIRE((stride1_elems * 2) % 16 == 0, AR_E_BADARG, "TMA leading dimension must be a multiple of 8 elements (got %llu)",
             (unsigned long long)stride1_elems);
  cuuint64_t gdim[2] = {dim0, dim1};
  cuuint64_t gstr[1] = {stride1_elems * 2};
  cuuint32_t box[2] = {box0, box1};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), gdim, gstr, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  AR_REQUIRE(r == CUDA_SUCCESS, AR_E_DRIVER, "cuTensorMapEncodeTiled failed (%d) dims=%llu,%llu stride=%llu box=%u,%u", (int)r,
             (unsigned long long)dim0, (unsigned long long)dim1, (unsigned long long)stride1_elems, box0, box1);
  return AR_OK;
}

static int check_device() {
  static int ok = -1;
  if (ok < 0) {
    int dev = 0, major = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    ok = (major == 9) ? 1 : 0;
  }
  AR_REQUIRE(ok == 1, AR_E_ARCH, "wgmma kernels need an sm_90 device");
  return AR_OK;
}

// ticket counters of the dynamic tile scheduler: one per launch in flight, handed out round-robin (a counter is back at 0
// when its kernel exits; 1024 launches later nothing of that kernel is still running on any stream)
constexpr int kCtrSlots = 1024;
__device__ unsigned int g_tile_ctr[kCtrSlots];

static unsigned int* next_tile_counter() {
  static unsigned int* base[64] = {nullptr};
  static std::atomic<unsigned> next{0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return nullptr;
  if (base[dev] == nullptr) {
    void* ptr = nullptr;
    if (cudaGetSymbolAddress(&ptr, g_tile_ctr) != cudaSuccess) return nullptr;
    base[dev] = (unsigned int*)ptr;
  }
  return base[dev] + (next.fetch_add(1) % kCtrSlots);
}

template <bool A_MN, bool B_MN>
static int launch(const void* a, const void* b, void* d, int m, int n, int k, int64_t lda, int64_t ldb, int64_t ldd,
                  const GemmParams& base, cudaStream_t st) {
  using L = Smem;
  auto kern = gemm_kernel<A_MN, B_MN>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::kTotal);
    AR_REQUIRE(e == cudaSuccess, (int)e, "cudaFuncSetAttribute(smem=%d): %s", L::kTotal, cudaGetErrorString(e));
    attr_set = true;
  }
  CUtensorMap ma, mb;
  int rc;
  const uint64_t a_rows = base.a_rows_map > 0 ? (uint64_t)base.a_rows_map : (uint64_t)m;
  if (!A_MN) rc = make_map(&ma, a, (uint64_t)k, a_rows, (uint64_t)lda, 64, BLOCK_M);         // stored [m, k]
  else rc = make_map(&ma, a, a_rows, (uint64_t)k, (uint64_t)lda, 64, BLOCK_K);               // stored [k, m]
  if (rc) return rc;
  const uint64_t b_rows = base.b_rows_map > 0 ? (uint64_t)base.b_rows_map : (uint64_t)n;
  const uint64_t b_k = base.b_k_map > 0 ? (uint64_t)base.b_k_map : (uint64_t)k;
  if (!B_MN) rc = make_map(&mb, b, b_k, b_rows, (uint64_t)ldb, 64, BLOCK_N);
  else rc = make_map(&mb, b, b_rows, b_k, (uint64_t)ldb, 64, BLOCK_K);
  if (rc) return rc;
  AR_REQUIRE(((uintptr_t)d & 15u) == 0, AR_E_BADARG, "GEMM output must be 16-byte aligned");
  AR_REQUIRE(ldd % 8 == 0, AR_E_BADARG, "GEMM output leading dimension must be a multiple of 8 elements (got %lld)",
             (long long)ldd);
  GemmParams p = base;
  p.d = (uint16_t*)d;
  p.ldd = ldd;
  p.d_rows = base.d_rows_map > 0 ? base.d_rows_map : m;
  p.m = m; p.n = n; p.k = k;
  p.tile_ctr = next_tile_counter();
  AR_REQUIRE(p.tile_ctr != nullptr, AR_E_DRIVER, "tile counter symbol not available on this device");
  p.m_tiles = (m + BLOCK_M - 1) / BLOCK_M;
  p.n_tiles = (n + BLOCK_N - 1) / BLOCK_N;
  const int tiles = base.max_tiles > 0 ? base.max_tiles : p.m_tiles * p.n_tiles;
  const int ctas = tiles < sm_count() ? tiles : sm_count();
  kern<<<(unsigned)ctas, kNumThreads, L::kTotal, st>>>(ma, mb, p);
  AR_CHECK_LAUNCH();
  return AR_OK;
}

}  // namespace ar

using namespace ar;

extern "C" int ar_gemm_bf16(const void* a, const void* b, void* d, int m, int n, int k, int a_mn, int b_mn, int64_t lda,
                            int64_t ldb, int64_t ldd, const void* bias, void* stream) {
  AR_REQUIRE(a && b && d && m > 0 && n > 0 && k > 0, AR_E_BADARG, "bad gemm args m=%d n=%d k=%d", m, n, k);
  if (int rc = check_device()) return rc;
  GemmParams p{};
  p.bias = (const uint16_t*)bias;
  cudaStream_t st = (cudaStream_t)stream;
  if (!a_mn && !b_mn) return launch<false, false>(a, b, d, m, n, k, lda, ldb, ldd, p, st);
  if (!a_mn && b_mn) return launch<false, true>(a, b, d, m, n, k, lda, ldb, ldd, p, st);
  if (a_mn && !b_mn) return launch<true, false>(a, b, d, m, n, k, lda, ldb, ldd, p, st);
  return launch<true, true>(a, b, d, m, n, k, lda, ldb, ldd, p, st);
}

extern "C" int ar_gemm_bf16_grouped(const void* a, const void* b, void* d, int mode, int rows, int n, int k, int a_mn, int b_mn,
                                    int64_t lda, int64_t ldb, int64_t ldd, int group_rows, int num_groups,
                                    const int32_t* table, const int32_t* num, int max_entries, int a_features, void* stream) {
  AR_REQUIRE(a && b && d && table && num && rows > 0 && n > 0 && k > 0 && group_rows > 0 && num_groups > 0 && max_entries > 0,
             AR_E_BADARG, "bad grouped gemm args");
  AR_REQUIRE(mode == GROUP_M || mode == GROUP_K, AR_E_BADARG, "mode must be 1 (GROUP_M) or 2 (GROUP_K)");
  if (int rc = check_device()) return rc;
  GemmParams p{};
  p.grp.mode = mode;
  p.grp.table = table;
  p.grp.num = num;
  cudaStream_t st = (cudaStream_t)stream;
  const int n_tiles = (n + BLOCK_N - 1) / BLOCK_N;
  if (mode == GROUP_M) {
    // D[rows, n] = A[rows, k] * B_e^T, e = expert of the row tile.  B stacked over experts: K-major [G * group_rows, k]
    // (forward: group_rows = n) or stored [G * group_rows, n] read MN-major with the reduction inside the expert's rows
    // (grad-in: group_rows = k)
    AR_REQUIRE(!a_mn, AR_E_UNSUPPORTED, "GROUP_M: A must be K-major");
    AR_REQUIRE(rows % kTableRows == 0, AR_E_UNSUPPORTED, "GROUP_M: the padded row count must be a multiple of 256");
    p.grp.b_group_rows = group_rows;
    p.max_tiles = max_entries * (kTableRows / BLOCK_M) * n_tiles;
    if (!b_mn) {
      p.b_rows_map = group_rows * num_groups;
      return launch<false, false>(a, b, d, rows, n, k, lda, ldb, ldd, p, st);
    }
    p.b_k_map = group_rows * num_groups;
    return launch<false, true>(a, b, d, rows, n, k, lda, ldb, ldd, p, st);
  }
  // GROUP_K: D_e[n_out = `n`... ] -- here the logical problem per active expert is D[m = group_rows, n] = A^T B over that
  // expert's rows; A stored [rows, m] and B stored [rows, n] (both MN-major), D stacked [G * group_rows, n]
  AR_REQUIRE(a_mn && b_mn, AR_E_UNSUPPORTED, "GROUP_K: A and B must be MN-major (stored [rows, features])");
  AR_REQUIRE(group_rows % kTableRows == 0, AR_E_UNSUPPORTED,
             "GROUP_K: the row pitch of the stacked output must be a multiple of 256 (pad the per-expert slab)");
  AR_REQUIRE(a_features > 0 && a_features <= group_rows, AR_E_BADARG, "GROUP_K: a_features must be in (0, group_rows]");
  p.a_rows_map = a_features;                 // feature columns of A beyond the real count are zero-filled by TMA
  p.grp.d_group_rows = group_rows;
  p.d_rows_map = group_rows * num_groups;
  p.max_tiles = max_entries * (group_rows / BLOCK_M) * n_tiles;
  return launch<true, true>(a, b, d, group_rows, n, rows, lda, ldb, ldd, p, st);
}

extern "C" int ar_fq_linear_bwd_dx(const ar_qspec* q, const void* dy, int64_t t, const void* wq, void* dx, void* stream) {
  AR_REQUIRE(q && dy && wq && dx && t > 0, AR_E_BADARG, "null pointer");
  // dX[T,K] = dY[T,N] · Wq[N,K]:  A = dY (K-major over N), B = Wq viewed as [K_out, N_red] -> MN-major
  return ar_gemm_bf16(dy, wq, dx, (int)t, q->k, q->n, 0, 1, q->n, q->k, q->k, nullptr, stream);
}
