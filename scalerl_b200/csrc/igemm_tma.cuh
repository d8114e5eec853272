// TMA-fed implicit-GEMM mainloop on Hopper warpgroup MMA (wgmma, sm_90a).
//
//   warp 8 lane 0 : producer -- one cp.async.bulk.tensor (TMA) box per operand block per stage; im2col is expressed
//                   as a multi-dimensional box over the NHWC activation (negative / out-of-range coordinates are
//                   zero-filled by the TMA unit, which gives convolution padding and batch tails for free)
//   warps 0-7     : two consumer warpgroups; warpgroup g owns columns [g BN/2, (g+1) BN/2) of the 128 x BN tile: it issues
//                   the wgmma (two m64 halves per K = 16 step), keeps the accumulator in registers and runs the epilogue
//                   (registers -> shared-memory row hand-off -> global)
//   full[s]  : mbarrier, 1 arrival (producer's arrive.expect_tx) + TMA complete_tx bytes
//   empty[s] : mbarrier, 8 arrivals (one per consumer warp, once the wgmma group reading the stage retired: the consumers keep one
//              k-block's MMAs in flight and release its stage after issuing the next one)
//
// Shared-memory tiles are SWIZZLE_128B (the tensor maps are encoded with CU_TENSOR_MAP_SWIZZLE_128B, so the bytes
// land exactly where the wgmma descriptors of common.cuh's make_smem_desc expect them).
//   K-major problems : A = 128 rows x 128 B (one row per output pixel, 64 contraction elements), 4 MMAs (K=16) per stage
//   MN-major problems: A = 2 blocks x KROWS rows x 128 B, B = KROWS rows x 128 B (row = one contraction index = one
//                      pixel/frame, 64 channels); KROWS/16 MMAs per stage.  Rows a box does not write stay zero
//                      (the stage buffers are zero-initialised once), so partial frames contribute nothing.
//
// A Problem P supplies: BN, A_MN, B_MN, STAGES, KROWS (MN-major only), ZERO_INIT, Params (holds the CUtensorMaps),
//   num_kblocks(p,tm,ty), issue(p,tm,ty,kb,sA,sB,bar), init_smem(p,tm,ty,stage_base,tid) [ZERO_INIT only, once per stage],
//   epilogue16(p,tm,ty,row,c0,v), TILE_ROWB.
//   TILE_ROWB: 0, or (bf16 mode) the row pitch in bytes of an fp32 image of the whole 128 x BN output tile that the kernel stages
//   in the stage ring once the last k-block has retired; epilogue_tile(p,tm,ty,t,image,pre) then copies it out in whole, coalesced
//   output rows with all 256 consumer threads t, and prefetch_tile(p,tm,ty,t,pre) requests its global operands instead of prefetch16.
#pragma once
#include <cuda.h>
#include "common.cuh"
#include "kernels.h"

namespace srl {

SRL_DEVINL void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
SRL_DEVINL void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
// 1-D bulk copy (no tensor map) of `bytes` contiguous bytes global -> shared; source, destination and size 16-byte aligned
SRL_DEVINL void bulk_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
SRL_DEVINL void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
               ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
SRL_DEVINL void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
               ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
SRL_DEVINL void tma_load_5d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3, int c4) {
  asm volatile("cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
               ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
               : "memory");
}

constexpr int IGT_THREADS = 288;

// SPLIT = 1: fp32-accurate operand mode (see igemm_res.cuh): a stage holds [A hi][B hi][A lo][B lo]; the problem supplies
// issue_split(p, tm, ty, kb, stage_base, half_bytes, bar) (one expect_tx + the loads of all four tiles) and
// epilogue16<SPLIT>.  Problems that never run split (the LSTM GEMMs) only need the SPLIT = 0 interface.
template <class P, int SPLIT = 0>
struct TmaCfg {
  static constexpr int KROWS = P::A_MN ? P::KROWS : 64;
  static constexpr int A_BYTES = P::A_MN ? 2 * KROWS * 128 : 128 * 128;
  static constexpr int B_BLOCKS = (P::BN + 63) / 64;
  static constexpr int B_BYTES = P::B_MN ? B_BLOCKS * KROWS * 128 : P::BN * 128;
  static constexpr int HALF_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGE_BYTES = HALF_BYTES * (1 + SPLIT);
  static constexpr int NB = P::BN / 2;                    // columns per consumer warpgroup
  static constexpr int STAGES = fit_stages(P::STAGES, 2 * WG_IMG_BYTES + 1024 + 256, STAGE_BYTES);
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 2 * WG_IMG_BYTES + 1024 + 256;
  static_assert(SMEM_BYTES <= 232448, "shared memory budget (227 KB)");
  static_assert(NB == 32 || NB == 64 || NB == 128, "MMA N per warpgroup");
  static constexpr int MMAS = P::A_MN ? KROWS / 16 : 4;
  // the output tile leaves through an fp32 image in the stage ring (bf16 mode of the problems that define one), or row by row
  static constexpr bool TILE_EPI = P::TILE_ROWB > 0 && !SPLIT;
  static_assert(!TILE_EPI || (P::TILE_ROWB >= 4 * P::BN && P::TILE_ROWB % 16 == 0 && 128 * P::TILE_ROWB <= STAGES * STAGE_BYTES),
                "the tile image holds 128 rows of BN fp32 in 16-byte aligned rows inside the stage ring");
  static_assert(A_BYTES % 1024 == 0 && B_BYTES % 1024 == 0, "operand tiles must keep 1024 B alignment (SWIZZLE_128B atoms)");
  static_assert(P::A_MN == P::B_MN, "mixed majors are not used");
  static_assert(KROWS % 16 == 0, "contraction rows per stage must be a multiple of MMA K = 16");
};

// fp32 image of a warpgroup's 128 x N accumulator (wgmma fragment layout) in shared memory: row r at img + r * ROWB bytes, column c
// at byte 4c.  With ROWB = 8N + 32 (the tile's BN = 2N = 64 or 256) a half-warp's float2 stores (4 rows x 8 words) hit 32 banks.
template <int N, int ROWB>
SRL_DEVINL void wg_acc_stage_f32(const float (&d)[2][N / 2], uint8_t* img, int wt) {
  const int w = wt >> 5, l = wt & 31;
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int i = 0; i < N / 2; i += 2) {
      const int row = 64 * h + 16 * w + (l >> 2) + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + 2 * (l & 3);
      *reinterpret_cast<float2*>(img + row * ROWB + col * 4) = make_float2(d[h][i], d[h][i + 1]);
    }
}

template <class P, int SPLIT>
SRL_DEVINL void igt_epilogue(const typename P::Params& p, int tm, int ty, int row, int c0, float (&v)[16]) {
  if constexpr (SPLIT) P::template epilogue16<1>(p, tm, ty, row, c0, v); else P::epilogue16(p, tm, ty, row, c0, v);
}
template <class P, int SPLIT>
SRL_DEVINL void igt_epilogue(const typename P::Params& p, int tm, int ty, int row, int c0, float (&v)[16], const uint4 (&pre)[2]) {
  if constexpr (SPLIT) P::template epilogue16<1>(p, tm, ty, row, c0, v, pre); else P::epilogue16(p, tm, ty, row, c0, v, pre);
}

template <class P, int SPLIT = 0>
__global__ void __launch_bounds__(IGT_THREADS) igemm_tma_kernel(const __grid_constant__ typename P::Params p) {
  using C = TmaCfg<P, SPLIT>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* img = reinterpret_cast<float*>(smem + C::STAGES * C::STAGE_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::STAGES * C::STAGE_BYTES + 2 * WG_IMG_BYTES);
  uint64_t* full = bars;
  uint64_t* empty = bars + C::STAGES;

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int tm = blockIdx.x, ty = blockIdx.y;
  const int nkb = P::num_kblocks(p, tm, ty);

  if constexpr (P::ZERO_INIT) {
    if (P::zero_cta(ty)) {
      uint4* z = reinterpret_cast<uint4*>(smem);
      for (int i = tid; i < C::STAGES * C::STAGE_BYTES / 16; i += IGT_THREADS) z[i] = make_uint4(0, 0, 0, 0);
    }
    __syncthreads();
    for (int s = 0; s < C::STAGES; ++s) P::init_smem(p, tm, ty, smem + s * C::STAGE_BYTES, tid);
    fence_proxy_async_smem();
  }
  if (warp == 8 && (tid & 31) == 0) {
    for (int s = 0; s < C::STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    mbar_fence_init();
    P::prefetch(p);
  }
  __syncthreads();
  pdl_wait(P::KID);                   // prologue above overlaps the previous kernel's tail
  if (tid == 256) pdl_launch();

  if (warp == 8) {
    const uint32_t leader = elect_one_sync();
    for (int kb = 0; kb < nkb; ++kb) {
      const int s = kb % C::STAGES;
      mbar_wait(&empty[s], ((kb / C::STAGES) & 1) ^ 1);
      if (leader) {
        uint8_t* sA = smem + s * C::STAGE_BYTES;
        if constexpr (SPLIT) P::issue_split(p, tm, ty, kb, sA, C::A_BYTES, C::HALF_BYTES, &full[s]);
        else P::issue(p, tm, ty, kb, sA, sA + C::A_BYTES, &full[s]);
      }
      __syncwarp();
    }
  } else {
    const int g = warp >> 2, wt = tid & 127;
    constexpr int NB = C::NB;
    // global operands of the epilogue (ReLU mask) are requested before the mainloop: their latency overlaps the MMAs
    // (tile epilogue: the same NB / 8 pieces of 16 bytes per thread hold the tile's bf16 mask, 128 rows x BN, over all 256 threads)
    uint4 pre[P::PREFETCH ? NB / 16 : 1][2];
    if constexpr (C::TILE_EPI) {
      if constexpr (P::PREFETCH) P::prefetch_tile(p, tm, ty, tid, pre);
    } else if constexpr (P::PREFETCH) {
#pragma unroll
      for (int c = 0; c < NB / 16; ++c) P::prefetch16(p, tm, ty, wt, g * NB + c * 16, pre[c]);
    }
    float acc[2][NB / 2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < NB / 2; ++i) acc[h][i] = 0.f;
    constexpr uint32_t ASTEP = P::A_MN ? 2048 / 16 : 32 / 16, BSTEP = P::B_MN ? 2048 / 16 : 32 / 16;     // descriptor address units per K = 16
    constexpr uint32_t A_HI = (P::A_MN ? C::KROWS * 128 : 64 * 128) / 16;         // rows 64..127 of the tile
    // this warpgroup's columns of B.  MN-major: 64-column blocks KROWS rows apart, then 2 B per column inside the swizzled row
    const uint32_t b_off = P::B_MN ? (g * NB / 64) * C::KROWS * 128 + (g * NB % 64) * 2 : g * NB * 128;
    for (int kb = 0; kb < nkb; ++kb) {
      const int s = kb % C::STAGES;
      mbar_wait(&full[s], (kb / C::STAGES) & 1);
      const uint32_t a0 = smem_u32(smem + s * C::STAGE_BYTES);
      const uint64_t ad0 = P::A_MN ? make_smem_desc(a0, C::KROWS * 128, 1024) : make_smem_desc(a0, 16, 1024);
      const uint64_t bd0 = P::B_MN ? make_smem_desc(a0 + C::A_BYTES + b_off, C::KROWS * 128, 1024) : make_smem_desc(a0 + C::A_BYTES + b_off, 16, 1024);
      wg_fence();
#pragma unroll
      for (int k = 0; k < C::MMAS; ++k) {
        const uint64_t ad = ad0 + (uint64_t)(k * ASTEP), bd = bd0 + (uint64_t)(k * BSTEP);
        wg_mma128<NB, P::A_MN ? 1 : 0, P::B_MN ? 1 : 0>(acc, ad, A_HI, bd, (kb | k) != 0);
        if constexpr (SPLIT) {        // hi * lo, lo * hi (the low tiles sit HALF_BYTES further into the stage)
          wg_mma128<NB, P::A_MN ? 1 : 0, P::B_MN ? 1 : 0>(acc, ad, A_HI, bd + (uint64_t)(C::HALF_BYTES / 16), 1);
          wg_mma128<NB, P::A_MN ? 1 : 0, P::B_MN ? 1 : 0>(acc, ad + (uint64_t)(C::HALF_BYTES / 16), A_HI, bd, 1);
        }
      }
      wg_commit();
      if constexpr (C::STAGES > 1) {
        // k-block kb stays in flight while kb + 1 is awaited and issued; kb - 1's stage is released as soon as it retired
        wg_wait_prev();
        __syncwarp();
        if (kb > 0 && (tid & 31) == 0) mbar_arrive(&empty[(kb - 1) % C::STAGES]);
      } else {
        wg_wait_all();
        __syncwarp();
        if ((tid & 31) == 0) mbar_arrive(&empty[s]);
      }
    }
    wg_wait_all();
    wg_fence_regs(acc[0]); wg_fence_regs(acc[1]);
    if constexpr (C::TILE_EPI) {
      // one tile per CTA: once both warpgroups' last wgmma retired, every TMA write has landed and no MMA reads the ring (nor its
      // zero-filled B rows) any more, so the image overwrites it
      named_bar(1, 256);
      wg_acc_stage_f32<NB, P::TILE_ROWB>(acc, smem + g * NB * 4, wt);
      named_bar(1, 256);
      P::epilogue_tile(p, tm, ty, tid, smem, pre);
    } else {
      float* my_img = img + g * (WG_IMG_BYTES / 4);
#pragma unroll
      for (int c = 0; c < NB / 16; ++c) {
        float v[16];
        wg_acc_row16<NB>(acc, c, my_img, wt, 2 + g, v);
        if constexpr (P::PREFETCH) igt_epilogue<P, SPLIT>(p, tm, ty, wt, g * NB + c * 16, v, pre[c]);
        else igt_epilogue<P, SPLIT>(p, tm, ty, wt, g * NB + c * 16, v);
      }
    }
  }
}

template <class P, int SPLIT = 0>
cudaError_t igemm_tma_launch(const typename P::Params& p, dim3 grid, cudaStream_t stream) {
  using C = TmaCfg<P, SPLIT>;
  if (grid.x == 0 || grid.y == 0) return cudaSuccess;
  static PerDeviceOnce once;      // set once per device (outside any stream capture: the first step always runs eagerly)
  { cudaError_t e = ensure_max_dynamic_smem(once, igemm_tma_kernel<P, SPLIT>, C::SMEM_BYTES); if (e != cudaSuccess) return e; }
  return launch_chain(igemm_tma_kernel<P, SPLIT>, grid, dim3(IGT_THREADS), C::SMEM_BYTES, stream, p);
}

}  // namespace srl
