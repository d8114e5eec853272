// Fused front of the encoder: u8 frame -> space-to-depth -> conv1 (8x8 s4, 4->32, ReLU) -> conv2 (4x4 s2, 32->64, ReLU), one
// persistent kernel, one frame at a time per CTA, everything between the u8 frame and conv2's output kept on the SM
// (reference: scalerl/algorithms/utils/atari_model.py:93-98: x.float()/255, relu(conv1), relu(conv2)).
//
// Replaces three dependent launches of the step's chain (obs_s2d_kernel, res_fwd_kernel<RConv1Fwd>, res_fwd_kernel<RConv2Fwd>)
// and the HBM round trips between them; what the BACKWARD pass needs is still written out once: xs (the space-to-depth frame:
// conv1 wgrad's operand) and a1 (conv2's wgrad operand and dgrad mask), plus a2, the input of conv3.
//
//   warp 16     producer: ONE cp.async.bulk (1-D TMA) per frame, 28,224 contiguous bytes of u8 -> shared memory, double-buffered
//               (frame f+1 lands while frame f is being computed)
//   warps 8-15  converters: u8 -> bf16 space-to-depth operand tile of conv1 (128 output positions + 22 halo rows of the 21x21
//               grid, 64 channels (c,dy,dx), SWIZZLE_128B) written with generic stores + fence.proxy.async; three tile stages;
//               the same values go to global `xs`
//   warps 0-3   conv1 warpgroup: wgmma, 4 position tiles x (4 taps x 4 K-steps), N = 32, accumulator in registers; epilogue
//               registers -> (x/255 + b1, ReLU) -> bf16 -> shared a1 planes + global a1
//   warps 4-7   conv2 warpgroup: wgmma, 8 taps x 4 K-steps, N = 64, reading conv1's output from SHARED memory (the two row-parity
//               planes of the layout in res_problems.cuh, so a stride-2 tap is a row shift); epilogue (+ b2, ReLU) -> global a2.
//               Two warpgroups so that conv2(f) does not queue behind conv1(f+1).
// The conv weights are converted from the fp32 master parameters inside the prologue (80 KB of bf16 per CTA, from L2), so the
// kernel does not depend on pack_weights_kernel -- that kernel (needed by conv3 / fc) runs beside it.
// Opt-in (SRL_FUSED_FWD=1): bit-identical to the three kernels.
#pragma once
#include "igemm_tma.cuh"
#include "encoder_problems.cuh"

namespace srl {

constexpr int FF_THREADS = 544;          // warps 0-3 conv1 warpgroup, 4-7 conv2 warpgroup, 8-15 converters, 16 producer
constexpr int FF_CONV_WARPS = 8;
constexpr int FF_W1_BYTES = 4 * 32 * 128;          // 4 taps x [32 co][64 k]
constexpr int FF_W2_BYTES = 8 * 64 * 128;          // 8 taps x [64 co][64 k]
constexpr int FF_U8_BYTES = 28 * 1024;             // one frame (28,224 B) rounded up
constexpr int FF_X_BYTES = 19 * 1024;              // 150 rows x 128 B rounded up
constexpr int FF_A1_PLANE = 13 * 1024;             // 100 rows x 128 B rounded up (13,312)
constexpr int FF_A1_BYTES = 31 * 1024;             // plane 1 starts at 13,312; conv2 reads 139 rows of it -> 31,104 B
constexpr int FF_OFF_W2 = FF_W1_BYTES;
constexpr int FF_OFF_U8 = FF_OFF_W2 + FF_W2_BYTES;
constexpr int FF_OFF_X = FF_OFF_U8 + 2 * FF_U8_BYTES;
constexpr int FF_XS = 2;                     // X-tile stages: the converters fill one while conv1 multiplies the other
constexpr int FF_OFF_A1 = FF_OFF_X + FF_XS * FF_X_BYTES;
constexpr int FF_OFF_IMG = FF_OFF_A1 + FF_A1_BYTES;  // two single-buffer accumulator row hand-offs (conv1, conv2)
constexpr int FF_OFF_BAR = FF_OFF_IMG + WG_IMG_BYTES;
constexpr int FF_SMEM_BYTES = FF_OFF_BAR + 1024 + 1024;      // barriers + the two bias vectors
static_assert(FF_SMEM_BYTES <= 232448, "shared memory budget");
static_assert(FF_OFF_U8 % 1024 == 0 && FF_OFF_X % 1024 == 0 && FF_OFF_A1 % 1024 == 0, "swizzle atoms need 1024-byte aligned tiles");

struct EncFusedParams {
  const uint8_t* obs;        // [frames][4][84][84]
  const float* w1;           // conv1.weight [32][4][8][8]   (fp32 master)
  const float* b1;
  const float* w2;           // conv2.weight [64][32][4][4]
  const float* b2;
  bf16* xs;                  // [frames*441][64]
  bf16* a1;                  // [2 planes][NFS*100][64]
  bf16* a2;                  // [frames*81][64]
  int frames;
  int NFS;                   // frame capacity of the a1 planes (plane stride)
};

// mbarrier wait for the roles that are not on the critical issue path: back off between polls so the spinning warps do not
// take issue slots from the converter / epilogue warps sharing their schedulers
SRL_DEVINL void mbar_wait_relaxed(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    __nanosleep(32);
    if (++spins > SRL_SPIN_LIMIT) __trap();
  }
}

__global__ void __launch_bounds__(FF_THREADS, 1) enc_fused_fwd_kernel(const EncFusedParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sW1 = smem;
  uint8_t* sW2 = smem + FF_OFF_W2;
  uint8_t* sU8 = smem + FF_OFF_U8;
  uint8_t* sX = smem + FF_OFF_X;
  uint8_t* sA1 = smem + FF_OFF_A1;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + FF_OFF_BAR);
  uint64_t* u8_full = bars;            // [2] producer tx
  uint64_t* u8_empty = bars + 2;       // [2] 8 converter warps
  uint64_t* x_full = bars + 4;         // [FF_XS] 8 converter warps
  uint64_t* x_empty = bars + 7;        // [FF_XS] 4 conv1 warps (after their wgmma wait)
  uint64_t* a1_full = bars + 18;       // 4 conv1 warps
  uint64_t* a1_empty = bars + 19;      // 4 conv2 warps (after their wgmma wait)
  float* img = reinterpret_cast<float*>(smem + FF_OFF_IMG);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nmine = p.frames > (int)blockIdx.x ? (p.frames - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;

  float* s_b1 = reinterpret_cast<float*>(smem + FF_OFF_BAR + 256);      // [32]
  float* s_b2 = s_b1 + 32;                                               // [64]
  if (tid < 32) s_b1[tid] = __ldg(p.b1 + tid);
  else if (tid < 96) s_b2[tid - 32] = __ldg(p.b2 + tid - 32);
  if (warp == 16 && lane == 0) {
    for (int i = 0; i < 2; ++i) { mbar_init(&u8_full[i], 1); mbar_init(&u8_empty[i], FF_CONV_WARPS); }
    for (int i = 0; i < FF_XS; ++i) { mbar_init(&x_full[i], FF_CONV_WARPS); mbar_init(&x_empty[i], 4); }
    mbar_init(a1_full, 4); mbar_init(a1_empty, 4);
    mbar_fence_init();
  }
  // the halo rows of the a1 planes that no epilogue ever writes (rows 100.. of plane 1) feed only discarded MMA rows: zero them once
  for (int i = tid; i < (FF_A1_BYTES - 2 * FF_A1_PLANE) / 16; i += FF_THREADS)
    reinterpret_cast<uint4*>(sA1 + 2 * FF_A1_PLANE)[i] = make_uint4(0, 0, 0, 0);
  pdl_wait(54);                          // the parameters below were written by the previous step's optimizer kernel
  pdl_launch();
  // ---- conv weights: fp32 master -> bf16 K-major SWIZZLE_128B operand tiles (what pack_weights_kernel + TMA would deliver).
  //      Read in memory order as float4 (coalesced), several loads in flight per thread, scattered into the tiles.
  //  w1 tile j (= tap (kh2,kw2)): row co (32), k = c*16 + dy*4 + dx  <- W1[co][c][4kh2+dy][4kw2+dx]; a float4 = the 4 dx of one (co,c,kh,kw2)
  {
    constexpr int NQ = 2048, U = 4;                      // 2048 float4 / 544 threads -> <= 4 each
    float4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) { const int q = tid + u * FF_THREADS; if (q < NQ) v[u] = __ldg(reinterpret_cast<const float4*>(p.w1) + q); }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int q = tid + u * FF_THREADS;
      if (q < NQ) {
        const int co = q >> 6, c = (q >> 4) & 3, kh = (q >> 1) & 7, j = (kh >> 2) * 2 + (q & 1), g = c * 4 + (kh & 3);
        *reinterpret_cast<uint2*>(sW1 + j * 4096 + swz128(co, g >> 1) + (g & 1) * 8) = make_uint2(pack_bf16x2(v[u].x, v[u].y), pack_bf16x2(v[u].z, v[u].w));
      }
    }
  }
  //  w2 tile j (= (kh, kww)): row co (64), k = kwl*32 + c (kw = 2kww + kwl)  <- W2[co][c][kh][kw]; a float4 = the 4 kw of one (co,c,kh)
  {
    constexpr int NQ = 8192, U = 8;                      // two rounds of 8 loads in flight per thread
#pragma unroll 1
    for (int base = 0; base < NQ; base += U * FF_THREADS) {
      float4 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) { const int q = base + tid + u * FF_THREADS; if (q < NQ) v[u] = __ldg(reinterpret_cast<const float4*>(p.w2) + q); }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int q = base + tid + u * FF_THREADS;
        if (q < NQ) {
          const int co = q >> 7, c = (q >> 2) & 31, kh = q & 3;
          const float w[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
          for (int kw = 0; kw < 4; ++kw) {
            const int j = kh * 2 + (kw >> 1), k = (kw & 1) * 32 + c;
            *reinterpret_cast<__nv_bfloat16*>(sW2 + j * 8192 + swz128(co, k >> 3) + (k & 7) * 2) = __float2bfloat16_rn(w[kw]);
          }
        }
      }
    }
  }
  fence_proxy_async_smem();
  __syncthreads();

  if (warp == 16) {
    // ------------------------------------------------------------------------------------------------ producer
    if (lane == 0) {
      for (int it = 0; it < nmine; ++it) {
        const int f = blockIdx.x + it * gridDim.x, ub = it & 1;
        mbar_wait(&u8_empty[ub], ((it >> 1) & 1) ^ 1);
        mbar_arrive_expect_tx(&u8_full[ub], 28224);
        bulk_load_1d(sU8 + ub * FF_U8_BYTES, p.obs + (size_t)f * 28224, 28224, &u8_full[ub]);
      }
    }
  } else if (warp >= 8) {
    // ------------------------------------------------------------------------------------------------ converters (256 threads)
    // thread = (16-byte chunk gp = (c, dy pair), row slot rb); rows rb, rb + 32, ... of the 150-row tile (S2dWindow)
    const int t = tid - 256, gp = t & 7, rb = t >> 3;
    const int src_g = (gp >> 1) * 7056 + (gp & 1) * 168;           // (c, dy0 = 2 (gp & 1)) offset inside the u8 frame
    for (int it = 0; it < nmine; ++it) {
      const int f = blockIdx.x + it * gridDim.x, ub = it & 1;
      mbar_wait_relaxed(&u8_full[ub], (it >> 1) & 1);
      const uint8_t* u8 = sU8 + ub * FF_U8_BYTES + src_g;
      bf16* xs_f = p.xs + (size_t)f * 441 * 64 + gp * 8;
      for (int j = 0; j < 4; ++j) {
        const int n = 4 * it + j, s = n % FF_XS;
        // all ten source words of the thread's five rows first (the compiler cannot hoist shared loads above the shared stores below)
        S2dWindow<32> win;
        win.load(u8, rb, j * 128, 441);
        mbar_wait(&x_empty[s], ((n / FF_XS) & 1) ^ 1);    // on the critical cycle (MMA commit -> refill): tight poll
        win.store(sX + s * FF_X_BYTES, gp, rb, [&](int row, uint4 v) {
          if (row < 128) *reinterpret_cast<uint4*>(xs_f + (size_t)(j * 128 + row) * 64) = v;     // conv1 wgrad's operand
        });
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(&x_full[s]);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&u8_empty[ub]);
    }
  } else if (warp < 4) {
    // ------------------------------------------------------------------------------------------------ conv1 warpgroup (warps 0-3)
    // Descriptors are base + constant (the 14-bit address field cannot carry).
    const uint64_t w1d = make_smem_desc(smem_u32(sW1), 16, 1024);
    for (int it = 0; it < nmine; ++it) {
      const int f = blockIdx.x + it * gridDim.x;
      for (int j = 0; j < 4; ++j) {
        const int n = 4 * it + j, s = n % FF_XS;
        mbar_wait(&x_full[s], (n / FF_XS) & 1);
        const uint64_t xd = make_smem_desc(smem_u32(sX + s * FF_X_BYTES), 16, 1024);
        float acc[2][16];
        wg_fence();
#pragma unroll
        for (int tap = 0; tap < 4; ++tap)
#pragma unroll
          for (int k = 0; k < 4; ++k)
            wg_mma128<32, 0, 0>(acc, xd + (uint64_t)(((tap >> 1) * 21 + (tap & 1)) * 8 + k * 2), 64 * 128 / 16, w1d + (uint64_t)(tap * 256 + k * 2),
                                (tap | k) != 0);
        wg_commit();
        wg_wait_all();
        wg_fence_regs(acc[0]); wg_fence_regs(acc[1]);
        __syncwarp();
        if (lane == 0) mbar_arrive(&x_empty[s]);
        float r0[16], r1[16];
        wg_acc_row16<32, true>(acc, 0, img, tid, 2, r0);
        wg_acc_row16<32, true>(acc, 1, img, tid, 2, r1);
        if (j == 0) mbar_wait_relaxed(a1_empty, (it & 1) ^ 1);   // conv2 of the previous frame has finished reading the planes
        const int Q = j * 128 + tid, oh = Q / 21, ow = Q - oh * 21;
        if (Q < 441 && oh < 20 && ow < 20) {
          float v[32];
#pragma unroll
          for (int c = 0; c < 16; ++c) {
            v[c] = fmaxf(fmaf(r0[c], 1.0f / 255.0f, s_b1[c]), 0.f);
            v[16 + c] = fmaxf(fmaf(r1[c], 1.0f / 255.0f, s_b1[16 + c]), 0.f);
          }
          uint4 q[4];
#pragma unroll
          for (int k = 0; k < 4; ++k)
            q[k] = make_uint4(pack_bf16x2(v[8 * k], v[8 * k + 1]), pack_bf16x2(v[8 * k + 2], v[8 * k + 3]), pack_bf16x2(v[8 * k + 4], v[8 * k + 5]),
                              pack_bf16x2(v[8 * k + 6], v[8 * k + 7]));
          const int prow = (oh >> 1) * 10 + (ow >> 1), half = ow & 1;      // plane oh & 1, channel (ow & 1) * 32 + c
          uint8_t* pl = sA1 + (oh & 1) * FF_A1_PLANE;
          uint4* gdst = reinterpret_cast<uint4*>(p.a1 + ((size_t)(oh & 1) * p.NFS * 100 + (size_t)f * 100 + prow) * 64 + half * 32);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            *reinterpret_cast<uint4*>(pl + swz128(prow, half * 4 + k)) = q[k];
            gdst[k] = q[k];
          }
        }
      }
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) mbar_arrive(a1_full);
    }
  } else {
    // ------------------------------------------------------------------------------------------------ conv2 warpgroup (warps 4-7)
    const int row = tid - 128;
    const int oh2 = row / 10, ow2 = row - oh2 * 10;
    const bool ok = row < 100 && oh2 < 9 && ow2 < 9;
    const uint64_t w2d = make_smem_desc(smem_u32(sW2), 16, 1024), a1d = make_smem_desc(smem_u32(sA1), 16, 1024);
    for (int it = 0; it < nmine; ++it) {
      const int f = blockIdx.x + it * gridDim.x;
      mbar_wait_relaxed(a1_full, it & 1);
      float acc[2][32];
      wg_fence();
#pragma unroll
      for (int tap = 0; tap < 8; ++tap)         // tap = (kh, kww): plane kh & 1, shift (kh >> 1) * 10 + kww
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wg_mma128<64, 0, 0>(acc, a1d + (uint64_t)((((tap >> 1) & 1) * FF_A1_PLANE + ((tap >> 2) * 10 + (tap & 1)) * 128) / 16 + k * 2), 64 * 128 / 16,
                              w2d + (uint64_t)(tap * 512 + k * 2), (tap | k) != 0);
      wg_commit();
      wg_wait_all();
      wg_fence_regs(acc[0]); wg_fence_regs(acc[1]);
      __syncwarp();
      if (lane == 0) mbar_arrive(a1_empty);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float v[16];
        wg_acc_row16<64, true>(acc, q, img + WG_IMG_BYTES / 8, row, 3, v);
        if (ok) {
#pragma unroll
          for (int c = 0; c < 16; ++c) v[c] = fmaxf(v[c] + s_b2[q * 16 + c], 0.f);
          store_bf16x16(p.a2 + ((size_t)f * 81 + oh2 * 9 + ow2) * 64 + q * 16, v);
        }
      }
    }
  }
}

inline cudaError_t enc_fused_fwd_launch(const EncFusedParams& p, int max_ctas, cudaStream_t stream) {
  if (p.frames <= 0) return cudaSuccess;
  static PerDeviceOnce once;
  { cudaError_t e = ensure_max_dynamic_smem(once, enc_fused_fwd_kernel, FF_SMEM_BYTES); if (e != cudaSuccess) return e; }
  // balanced grid: 672 frames on 132 SMs would be 12 CTAs x 6 + 120 x 5 frames, exactly as slow as 112 x 6; the SMs left free run
  // the weight re-pack kernel (needed only by conv3 / fc) undisturbed
  const int per = (p.frames + max_ctas - 1) / max_ctas;
  const int grid = (p.frames + per - 1) / per;
  return launch_chain(enc_fused_fwd_kernel, dim3(grid), dim3(FF_THREADS), FF_SMEM_BYTES, stream, p);
}

}  // namespace srl
