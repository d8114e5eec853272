// "Resident window" convolution kernels on Hopper warpgroup MMA (wgmma, sm_90a).
//
// Every activation tensor is stored as rows of 64 bf16 channels (128 B) on the spatial grid of the conv INPUT it
// belongs to (frames concatenated: row = n * GRID + y * PITCH + x).  A filter tap is then a CONSTANT ROW SHIFT of the
// whole batch, so one shared-memory window of the input (loaded once with one 2-D TMA box) serves every tap: the wgmma
// operand descriptor of tap j simply starts  shift_j * 128 B  further into the window.  (wgmma applies SWIZZLE_128B to
// absolute shared-memory address bits, so a descriptor may start at any 128-byte row -- verified by
// srl_test_shifted_operand, tests/test_gpu_parity.py::test_shifted_operand_descriptors.)  Compared with one im2col box per tap this divides the
// L2->SM operand traffic by the number of taps (4 / 8 / 9) and keeps the weights stationary in shared memory.
// Output positions are enumerated on the same grid; positions outside the valid output range are computed and
// discarded (conv1 9 %, conv2 19 %, conv3 40 % of the MMA rows -- the MMA is not the limiter of these layers).
//
//   res_fwd_kernel<P>   K-major, persistent: forward convs and dgrads (dgrad = negative shifts over dY stored on the
//                       grid of the conv input with zeros outside the valid outputs, which doubles as padding).
//                       warps 8-11 = producer warpgroup: warp 8 issues the TMA loads (weights once, then one window per
//                       128-position tile, S-deep ring), warps 9-11 only give their registers back;
//                       warps 0-7 = two consumer warpgroups taking alternate tiles: each issues NT taps x 4 K-steps of
//                       wgmma into its register accumulator and runs that tile's epilogue while the other warpgroup
//                       multiplies the next tile.
//   res_wgrad_kernel<P> MN-major: dW[tap] = sum over positions X[pos + shift_tap]^T dY[pos].  One CTA owns a contiguous
//                       range of positions, streams (window, dY) chunks of 128 positions through a ring and keeps ALL
//                       taps' accumulators in registers: each 64-row tap block is one m64 accumulator, the blocks are
//                       spread over two or three consumer warpgroups.  A producer warpgroup issues the TMA loads and sums
//                       the staged dY columns (bias gradient) on a small register budget (setmaxnreg); the consumers keep
//                       one chunk's MMAs in flight while they issue the next.
#pragma once
#include "igemm_tma.cuh"
#include "encoder_problems.cuh"

namespace srl {

constexpr int RES_THREADS = 384;      // res_fwd_kernel: two consumer warpgroups + the producer warpgroup
// register budgets (per thread, setmaxnreg) of res_fwd_kernel: one warp of each warpgroup per sub-partition, 40 + 2 x 232 <= 3 x 168
// (the launch allocation, which the budgets only redistribute)
constexpr int RES_PRODUCER_REGS = 40, RES_CONSUMER_REGS = 232;
constexpr int RES_MAX_TAPS = 10;

// ------------------------------------------------------------------------------------------------------------------
// forward / dgrad
//   P: BN, NT (taps), NWIN (input windows per tile: 1, or 2 for conv2's two row-parity planes), WROWS (rows per window,
//      128 + max shift - min shift), SHIFT_MIN, STAGES, Params{ in[NWIN] maps, w map, ... },
//      tap_win(j), tap_shift(j) (relative to SHIFT_MIN, i.e. >= 0), num_tiles(p), epilogue16(p, tile, row, c0, v),
//      TILE_ROWB: 0, or (bf16 mode) the row pitch of a shared-memory bf16 image of the whole output tile that
//      epilogue_tile(p, tile, wt, acc, image, bar, pre) stages and copies out in whole, coalesced output rows
//      (prefetch_tile(p, tile, wt, pre) then requests its global operands instead of prefetch16)
// ------------------------------------------------------------------------------------------------------------------

// bf16 image of a warpgroup's 128 x N accumulator in shared memory: row r at buf + r * ROWB bytes, column c at byte 2c, each value
// f(column, value) rounded as store_bf16x16 rounds it.  With ROWB = 2N + 16 the 8 rows x 4 words of a warp's stores hit 32
// distinct banks.  Brackets the writes with the warpgroup's named barrier: the previous tile's readers are done before, every
// row is complete after.
template <int N, int ROWB, class F>
SRL_DEVINL void wg_acc_stage_bf16(const float (&d)[2][N / 2], uint8_t* buf, int wt, int bar, F f) {
  static_assert(ROWB % 16 == 0 && ROWB >= 2 * N, "16-byte aligned rows that hold N bf16");
  const int w = wt >> 5, l = wt & 31;
  named_bar(bar, 128);
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int i = 0; i < N / 2; i += 2) {
      const int row = 64 * h + 16 * w + (l >> 2) + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + 2 * (l & 3);
      *reinterpret_cast<uint32_t*>(buf + row * ROWB + col * 2) = pack_bf16x2(f(col, d[h][i]), f(col + 1, d[h][i + 1]));
    }
  named_bar(bar, 128);
}
//
// SPLIT = 1 is the fp32-accurate operand mode (srl_config_t.precision = 1): every bf16 operand tensor has a second, "low"
// tensor holding bf16(v - bf16(v)), and each product is issued as hi*hi + hi*lo + lo*hi into the same fp32 accumulator
// (the dropped lo*lo term is ~2^-18 relative; operands carry 16 significant bits, tighter than kind::tf32's 11).  Layouts,
// descriptors and tensor maps are those of the bf16 mode -- the low tensors are simply a second copy of everything -- so
// the mode exercises exactly the same data paths the fast mode uses.  It is for whole-step parity, not speed: 3x (2x where an
// operand is exact: the u8 frames) the MMAs, twice the operand traffic, fewer pipeline stages.
template <class P, int SPLIT>
struct ResFwdCfg {
  static constexpr int ALO = (SPLIT && P::A_LO) ? 1 : 0;          // the A operand has a low tensor (everything but the u8 frames)
  static constexpr int WIN_BYTES = ((P::WROWS * 128 + 1023) / 1024) * 1024;
  static constexpr int IN_HI_BYTES = P::NWIN * WIN_BYTES;
  static constexpr int IN_BYTES = IN_HI_BYTES * (1 + ALO);
  // U8: the producer warpgroup converts each window from u8 frame rows staged beside it (U8_BYTES per stage, RConv1Fwd::FromFrames); the
  // converters' registers come from the consumers
  static constexpr bool U8 = P::U8_BYTES > 0;
  static constexpr int U8_BYTES = P::U8_BYTES;
  static_assert(!U8 || (!SPLIT && P::NWIN == 1), "u8-fed windows: bf16 mode, one window");
  static constexpr int PRODUCER_REGS = U8 ? 72 : RES_PRODUCER_REGS, CONSUMER_REGS = U8 ? 216 : RES_CONSUMER_REGS;
  // setmaxnreg moves registers inside the CTA's launch allocation (168 per thread): the consumers can only claim what the producer gave back
  static_assert(PRODUCER_REGS + 2 * CONSUMER_REGS <= 3 * (65536 / RES_THREADS & ~7), "register budgets within the launch allocation");
  static constexpr int W_HI_BYTES = P::NT * P::BN * 128;
  static constexpr int W_BYTES = W_HI_BYTES * (1 + SPLIT);
  // the output tile leaves through a bf16 image in shared memory (bf16 mode of the problems that define one), or row by row
  static constexpr bool TILE_EPI = P::TILE_ROWB > 0 && !SPLIT;
  static constexpr int TILE_IMG_BYTES = 128 * P::TILE_ROWB > WG_IMG_BYTES ? 128 * P::TILE_ROWB : WG_IMG_BYTES;
  // row hand-off buffers of the two consumer warpgroups: single-buffered where one input stage would not fit beside double ones
  static constexpr bool IMG1 = !TILE_EPI && W_BYTES + IN_BYTES + 2 * WG_IMG_BYTES + 1024 + 256 > 232448;
  static constexpr int IMG_BYTES = TILE_EPI ? TILE_IMG_BYTES : IMG1 ? WG_IMG_BYTES / 2 : WG_IMG_BYTES;
  // the two consumer warpgroups take alternate tiles: with an even depth every stage (and every phase of its barrier) belongs to one
  // warpgroup, so a warpgroup never waits for phase k of a stage whose phase k-1 (the other warpgroup's tile) may still be filling
  static constexpr int FIT = fit_stages(SPLIT ? P::SPLIT_STAGES : P::STAGES, W_BYTES + 2 * IMG_BYTES + 1024 + 256, IN_BYTES + U8_BYTES);
  static constexpr int STAGES = FIT > 1 ? FIT & ~1 : 1;
  static constexpr int SMEM_BYTES = W_BYTES + STAGES * (IN_BYTES + U8_BYTES) + 2 * IMG_BYTES + 1024 + 256;
  static_assert(SMEM_BYTES <= 232448, "shared memory budget (227 KB)");
  static_assert(W_BYTES % 1024 == 0, "weight block alignment");
  static_assert(P::BN == 32 || P::BN == 64 || P::BN == 128, "MMA N");
};

// Converter warps 9-11 of a u8-fed res_fwd_kernel (C::U8): tile it's window, from the source rows staged in u8 stage it % STAGES,
// into input stage it % STAGES, and its rows 0..127 that lie inside the frames to xs (a warp's store is 4 whole, consecutive xs rows)
template <class P, class C>
SRL_DEVINL void res_u8_converters(const typename P::Params& p, uint8_t* sIn, uint8_t* sU8, uint64_t* in_full, uint64_t* in_empty,
                                  uint64_t* u8_full, uint64_t* u8_empty, int tid) {
  constexpr int STAGES = C::STAGES;
  static_assert(P::CONV_SLOTS == 12, "warps 9-11");
  const int ct = tid - 288, gp = ct & 7, rb = ct >> 3;
  const int ntiles = P::num_tiles(p), qend = p.NF * 441;
  const int plane = (gp >> 1) * P::U8_PLANE + (gp & 1) * 168;       // chunk gp's channel plane c and source row dy = 2 (gp & 1)
  int it = 0;
  for (int t = blockIdx.x; t < ntiles; t += gridDim.x, ++it) {
    const int s = it % STAGES, q0 = t * 128, r0 = q0 / 21;
    const uint32_t ph = (it / STAGES) & 1;
    S2dWindow<P::CONV_SLOTS> w;
    mbar_wait(&u8_full[s], ph);
    w.load(sU8 + s * C::U8_BYTES + plane, rb, q0 - r0 * 21, qend - r0 * 21);
    mbar_wait(&in_empty[s], ph ^ 1);
    bf16* xs = p.xs + (size_t)q0 * 64 + gp * 8;
    w.store(sIn + s * C::IN_BYTES, gp, rb, [&](int row, uint4 v) { if (row < 128) *reinterpret_cast<uint4*>(xs + (size_t)row * 64) = v; });
    fence_proxy_async_smem();                        // the window's generic stores -> the MMAs' reads
    __syncwarp();
    if ((tid & 31) == 0) { mbar_arrive(&u8_empty[s]); mbar_arrive(&in_full[s]); }    // the stores consumed every staged word read
  }
}

template <class P, int SPLIT>
__global__ void __launch_bounds__(RES_THREADS, 1) res_fwd_kernel(const __grid_constant__ typename P::Params p) {
  using C = ResFwdCfg<P, SPLIT>;
  constexpr int STAGES = C::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sW = smem;
  uint8_t* sIn = smem + C::W_BYTES;
  float* img = reinterpret_cast<float*>(sIn + STAGES * C::IN_BYTES);
  uint8_t* sU8 = sIn + STAGES * C::IN_BYTES + 2 * C::IMG_BYTES;           // U8 only
  uint64_t* bars = reinterpret_cast<uint64_t*>(sU8 + STAGES * C::U8_BYTES);
  uint64_t* in_full = bars;
  uint64_t* in_empty = bars + STAGES;
  uint64_t* w_full = bars + 2 * STAGES;
  uint64_t* u8_full = bars + 2 * STAGES + 1;         // U8 only
  uint64_t* u8_empty = bars + 3 * STAGES + 1;
  const int tid = threadIdx.x, warp = tid >> 5;
  const int ntiles = P::num_tiles(p);

  if (warp == 8 && (tid & 31) == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&in_full[s], C::U8 ? 3 : 1); mbar_init(&in_empty[s], 4); }
    if constexpr (C::U8)
      for (int s = 0; s < STAGES; ++s) { mbar_init(&u8_full[s], 1); mbar_init(&u8_empty[s], 3); }
    mbar_init(w_full, 1);
    mbar_fence_init();
    P::prefetch(p);
  }
  __syncthreads();

  if (warp >= 8) {
    reg_release<C::PRODUCER_REGS>();
    if constexpr (C::U8) {
      if (warp != 8) { res_u8_converters<P, C>(p, sIn, sU8, in_full, in_empty, u8_full, u8_empty, tid); return; }
    } else if (warp != 8) return;          // warps 9-11 only give their registers back
    const uint32_t leader = elect_one_sync();      // converged warp, one elected issuing lane: no vote loop around every TMA instruction
    // the packed weights were complete before the first kernel of the chain started: their load overlaps the previous
    // kernel's tail; the activations are only touched after pdl_wait().  (W_AFTER_WAIT: the weights come from the stream predecessor.)
    auto load_weights = [&]() {
      mbar_arrive_expect_tx(w_full, C::W_BYTES);
      for (int j = 0; j < P::NT; ++j) tma_load_2d(sW + j * P::BN * 128, &p.w, w_full, j * 64, 0);
      if constexpr (SPLIT)
        for (int j = 0; j < P::NT; ++j) tma_load_2d(sW + C::W_HI_BYTES + j * P::BN * 128, &p.w_lo, w_full, j * 64, 0);
    };
    if (leader && !P::W_AFTER_WAIT) load_weights();
    __syncwarp();
    pdl_wait();
    if (leader) pdl_launch();
    if (leader && P::W_AFTER_WAIT) load_weights();
    __syncwarp();
    int it = 0;
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x, ++it) {
      const int s = it % STAGES;
      if constexpr (C::U8) {        // the frame rows of the window: up to STAGES tiles ahead of the converters
        mbar_wait(&u8_empty[s], ((it / STAGES) & 1) ^ 1);
        if (leader) P::load_u8(p, t, sU8 + s * C::U8_BYTES, &u8_full[s]);
      } else {
        mbar_wait(&in_empty[s], ((it / STAGES) & 1) ^ 1);
        if (leader) {
          mbar_arrive_expect_tx(&in_full[s], P::NWIN * P::WROWS * 128 * (1 + C::ALO));
          P::load_windows(p, t, sIn + s * C::IN_BYTES, C::WIN_BYTES, &in_full[s], false);
          if constexpr (C::ALO) P::load_windows(p, t, sIn + s * C::IN_BYTES + C::IN_HI_BYTES, C::WIN_BYTES, &in_full[s], true);
        }
      }
      __syncwarp();
    }
  } else {
    reg_claim<C::CONSUMER_REGS>();
    pdl_wait(P::KID);
    // consumer warpgroup g takes this CTA's tiles it = g, g + 2, ...: its epilogue overlaps the other warpgroup's MMAs.  With a
    // single input stage warpgroup 0 takes every tile: tile it + 2 would be awaited on the same barrier with the parity of the
    // phase that just completed (tile it), before tile it + 1 was even loaded.
    // Descriptors are base + constant: the 14-bit address field cannot carry.
    const int g = warp >> 2, wt = tid & 127;
    float* my_img = img + g * (C::IMG_BYTES / 4);
    constexpr uint32_t A_HI = 64 * 128 / 16;       // rows 64..127 of the position tile
    mbar_wait(w_full, 0);
    const uint64_t wd = make_smem_desc(smem_u32(sW), 16, 1024);
    int it = 0;
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x, ++it) {
      if (STAGES > 1 ? (it & 1) != g : g != 0) continue;
      const int s = it % STAGES;
      // global operands of the epilogue (ReLU masks of the dgrads) are requested before the MMAs: their L2 latency overlaps them
      uint4 pre[P::BN / 16][2];
      if constexpr (C::TILE_EPI) P::prefetch_tile(p, t, wt, pre);
      else {
#pragma unroll
        for (int c = 0; c < P::BN / 16; ++c) P::prefetch16(p, t, wt, c * 16, pre[c]);
      }
      float acc[2][P::BN / 2];
      mbar_wait(&in_full[s], (it / STAGES) & 1);
      const uint64_t ind = make_smem_desc(smem_u32(sIn + s * C::IN_BYTES), 16, 1024);
      wg_fence();
#pragma unroll
      for (int j = 0; j < P::NT; ++j) {
        const uint64_t ad = ind + (uint64_t)((P::tap_win(j) * C::WIN_BYTES + P::tap_shift(j) * 128) / 16);
        const uint64_t bd = wd + (uint64_t)(j * P::BN * 128 / 16);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          wg_mma128<P::BN, 0, 0>(acc, ad + 2 * k, A_HI, bd + 2 * k, (j | k) != 0);
          if constexpr (SPLIT)          // hi * lo(weights)
            wg_mma128<P::BN, 0, 0>(acc, ad + 2 * k, A_HI, bd + (uint64_t)(C::W_HI_BYTES / 16 + 2 * k), 1);
          if constexpr (C::ALO)         // lo(activations) * hi
            wg_mma128<P::BN, 0, 0>(acc, ad + (uint64_t)(C::IN_HI_BYTES / 16 + 2 * k), A_HI, bd + 2 * k, 1);
        }
      }
      wg_commit();
      wg_wait_all();
      wg_fence_regs(acc[0]); wg_fence_regs(acc[1]);
      __syncwarp();
      if ((tid & 31) == 0) mbar_arrive(&in_empty[s]);
      if constexpr (C::TILE_EPI) P::epilogue_tile(p, t, wt, acc, reinterpret_cast<uint8_t*>(my_img), 2 + g, pre);
      else {
#pragma unroll
        for (int c = 0; c < P::BN / 16; ++c) {
          float v[16];
          wg_acc_row16<P::BN, C::IMG1>(acc, c, my_img, wt, 2 + g, v);
          P::template epilogue16<SPLIT>(p, t, wt, c * 16, v, pre[c]);
        }
      }
    }
  }
}

template <class P, int SPLIT>
cudaError_t res_fwd_launch_t(const typename P::Params& p, int ntiles, int max_ctas, cudaStream_t stream) {
  using C = ResFwdCfg<P, SPLIT>;
  if (ntiles <= 0) return cudaSuccess;
  static PerDeviceOnce once;
  { cudaError_t e = ensure_max_dynamic_smem(once, res_fwd_kernel<P, SPLIT>, C::SMEM_BYTES); if (e != cudaSuccess) return e; }
  const int grid = ntiles < max_ctas ? ntiles : max_ctas;
  return launch_chain(res_fwd_kernel<P, SPLIT>, dim3(grid), dim3(RES_THREADS), C::SMEM_BYTES, stream, p);
}
template <class P>
cudaError_t res_fwd_launch(const typename P::Params& p, int ntiles, int max_ctas, cudaStream_t stream, int split = 0) {
  return split ? res_fwd_launch_t<P, 1>(p, ntiles, max_ctas, stream) : res_fwd_launch_t<P, 0>(p, ntiles, max_ctas, stream);
}

// ------------------------------------------------------------------------------------------------------------------
// wgrad
//   P: NBLK tap blocks (each M = 64 rows of dW = 64 window rows, N = DY_CH), CWG consumer warpgroups, NWIN, WROWS
//      (= 128 + max shift), STAGES, blk_win(b), blk_shift(b), PART (floats per CTA slice: tap blocks [b][row][co], then
//      BIAS_CH bias sums), Params{ in[NWIN] maps, dy map, ws, P (positions), chunks_per_cta }
// ------------------------------------------------------------------------------------------------------------------
template <class P, int SPLIT>
struct ResWgradCfg {
  static constexpr int ALO = (SPLIT && P::A_LO) ? 1 : 0;          // the input window has a low tensor (not conv1: exact u8 frames)
  static constexpr int WIN_BYTES = ((P::WROWS * 128 + 1023) / 1024) * 1024;
  static constexpr int DY_BYTES = 128 * P::DY_CH * 2;             // 128 positions x DY_CH channels (64: SWIZZLE_128B rows, 32: SWIZZLE_64B rows)
  static constexpr int X_HI_BYTES = P::NWIN * WIN_BYTES;
  static constexpr int X_BYTES = X_HI_BYTES * (1 + ALO);
  static constexpr int STAGE_BYTES = X_BYTES + DY_BYTES * (1 + SPLIT);     // [windows hi][windows lo][dY hi][dY lo]
  // warps: [CWG consumer warpgroups] [producer warpgroup: warp 0 also issues the TMA loads; the four warps produce the bias gradient]
  // bias gradient: column sums of the staged dY tiles, or (BIAS_MMA: conv3 in the bf16 mode) a wgmma of an all-ones block with the
  // dY tile -- the tensor cores' sum, the bits conv3's bias gradient has always had
  static constexpr bool BIAS_MMA = !P::SMEM_BIAS && !SPLIT;
  static constexpr int ONES_BYTES = BIAS_MMA ? 128 * 128 : 0;
  // consumer warpgroup w holds tap blocks w * BPW .. w * BPW + BPW - 1 (fewer in the last one)
  static constexpr int CWG = P::CWG, BPW = (P::NBLK + CWG - 1) / CWG;
  static constexpr int PRODUCER_WARP = 4 * CWG;
  static constexpr int THREADS = 32 * (PRODUCER_WARP + 4);
  // ptxas keeps wgmma accumulators within the kernel's launch register count (65536 / THREADS), not within the setmaxnreg
  // budget: a warpgroup's accumulators must leave room there for descriptors and loop state, or every wgmma is serialized
  static_assert(BPW * P::DY_CH / 2 + 32 <= (65536 / THREADS & ~7), "wgmma accumulators exceed the launch register count");
  // per-thread register budgets: one warp of every warpgroup shares a sub-partition, PRODUCER + CWG x CONSUMER <= 512
  static constexpr int PRODUCER_REGS = BIAS_MMA ? 96 : 56;      // BIAS_MMA: one m64 accumulator (32 registers) on top
  static constexpr int CONSUMER_REGS = ((512 - PRODUCER_REGS) / CWG & ~7) < 232 ? ((512 - PRODUCER_REGS) / CWG & ~7) : 232;
  static constexpr int BIAS_BYTES = 2048;                          // bias partial sums of the four warps + the release-ordering slots
  static constexpr int FIXED_BYTES = ONES_BYTES + CWG * WG_IMG_BYTES + BIAS_BYTES + 1024 + 256;
  static constexpr int STAGES = fit_stages(SPLIT ? P::SPLIT_STAGES : P::STAGES, FIXED_BYTES, STAGE_BYTES);
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + FIXED_BYTES;
  static_assert(SMEM_BYTES <= 232448, "shared memory budget (227 KB)");
};

SRL_DEVINL void store16(float* dst, const float (&v)[16]) {
#pragma unroll
  for (int j = 0; j < 16; j += 4) *reinterpret_cast<float4*>(dst + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
}

// consumer warpgroup W of res_wgrad_kernel: its tap blocks are a compile-time set, so no wgmma sits behind a branch
template <class P, int SPLIT, int W>
SRL_DEVINL void res_wgrad_consumer(const typename P::Params& p, uint8_t* sSt, float* img, uint64_t* full, uint64_t* empty, int nch, int tid) {
  using C = ResWgradCfg<P, SPLIT>;
  constexpr int STAGES = C::STAGES, B0 = W * C::BPW, NB = P::NBLK - B0 < C::BPW ? P::NBLK - B0 : C::BPW;
  constexpr uint32_t DYK = P::DY_CH * 2;           // descriptor address units per K = 16 step of the dY tile (16 rows x row bytes / 16)
  const int wt = tid & 127;
  float acc[NB][P::DY_CH / 2];
#pragma unroll
  for (int b = 0; b < NB; ++b)
#pragma unroll
    for (int j = 0; j < P::DY_CH / 2; ++j) acc[b][j] = 0.f;
  for (int i = 0; i < nch; ++i) {
    const int s = i % STAGES;
    mbar_wait(&full[s], (i / STAGES) & 1);
    const uint32_t st = smem_u32(sSt + s * C::STAGE_BYTES);
    const uint64_t dyd = P::DY_CH == 64 ? make_smem_desc(st + C::X_BYTES, 8192, 1024) : make_smem_desc_sw64(st + C::X_BYTES, 4096, 512);
    wg_fence();
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      const uint64_t xd = make_smem_desc(st + P::blk_win(B0 + b) * C::WIN_BYTES + P::blk_shift(B0 + b) * 128, 8192, 1024);
#pragma unroll
      for (int k = 0; k < 8; ++k) {          // 128 positions = 8 x (K = 16): +2048 B per step
        Wgmma<P::DY_CH, 1, 1>::mma(acc[b], xd + 128 * k, dyd + DYK * k, 1);
        if constexpr (SPLIT)         // hi(x) * lo(dy)
          Wgmma<P::DY_CH, 1, 1>::mma(acc[b], xd + 128 * k, dyd + (uint64_t)(C::DY_BYTES / 16 + DYK * k), 1);
        if constexpr (C::ALO)        // lo(x) * hi(dy)
          Wgmma<P::DY_CH, 1, 1>::mma(acc[b], xd + (uint64_t)(C::X_HI_BYTES / 16 + 128 * k), dyd + DYK * k, 1);
      }
    }
    wg_commit();
    if constexpr (STAGES > 1) {
      // chunk i stays in flight while chunk i + 1 is awaited and issued; chunk i - 1's stage is released as soon as it retired
      wg_wait_prev();
      __syncwarp();
      if (i > 0 && (tid & 31) == 0) mbar_arrive(&empty[(i - 1) % STAGES]);
    } else {     // one stage: the next chunk can only be loaded once this one retired
      wg_wait_all();
      __syncwarp();
      if ((tid & 31) == 0) mbar_arrive(&empty[s]);
    }
  }
  wg_wait_all();
#pragma unroll
  for (int b = 0; b < NB; ++b) wg_fence_regs(acc[b]);
  if (nch > 0) {
    // tap blocks leave in pairs (thread wt: row wt & 63 of block b + wt / 64); an odd last block is paired with itself
    float* my_img = img + W * (WG_IMG_BYTES / 4);
    float* ws = p.ws + (size_t)blockIdx.x * P::PART;
#pragma unroll
    for (int b = 0; b < NB; b += 2) {
      const int b1 = b + 1 < NB ? b + 1 : b;
#pragma unroll
      for (int c = 0; c < P::DY_CH / 16; ++c) {       // an even number of 16-column chunks: the hand-off buffers keep alternating
        float v[16];
        wg_acc_rows16<P::DY_CH>(acc[b], acc[b1], c, my_img, wt, 2 + W, v);
        if (wt < 64 || b1 != b) store16(ws + ((size_t)(B0 + b) * 64 + wt) * P::DY_CH + c * 16, v);
      }
    }
  }
}

template <class P, int SPLIT>
__global__ void __launch_bounds__(ResWgradCfg<P, SPLIT>::THREADS, 1) res_wgrad_kernel(const __grid_constant__ typename P::Params p) {
  using C = ResWgradCfg<P, SPLIT>;
  constexpr int STAGES = C::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sSt = smem;
  uint8_t* sOnes = smem + STAGES * C::STAGE_BYTES;              // 1024-aligned: every stage is a multiple of 1024 bytes
  float* img = reinterpret_cast<float*>(sOnes + C::ONES_BYTES);
  uint8_t* sBias = sOnes + C::ONES_BYTES + C::CWG * WG_IMG_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sBias + C::BIAS_BYTES);
  uint64_t* full = bars;
  uint64_t* empty = bars + STAGES;
  const int tid = threadIdx.x, warp = tid >> 5;
  const int nchunks_total = (p.P + 127) >> 7;
  const int c_begin = blockIdx.x * p.chunks_per_cta;
  const int c_end = min(nchunks_total, c_begin + p.chunks_per_cta);
  const int nch = max(0, c_end - c_begin);

  if constexpr (C::BIAS_MMA) {  // all-ones block (bf16 1.0): 128 positions x 64 rows
    uint4* q = reinterpret_cast<uint4*>(sOnes);
    for (int i = tid; i < C::ONES_BYTES / 16; i += C::THREADS) q[i] = make_uint4(0x3F803F80u, 0x3F803F80u, 0x3F803F80u, 0x3F803F80u);
    fence_proxy_async_smem();
  }
  if (warp == C::PRODUCER_WARP && (tid & 31) == 0) {
    // a stage is free after every consumer warp passed its wgmma wait and the four producer warps used its dY tile
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 4 * C::CWG + 4); }
    mbar_fence_init();
    P::prefetch(p);
  }
  __syncthreads();
  pdl_wait(P::KID);
  if (warp == C::PRODUCER_WARP && (tid & 31) == 0) pdl_launch();

  // each role sets its register budget inside its own branch: ptxas ignores a setmaxnreg that is followed by shared code
  // the warpgroup index through a shuffle: ptxas then knows it is warp-uniform and does not serialize the wgmma behind the branches
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);
  if (wg < C::CWG) {
    static_assert(C::CWG == 2 || C::CWG == 3, "two or three consumer warpgroups");
    reg_claim<C::CONSUMER_REGS>();
    if (wg == 0) res_wgrad_consumer<P, SPLIT, 0>(p, sSt, img, full, empty, nch, tid);
    else if (C::CWG == 2 || wg == 1) res_wgrad_consumer<P, SPLIT, 1>(p, sSt, img, full, empty, nch, tid);
    else if constexpr (C::CWG == 3) res_wgrad_consumer<P, SPLIT, 2>(p, sSt, img, full, empty, nch, tid);
  } else {
    reg_release<C::PRODUCER_REGS>();
    // warp 0 of this warpgroup keeps the ring full: chunks 0 .. STAGES-1 up front, chunk i + STAGES once chunk i is summed
    // (its stage is free as soon as the consumers retired chunk i too)
    const bool issuer = warp == C::PRODUCER_WARP;
    const uint32_t leader = elect_one_sync();
    auto load = [&](int i) {
      const int s = i % STAGES;
      mbar_wait(&empty[s], ((i / STAGES) & 1) ^ 1);
      if (leader) {
        mbar_arrive_expect_tx(&full[s], P::NWIN * P::WROWS * 128 * (1 + C::ALO) + C::DY_BYTES * (1 + SPLIT));
        uint8_t* st = sSt + s * C::STAGE_BYTES;
        P::load_windows(p, c_begin + i, st, C::WIN_BYTES, &full[s], false);
        if constexpr (C::ALO) P::load_windows(p, c_begin + i, st + C::X_HI_BYTES, C::WIN_BYTES, &full[s], true);
        tma_load_2d(st + C::X_BYTES, &p.dy, &full[s], 0, (c_begin + i) * 128);
        if constexpr (SPLIT) tma_load_2d(st + C::X_BYTES + C::DY_BYTES, &p.dy_lo, &full[s], 0, (c_begin + i) * 128);
      }
      __syncwarp();
    };
    if (issuer)
      for (int i = 0; i < STAGES && i < nch; ++i) load(i);
    if constexpr (C::BIAS_MMA) {
      // bias gradient = ones^T dY: every row of the m64 accumulator holds the column sums; row 0 sits in lanes 0-3 of warp 0
      constexpr uint32_t DYK = P::DY_CH * 2;
      float bacc[P::DY_CH / 2];
#pragma unroll
      for (int j = 0; j < P::DY_CH / 2; ++j) bacc[j] = 0.f;
      const uint64_t od = make_smem_desc(smem_u32(sOnes), 8192, 1024);
      for (int i = 0; i < nch; ++i) {
        const int s = i % STAGES;
        mbar_wait(&full[s], (i / STAGES) & 1);
        const uint64_t dyd = make_smem_desc(smem_u32(sSt + s * C::STAGE_BYTES + C::X_BYTES), 8192, 1024);
        wg_fence();
#pragma unroll
        for (int k = 0; k < 8; ++k) Wgmma<P::DY_CH, 1, 1>::mma(bacc, od + 128 * k, dyd + DYK * k, 1);
        wg_commit();
        if constexpr (STAGES > 1) {        // as in the consumers: chunk i - 1's stage is released (and refilled) once it retired
          wg_wait_prev();
          __syncwarp();
          if (i > 0 && (tid & 31) == 0) mbar_arrive(&empty[(i - 1) % STAGES]);
          if (issuer && i > 0 && i - 1 + STAGES < nch) load(i - 1 + STAGES);
        } else {
          wg_wait_all();
          __syncwarp();
          if ((tid & 31) == 0) mbar_arrive(&empty[s]);
          if (issuer && i + 1 < nch) load(i + 1);
        }
      }
      wg_wait_all();
      wg_fence_regs(bacc);
      const int bt = tid & 127;
      if (bt < 4 && nch > 0) {
        float* db = p.ws + (size_t)blockIdx.x * P::PART + P::PART - P::BIAS_CH;
#pragma unroll
        for (int j = 0; j < P::DY_CH / 8; ++j) { db[8 * j + 2 * bt] = bacc[4 * j]; db[8 * j + 2 * bt + 1] = bacc[4 * j + 1]; }
      }
      return;
    }
    // bias gradient = column sums of dy, taken from the staged dy tiles while the MMAs run.
    // dy tile rows: DY_CH channels = NG 16-byte groups; thread -> group g, rows q + RP k (RP rows per pass, NG passes)
    constexpr int NG = P::DY_CH / 8, RP = 128 / NG;
    const int bt = tid & 127, bw = bt >> 5;
    const int g = bt & (NG - 1), q = bt / NG;
    float bs[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) bs[j] = 0.f;
    // Releasing a stage lets the producer's TMA overwrite it.  mbarrier.arrive does NOT wait for this warp's loads that
    // are still in flight (a generic LD.E.128 of the tile can be overtaken by the arrive -> rows of the NEXT chunk would be
    // summed).  So the tile is read with ld.shared (same pipe as the mbarrier op), and every lane stores a value that
    // depends on all of its loads before the warp arrives: the store cannot issue until the loads returned, and the
    // arrive (release) is ordered after the store.
    const uint32_t dep_slot = smem_u32(sBias) + 1024 + bt * 4;
    for (int i = 0; i < nch; ++i) {
      const int s = i % STAGES;
      mbar_wait(&full[s], (i / STAGES) & 1);
      const uint32_t dyt = smem_u32(sSt + s * C::STAGE_BYTES + C::X_BYTES);
      float dep = 0.f;
#pragma unroll
      for (int part = 0; part <= SPLIT; ++part) {        // split mode: the low tile's column sums are added too
#pragma unroll
        for (int k = 0; k < NG; ++k) {
          const uint4 v = lds128(dyt + part * C::DY_BYTES + (P::DY_CH == 64 ? swz128(q + RP * k, g) : swz64(q + RP * k, g)));
          bs[0] += bf16_lo(v.x); bs[1] += bf16_hi(v.x); bs[2] += bf16_lo(v.y); bs[3] += bf16_hi(v.y);
          bs[4] += bf16_lo(v.z); bs[5] += bf16_hi(v.z); bs[6] += bf16_lo(v.w); bs[7] += bf16_hi(v.w);
          dep += __uint_as_float(v.x ^ v.y ^ v.z ^ v.w);
        }
      }
      sts_volatile_f32(dep_slot, dep);
      __syncwarp();
      if ((tid & 31) == 0) mbar_arrive(&empty[s]);
      if (issuer && i + STAGES < nch) load(i + STAGES);
    }
    float* red = reinterpret_cast<float*>(sBias);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (NG == 4) bs[j] += __shfl_xor_sync(0xffffffffu, bs[j], 4);
      bs[j] += __shfl_xor_sync(0xffffffffu, bs[j], 8);
      bs[j] += __shfl_xor_sync(0xffffffffu, bs[j], 16);
    }
    if ((tid & 31) < NG) {
#pragma unroll
      for (int j = 0; j < 8; ++j) red[bw * 64 + g * 8 + j] = bs[j];
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");        // this warpgroup only
    if (bt < P::BIAS_CH && nch > 0) p.ws[(size_t)blockIdx.x * P::PART + P::PART - P::BIAS_CH + bt] = red[bt] + red[64 + bt] + red[128 + bt] + red[192 + bt];
  }
}

// *ctas: the CTAs launched, i.e. the per-CTA partial slices conv_wgrad_reduce_kernel<layer> must add (0: nothing launched)
template <class P, int SPLIT>
cudaError_t res_wgrad_launch_t(typename P::Params p, int target_ctas, cudaStream_t stream, int* ctas) {
  using C = ResWgradCfg<P, SPLIT>;
  static_assert(P::PART >= P::NBLK * 64 * P::DY_CH + P::BIAS_CH, "partial slice layout");
  const int nchunks = (p.P + 127) >> 7;
  *ctas = 0;
  if (nchunks <= 0) return cudaSuccess;
  if (target_ctas > WG_PART_CTAS) target_ctas = WG_PART_CTAS;
  static PerDeviceOnce once;
  { cudaError_t e = ensure_max_dynamic_smem(once, res_wgrad_kernel<P, SPLIT>, C::SMEM_BYTES); if (e != cudaSuccess) return e; }
  p.chunks_per_cta = (nchunks + target_ctas - 1) / target_ctas;
  const int grid = (nchunks + p.chunks_per_cta - 1) / p.chunks_per_cta;
  *ctas = grid;
  return launch_chain(res_wgrad_kernel<P, SPLIT>, dim3(grid), dim3(C::THREADS), C::SMEM_BYTES, stream, p);
}
template <class P>
cudaError_t res_wgrad_launch(const typename P::Params& p, int target_ctas, cudaStream_t stream, int* ctas, int split = 0) {
  return split ? res_wgrad_launch_t<P, 1>(p, target_ctas, stream, ctas) : res_wgrad_launch_t<P, 0>(p, target_ctas, stream, ctas);
}

}  // namespace srl
