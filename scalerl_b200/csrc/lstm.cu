// 2-layer LSTM core of AtariNet(use_lstm=True): forward over T1 steps with done-resets and BPTT over the first T steps (the learner:
// T = T1 - 1; the trainable AtariNet's stand-alone core: T = T1, with the gradients of the initial and the returned state)
// (reference: scalerl/algorithms/utils/atari_model.py:52-55,61-75,109-120; SURVEY.md §8 row a17).
//
//   gates_t = x_t Wih^T + b_ih + (m_t . h_{t-1}) Whh^T + b_hh ;  i,f,g,o ;  c_t = f (m_t . c_{t-1}) + i g ;  h_t = o tanh(c_t)
//
// Work split per layer:
//   * input projection of ALL steps in one wgmma GEMM     [T1*B x Hp] x [Hp x 4Hp]          (LGemmK)
//   * per step: recurrent wgmma GEMM [B x Hp] x [Hp x 4Hp] + one fused cell kernel     (sequential over t)
//   * BPTT per step: cell backward kernel + recurrent GEMM [B x 4Hp] x [4Hp x Hp]
//   * after the scan: dX (one GEMM), dWih / dWhh (two MN-major GEMMs over all T*B rows), bias gradients (column sums over fixed
//     64-row chunks, added in chunk order: no atomics)
// H = 513 + A is padded to Hp (multiple of 64); the gate dimension is laid out [4][Hp] so every GEMM has K = Hp or 4Hp.
// All GEMM operands are bf16 (fp32 accumulate); cell state, gate activations and gradients are fp32.
// The actor's single step (one row of B environments, no BPTT) has its own fused kernel further down (lstm_step_kernel).
#include <cstring>
#include <new>
#include "tma_problems.cuh"
#include "kernels.h"
#include "errors.h"
#include "../../include/scalerl_b200.h"

namespace srl {

// ------------------------------------------------------------------------------------------------ generic GEMM problems
struct LGemmK {
  static constexpr int KID = 34;
  static constexpr bool PREFETCH = false;      // C[c_row0 + m][n] = sum_k A[a_row0 + m][k] * B[n][k];  grid = (ceil(M/128), Npad/64)
  static constexpr int BN = 64, STAGES = 4, KROWS = 64;
  static constexpr bool A_MN = false, B_MN = false, ZERO_INIT = false;
  static constexpr int TILE_ROWB = 0;          // row hand-off
  struct Params { SRL_TMAP a; SRL_TMAP b; float* C; int M, nkb, ldc, a_row0, c_row0; };
  SRL_DEVINL static void prefetch(const Params& p) { tma_prefetch_desc(&p.a); tma_prefetch_desc(&p.b); }
  SRL_DEVINL static int num_kblocks(const Params& p, int, int) { return p.nkb; }
  SRL_DEVINL static void issue(const Params& p, int tm, int ty, int kb, uint8_t* sA, uint8_t* sB, uint64_t* bar) {
    mbar_arrive_expect_tx(bar, 128 * 128 + 64 * 128);
    tma_load_2d(sA, &p.a, bar, kb * 64, p.a_row0 + tm * 128);
    tma_load_2d(sB, &p.b, bar, kb * 64, ty * 64);
  }
  SRL_DEVINL static void epilogue16(const Params& p, int tm, int ty, int row, int c0, float (&v)[16]) {
    const int m = tm * 128 + row;
    if (m >= p.M) return;
    float4* o = reinterpret_cast<float4*>(p.C + (size_t)(p.c_row0 + m) * p.ldc + ty * 64 + c0);
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
  }
};
struct LGemmMN {
  static constexpr int KID = 35;
  static constexpr bool PREFETCH = false;     // C[i][j] = sum_r A[r][i] * B[r][j]  (rows r = samples, MN-major operands); grid = (Ipad/128, Jpad/64)
  static constexpr int BN = 64, STAGES = 4, KROWS = 64;
  static constexpr bool A_MN = true, B_MN = true, ZERO_INIT = false;
  static constexpr int TILE_ROWB = 0;         // row hand-off
  struct Params { SRL_TMAP a; SRL_TMAP b; float* C; int R, ldc; };
  SRL_DEVINL static void prefetch(const Params& p) { tma_prefetch_desc(&p.a); tma_prefetch_desc(&p.b); }
  SRL_DEVINL static int num_kblocks(const Params& p, int, int) { return (p.R + 63) >> 6; }
  SRL_DEVINL static void init_smem(const Params&, int, int, uint8_t*, int, int) {}
  SRL_DEVINL static void issue(const Params& p, int tm, int ty, int kb, uint8_t* sA, uint8_t* sB, uint64_t* bar) {
    mbar_arrive_expect_tx(bar, 3 * 64 * 128);
    tma_load_2d(sA, &p.a, bar, tm * 128, kb * 64);
    tma_load_2d(sA + KROWS * 128, &p.a, bar, tm * 128 + 64, kb * 64);
    tma_load_2d(sB, &p.b, bar, ty * 64, kb * 64);
  }
  SRL_DEVINL static void epilogue16(const Params& p, int tm, int ty, int row, int c0, float (&v)[16]) {
    float4* o = reinterpret_cast<float4*>(p.C + (size_t)(tm * 128 + row) * p.ldc + ty * 64 + c0);
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
  }
};

// ------------------------------------------------------------------------------------------------ element-wise kernels
SRL_DEVINL float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

// fp32 [rows][H] -> bf16 [rows][Hp] (zero padded)
__global__ void lstm_pad_bf16_kernel(const float* __restrict__ x, int rows, int H, int Hp, __nv_bfloat16* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)rows * Hp) return;
  const int r = (int)(i / Hp), j = (int)(i - (int64_t)r * Hp);
  out[i] = __float2bfloat16_rn(j < H ? x[(size_t)r * H + j] : 0.f);
}
// weights fp32 [4H][H] -> bf16 Wp [4Hp][Hp] (gate-major rows, zero padded) and its transpose WTp [Hp][4Hp]
__global__ void lstm_pack_w_kernel(const float* __restrict__ w, int H, int Hp, __nv_bfloat16* __restrict__ Wp, __nv_bfloat16* __restrict__ WTp) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int G = 4 * Hp;
  if (i >= (int64_t)G * Hp) return;
  const int row = (int)(i / Hp), k = (int)(i - (int64_t)row * Hp), q = row / Hp, j = row - q * Hp;
  const float v = (j < H && k < H) ? w[(size_t)(q * H + j) * H + k] : 0.f;
  const __nv_bfloat16 b = __float2bfloat16_rn(v);
  Wp[i] = b;
  WTp[(size_t)k * G + row] = b;
}
// state for step 0: hm[0] = m_0 . h_init (bf16, padded)
__global__ void lstm_init_hm_kernel(const float* __restrict__ h_init, const uint8_t* __restrict__ done, int B, int H, int Hp,
                                    __nv_bfloat16* __restrict__ hm0) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * Hp) return;
  const int b = i / Hp, j = i - b * Hp;
  const float m = done[b] ? 0.f : 1.f;
  hm0[i] = __float2bfloat16_rn(j < H ? m * h_init[(size_t)b * H + j] : 0.f);
}

// fused cell, one thread per (b, j): consumes gx[t], the recurrent product r, biases; writes gate activations, c_t, h_t (fp32),
// h_t (bf16, input of the next layer / wgrad operand) and hm[t+1] = m_{t+1} . h_t (bf16, next step's recurrent operand)
__global__ void lstm_cell_fwd_kernel(const float* __restrict__ gx, const float* __restrict__ r, const float* __restrict__ b_ih,
                                     const float* __restrict__ b_hh, const float* __restrict__ c_prev, const uint8_t* __restrict__ done_t,
                                     const uint8_t* __restrict__ done_next, int B, int H, int Hp, float* __restrict__ gates,
                                     float* __restrict__ c_out, float* __restrict__ h_out, __nv_bfloat16* __restrict__ h_bf,
                                     __nv_bfloat16* __restrict__ hm_next) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * Hp) return;
  const int b = i / Hp, j = i - b * Hp, G = 4 * Hp;
  float hv = 0.f, cv = 0.f, a[4] = {0.f, 0.f, 0.f, 0.f};
  if (j < H) {
    float pre[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) pre[q] = gx[(size_t)b * G + q * Hp + j] + r[(size_t)b * G + q * Hp + j] + b_ih[q * H + j] + b_hh[q * H + j];
    a[0] = sigmoidf_(pre[0]); a[1] = sigmoidf_(pre[1]); a[2] = tanhf(pre[2]); a[3] = sigmoidf_(pre[3]);
    const float cp = done_t[b] ? 0.f : c_prev[(size_t)b * Hp + j];
    cv = a[1] * cp + a[0] * a[2];
    hv = a[3] * tanhf(cv);
  }
#pragma unroll
  for (int q = 0; q < 4; ++q) gates[(size_t)b * G + q * Hp + j] = a[q];
  c_out[i] = cv;
  h_out[i] = hv;
  h_bf[i] = __float2bfloat16_rn(hv);
  if (hm_next) hm_next[i] = __float2bfloat16_rn(done_next[b] ? 0.f : hv);
}

// BPTT cell: dh = dh_out[t] + m_{t+1} . dhm_{t+1};  writes dgates (bf16) and the carried dc.  done_next == nullptr: dhm_next is added
// unmasked (the gradient of the returned state hT, seeding the last step)
__global__ void lstm_cell_bwd_kernel(const float* __restrict__ dh_out, const float* __restrict__ dhm_next, const uint8_t* __restrict__ done_next,
                                     const float* __restrict__ gates, const float* __restrict__ c_t, const float* __restrict__ c_prev,
                                     const uint8_t* __restrict__ done_t, float* __restrict__ dc_carry, int B, int H, int Hp,
                                     __nv_bfloat16* __restrict__ dgates) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * Hp) return;
  const int b = i / Hp, j = i - b * Hp, G = 4 * Hp;
  float d[4] = {0.f, 0.f, 0.f, 0.f};
  float dc_out = 0.f;
  if (j < H) {
    float dh = dh_out ? dh_out[i] : 0.f;
    if (dhm_next && !(done_next && done_next[b])) dh += dhm_next[i];
    const float ig = gates[(size_t)b * G + j], fg = gates[(size_t)b * G + Hp + j], gg = gates[(size_t)b * G + 2 * Hp + j],
                og = gates[(size_t)b * G + 3 * Hp + j];
    const float tc = tanhf(c_t[i]);
    const float dct = dh * og * (1.f - tc * tc) + dc_carry[i];
    const float cp = done_t[b] ? 0.f : c_prev[i];
    d[0] = dct * gg * ig * (1.f - ig);
    d[1] = dct * cp * fg * (1.f - fg);
    d[2] = dct * ig * (1.f - gg * gg);
    d[3] = dh * tc * og * (1.f - og);
    dc_out = done_t[b] ? 0.f : dct * fg;     // flows into c_{t-1} through m_t
  }
  dc_carry[i] = dc_out;
#pragma unroll
  for (int q = 0; q < 4; ++q) dgates[(size_t)b * G + q * Hp + j] = __float2bfloat16_rn(d[q]);
}

// Bias gradient without atomics, the same bits on every run: part[c][col] = sum of dgates[row][col] over the fixed chunk
// c = [64c, 64c + 64) of rows counted from row 0 (grid.y = chunk), then db[q*H + j] += sum_c part[c][q*Hp + j] in chunk order
constexpr int LSTM_BIAS_CHUNK = 64;
__global__ void lstm_bias_part_kernel(const __nv_bfloat16* __restrict__ dgates, int rows, int G, float* __restrict__ part) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= G) return;
  const int r0 = blockIdx.y * LSTM_BIAS_CHUNK, r1 = min(rows, r0 + LSTM_BIAS_CHUNK);
  float s = 0.f;
  for (int r = r0; r < r1; ++r) s += __bfloat162float(dgates[(size_t)r * G + col]);
  part[(size_t)blockIdx.y * G + col] = s;
}
__global__ void lstm_bias_sum_kernel(const float* __restrict__ part, int chunks, int H, int Hp, float* __restrict__ db_ih, float* __restrict__ db_hh) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 4 * H) return;
  const int q = i / H, col = q * Hp + (i - q * H), G = 4 * Hp;
  float s = 0.f;
  for (int c = 0; c < chunks; ++c) s += part[(size_t)c * G + col];
  db_ih[i] += s;
  db_hh[i] += s;
}
// dst[b][j] = done[b] ? 0 : src[b][j] for j < H: the gradient w.r.t. the initial h, which reaches the cell through m_0 . h0
__global__ void lstm_unpad_masked_kernel(const float* __restrict__ src, const uint8_t* __restrict__ done, int B, int H, int Hp, float* __restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * H) return;
  const int b = i / H, j = i - b * H;
  dst[i] = done[b] ? 0.f : src[(size_t)b * Hp + j];
}
// padded fp32 [4Hp][Hp] -> PyTorch [4H][H] (accumulate)
__global__ void lstm_unpad_w_kernel(const float* __restrict__ src, int H, int Hp, float* __restrict__ dst) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)4 * H * H) return;
  const int row = (int)(i / H), k = (int)(i - (int64_t)row * H), q = row / H, j = row - q * H;
  dst[i] += src[(size_t)(q * Hp + j) * Hp + k];
}
// fp32 [rows][Hp] -> fp32 [rows][H]
__global__ void lstm_unpad_rows_kernel(const float* __restrict__ src, int rows, int H, int Hp, float* __restrict__ dst) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)rows * H) return;
  const int r = (int)(i / H), j = (int)(i - (int64_t)r * H);
  dst[i] = src[(size_t)r * Hp + j];
}

// ------------------------------------------------------------------------------------------------ actor step (one row, no BPTT)
// One environment step of both layers for the N environments of an actor call.  Per layer, ONE swap-AB wgmma GEMM
//   gates^T [4Hp x N] = Wl [4Hp x 2Hp] . [x | m.h]^T [2Hp x N]      (Wl = [W_ih | W_hh], bf16; fp32 accumulate)
// with the LSTM cell in the epilogue: the gate pre-activations never leave the CTA.
//   * M = the 4Hp = 2304 gate rows of the packed weights (operand A, TMA); N = environments (operand B, TMA; rows past N are
//     zero-filled by the TMA unit); K = 2Hp = 1152.
//   * Row interleave of the packed weights: a 128-row M tile holds the 4 gates of 32 hidden units, placed so that the
//     wgmma accumulator fragment gives every thread all 4 gates of ONE unit for each of its columns (common.cuh fragment:
//     thread (w, l) of the warpgroup holds rows 16w + l/4 + 8rr of both m64 halves h):
//         tile row R(u, q) = 64 (q >> 1) + 16 (u >> 3) + 8 (q & 1) + (u & 7),   unit j = 32 tm + u,  gate q = 2h + rr.
//   * K split over a thread-block cluster of KS CTAs (grid.z): CTA rank r multiplies k-blocks [r, r+1) * 18/KS, stores its
//     partial accumulators in its own shared memory, and after a cluster barrier every rank reduces a 1/KS share of the
//     columns over distributed shared memory, always adding the ranks in order 0..KS-1 (the result does not depend on
//     which CTA reduces), then runs the cell for that share.
// bf16 rounding points are those of the rollout path: x = bf16(core) / bf16(h of layer 0), m.h = bf16(m * h) (lstm_pad_bf16_kernel,
// lstm_init_hm_kernel, lstm_cell_fwd_kernel), so an actor step and the learner's row differ only in summation order.
constexpr int LS_HP = 576;                       // Hp for every A in [1, 31]: H = 513 + A in [514, 544]
constexpr int LS_G = 4 * LS_HP, LS_K = 2 * LS_HP, LS_KB = LS_K / 64;      // 2304 gate rows, K = 1152, 18 k-blocks
constexpr int LS_BN = 128;                       // environments per CTA: two consumer warpgroups x 64 columns
constexpr int LS_STAGES = 4, LS_TILE = 128 * 128, LS_STAGE = 2 * LS_TILE;
constexpr int LS_PART = 64 * 256 * 4;            // K-split partials: 64 accumulators x 256 consumer threads
constexpr int LS_THREADS = 288;
constexpr int LS_SMEM = LS_STAGES * LS_STAGE + LS_PART + 256 + 1024;

struct LstmStepParams {
  SRL_TMAP w;                  // packed weights of both layers [2 * 4Hp][2Hp] bf16, box 64 x 128
  SRL_TMAP xh;                 // this layer's operand [N][2Hp] bf16 = [x | m.h], box 64 x 128
  const float *b_ih, *b_hh;    // this layer's biases, PyTorch layout [4H]
  const float* c_in;           // [N][H] (this layer's slice of c_in [2][N][H])
  const uint8_t* done;         // [N]
  float *c_out, *h_out;        // [N][H]
  __nv_bfloat16* x_next;       // layer 0: the x part of layer 1's operand (row stride 2Hp); layer 1: nullptr
  int N, H, w_row0;            // w_row0: first packed row of this layer
};

SRL_DEVINL uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
SRL_DEVINL void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
SRL_DEVINL float ld_dsmem_f32(uint32_t saddr, uint32_t rank) {
  uint32_t remote;
  float v;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(saddr), "r"(rank));
  asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(remote) : "memory");
  return v;
}

// the cell for environment n, hidden unit j: acc = the 4 gate products (i, f, g, o) without biases; bias = {b_ih, b_hh} per gate
SRL_DEVINL void lstm_step_cell(const LstmStepParams& p, int n, int j, const float (&acc)[4], const float (&bias)[8]) {
  if (n >= p.N || j >= p.H) return;
  float pre[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) pre[q] = acc[q] + bias[2 * q] + bias[2 * q + 1];
  const float a0 = sigmoidf_(pre[0]), a1 = sigmoidf_(pre[1]), a2 = tanhf(pre[2]), a3 = sigmoidf_(pre[3]);
  const size_t o = (size_t)n * p.H + j;
  const float cp = p.done[n] ? 0.f : p.c_in[o];
  const float cv = a1 * cp + a0 * a2;
  const float hv = a3 * tanhf(cv);
  p.c_out[o] = cv;
  p.h_out[o] = hv;
  if (p.x_next) p.x_next[(size_t)n * LS_K + j] = __float2bfloat16_rn(hv);
}

template <int KS>
__global__ void __cluster_dims__(1, 1, KS) __launch_bounds__(LS_THREADS) lstm_step_kernel(const __grid_constant__ LstmStepParams p) {
  static_assert(LS_KB % KS == 0, "the K split must divide the 18 k-blocks");
  constexpr int NKB = LS_KB / KS;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* part = reinterpret_cast<float*>(smem + LS_STAGES * LS_STAGE);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + LS_STAGES * LS_STAGE + LS_PART);
  uint64_t* empty = full + LS_STAGES;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tm = blockIdx.x, tn = blockIdx.y;
  const uint32_t rank = KS > 1 ? cluster_ctarank() : 0;
  if (warp == 8 && lane == 0) {
    for (int s = 0; s < LS_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    mbar_fence_init();
    tma_prefetch_desc(&p.w); tma_prefetch_desc(&p.xh);
  }
  __syncthreads();
  pdl_wait();                          // the operands (previous layer / prep kernel) and the state are complete from here on
  if (tid == 256) pdl_launch();
  const int kb0 = (int)rank * NKB;
  const int g = warp >> 2, wt = tid & 127, w = wt >> 5;
  const int j = tm * 32 + 8 * w + (lane >> 2);            // this thread's hidden unit
  const int col0 = tn * LS_BN + g * 64 + 2 * (lane & 3);    // its first environment; + 8 j8 + e
  if (warp == 8) {
    const uint32_t leader = elect_one_sync();
    for (int kb = 0; kb < NKB; ++kb) {
      const int s = kb % LS_STAGES;
      mbar_wait(&empty[s], ((kb / LS_STAGES) & 1) ^ 1);
      if (leader) {
        uint8_t* sA = smem + s * LS_STAGE;
        mbar_arrive_expect_tx(&full[s], LS_STAGE);
        tma_load_2d(sA, &p.w, &full[s], (kb0 + kb) * 64, p.w_row0 + tm * 128);
        tma_load_2d(sA + LS_TILE, &p.xh, &full[s], (kb0 + kb) * 64, tn * LS_BN);
      }
      __syncwarp();
    }
  } else {
    float acc[2][32];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[h][i] = 0.f;
    for (int kb = 0; kb < NKB; ++kb) {
      const int s = kb % LS_STAGES;
      mbar_wait(&full[s], (kb / LS_STAGES) & 1);
      const uint32_t a0 = smem_u32(smem + s * LS_STAGE);
      const uint64_t ad0 = make_smem_desc(a0, 16, 1024), bd0 = make_smem_desc(a0 + LS_TILE + g * 64 * 128, 16, 1024);
      wg_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) wg_mma128<64, 0, 0>(acc, ad0 + (uint64_t)(2 * k), 64 * 128 / 16, bd0 + (uint64_t)(2 * k), (kb | k) != 0);
      wg_commit();
      wg_wait_prev();
      __syncwarp();
      if (kb > 0 && lane == 0) mbar_arrive(&empty[(kb - 1) % LS_STAGES]);
    }
    wg_wait_all();
    wg_fence_regs(acc[0]); wg_fence_regs(acc[1]);
    if constexpr (KS == 1) {
      float bias[8];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        bias[2 * q] = j < p.H ? __ldg(p.b_ih + q * p.H + j) : 0.f;
        bias[2 * q + 1] = j < p.H ? __ldg(p.b_hh + q * p.H + j) : 0.f;
      }
#pragma unroll
      for (int j8 = 0; j8 < 8; ++j8)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float a4[4] = {acc[0][4 * j8 + e], acc[0][4 * j8 + 2 + e], acc[1][4 * j8 + e], acc[1][4 * j8 + 2 + e]};
          lstm_step_cell(p, col0 + 8 * j8 + e, j, a4, bias);
        }
    } else {
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 32; ++i) part[(h * 32 + i) * 256 + g * 128 + wt] = acc[h][i];
    }
  }
  if constexpr (KS > 1) {
    cluster_sync_all();                  // every rank's partials are in its shared memory
    if (warp < 8) {
      float bias[8];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        bias[2 * q] = j < p.H ? __ldg(p.b_ih + q * p.H + j) : 0.f;
        bias[2 * q + 1] = j < p.H ? __ldg(p.b_hh + q * p.H + j) : 0.f;
      }
      const uint32_t base = smem_u32(part) + (uint32_t)(g * 128 + wt) * 4;
#pragma unroll
      for (int j8 = 0; j8 < 8; ++j8) {
        if (j8 % KS != (int)rank) continue;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float a4[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const uint32_t addr = base + (uint32_t)(((q >> 1) * 32 + 4 * j8 + 2 * (q & 1) + e) * 256) * 4;
            float s = ld_dsmem_f32(addr, 0);
#pragma unroll
            for (int r = 1; r < KS; ++r) s += ld_dsmem_f32(addr, r);
            a4[q] = s;
          }
          lstm_step_cell(p, col0 + 8 * j8 + e, j, a4, bias);
        }
      }
    }
    cluster_sync_all();                  // no CTA leaves while a peer still reads its partials
  }
}

// step operands of layer 0 and the recurrent halves of both layers: xh[l][n] = [x | bf16(m_n h_l[n])], x = bf16(core[n]) (layer 0)
__global__ void lstm_step_prep_kernel(const float* __restrict__ core, const uint8_t* __restrict__ done, const float* __restrict__ h_in, int N, int H,
                                      __nv_bfloat16* __restrict__ xh) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * LS_HP) return;
  const int n = i / LS_HP, j = i - n * LS_HP;
  const float m = done[n] ? 0.f : 1.f;
  __nv_bfloat16* r0 = xh + (size_t)n * LS_K;
  __nv_bfloat16* r1 = xh + ((size_t)N + n) * LS_K;
  r0[j] = __float2bfloat16_rn(j < H ? core[(size_t)n * H + j] : 0.f);
  r0[LS_HP + j] = __float2bfloat16_rn(j < H ? m * h_in[(size_t)n * H + j] : 0.f);
  r1[LS_HP + j] = __float2bfloat16_rn(j < H ? m * h_in[((size_t)N + n) * H + j] : 0.f);
}

// packed step weights [2][4Hp][2Hp] bf16: row (layer, tile, R) = [W_ih | W_hh] row q H + j of that layer (interleave above), zero padded
__global__ void lstm_step_pack_kernel(const float* __restrict__ wih0, const float* __restrict__ whh0, const float* __restrict__ wih1,
                                      const float* __restrict__ whh1, int H, __nv_bfloat16* __restrict__ wp) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)2 * LS_G * LS_K) return;
  const int row = (int)(i / LS_K), k = (int)(i - (int64_t)row * LS_K);
  const int l = row / LS_G, R = row - l * LS_G, tile = R >> 7, r = R & 127;
  const int u = 8 * ((r >> 4) & 3) + (r & 7), q = 2 * (r >> 6) + ((r >> 3) & 1), j = 32 * tile + u;
  const int kk = k < LS_HP ? k : k - LS_HP;
  const float* src = k < LS_HP ? (l ? wih1 : wih0) : (l ? whh1 : whh0);
  wp[i] = __float2bfloat16_rn(j < H && kk < H ? src[(size_t)(q * H + j) * H + kk] : 0.f);
}

}  // namespace srl

using namespace srl;

// ------------------------------------------------------------------------------------------------ buffers
extern "C" const char* srl_lstm_last_error(void) { return srl_last_error(); }

namespace srl {
// shape of one forward over N1 = T1*B rows and its backward over the first NB rows (T*B for the learner, T1*B for the stand-alone core)
struct LstmDims {
  int T1, B, H, Hp, G;
  int64_t N1, NB;
};
static LstmDims lstm_dims(int T1, int B, int H, int64_t NB) {
  const int Hp = (H + 63) / 64 * 64;
  return {T1, B, H, Hp, 4 * Hp, (int64_t)T1 * B, NB};
}
struct LstmBuffers {
  // saved: what a backward reads of its forward
  __nv_bfloat16* xin0;                                    // layer 0 input rows [N1][Hp] (layer 1's input is hbf[0])
  __nv_bfloat16 *hm[2], *hbf[2];                          // m_t . h_{t-1} and h_t rows [N1][Hp]
  __nv_bfloat16 *Wih[2], *WihT[2], *Whh[2], *WhhT[2];     // the weights the forward ran with: [4Hp][Hp] and the transposes [Hp][4Hp]
  float *gates[2], *cseq[2];                              // gate activations [N1][4Hp], c_t [N1][Hp]
  float* c_init;                                          // padded initial cell state [2][B][Hp]
  uint8_t* done;                                          // copy of done [N1] (stand-alone core; the learner passes its own)
  // scratch: one call's temporaries
  float *gx, *r, *hseq[2];                                // input projections [N1][4Hp], one step's recurrent product [B][4Hp], h_t [N1][Hp]
  __nv_bfloat16* dgates[2];                               // [NB][4Hp]
  float *dx, *dwpad, *dc, *dhm;                           // dh_out / dx [NB][Hp], padded weight gradient [4Hp][Hp], carries [B][Hp]
  float* bias_part;                                       // per-chunk bias column sums [ceil(NB/64)][4Hp]
};
// The LSTM core's rows.  The first LSTM_SAVED_ROWS are what a backward reads of its forward; the rest live for one call.
constexpr int LSTM_SAVED_ROWS = 19, LSTM_ROWS = 30;
static int lstm_rows(LstmBuffers& b, const LstmDims& d, WsRow* t) {
  const int64_t N1 = d.N1, NB = d.NB, B = d.B, Hp = d.Hp, G = d.G;
  int n = 0;
  t[n++] = ws_row("xin0", N1 * Hp, &b.xin0);
  for (int l = 0; l < 2; ++l) {
    t[n++] = ws_row("hm", N1 * Hp, &b.hm[l]);
    t[n++] = ws_row("hbf", N1 * Hp, &b.hbf[l]);
    t[n++] = ws_row("Wih", G * Hp, &b.Wih[l]);
    t[n++] = ws_row("WihT", G * Hp, &b.WihT[l]);
    t[n++] = ws_row("Whh", G * Hp, &b.Whh[l]);
    t[n++] = ws_row("WhhT", G * Hp, &b.WhhT[l]);
    t[n++] = ws_row("gates", N1 * G, &b.gates[l]);
    t[n++] = ws_row("cseq", N1 * Hp, &b.cseq[l]);
  }
  t[n++] = ws_row("c_init", 2 * B * Hp, &b.c_init);
  t[n++] = ws_row("done", N1, &b.done);
  t[n++] = ws_row("gx", N1 * G, &b.gx);
  t[n++] = ws_row("r", B * G, &b.r);
  for (int l = 0; l < 2; ++l) t[n++] = ws_row("hseq", N1 * Hp, &b.hseq[l]);
  for (int l = 0; l < 2; ++l) t[n++] = ws_row("dgates", NB * G, &b.dgates[l]);
  t[n++] = ws_row("dx", NB * Hp, &b.dx);
  t[n++] = ws_row("dwpad", G * Hp, &b.dwpad);
  t[n++] = ws_row("dc", B * Hp, &b.dc);
  t[n++] = ws_row("dhm", B * Hp, &b.dhm);
  t[n++] = ws_row("bias_part", (NB + LSTM_BIAS_CHUNK - 1) / LSTM_BIAS_CHUNK * G, &b.bias_part);
  return n;
}
// the layer-th row of a carved table called `name` (the per-layer rows appear once per layer, l = 0 first; every other row once)
static int lstm_find_row(const WsRow* t, const char* name, int layer, void** ptr, int64_t* count, const char* what) {
  int seen = 0;
  for (int i = 0; i < LSTM_ROWS; ++i) {
    if (strcmp(t[i].name, name) != 0) continue;
    if (seen++ == layer) { *ptr = *t[i].hi; *count = t[i].count; return 0; }
  }
  if (!seen) return fail(SRL_EINVAL, "%s: unknown buffer '%s'", what, name);
  return fail(SRL_EINVAL, "%s: '%s' exists for layer 0%s only, not layer=%d", what, name, seen > 1 ? " and 1" : "", layer);
}

struct LstmMaps {
  CUtensorMap xin[2], hm[2], hm64[2], xin64[2], Wih[2], Whh[2], WihT[2], WhhT[2], dg128[2], dg64[2];
};
static bool map2(CUtensorMap* m, const void* base, uint64_t cols, uint64_t rows, uint32_t boxrows) {
  const uint64_t d[2] = {cols, rows}, s[1] = {cols};
  const uint32_t bx[2] = {64, boxrows};
  return make_map(m, base, 2, d, s, bx);
}
static bool lstm_maps(const LstmBuffers& b, const LstmDims& d, LstmMaps* m) {
  const uint64_t N1 = d.N1, NB = d.NB, Hp = d.Hp, G = d.G;
  bool ok = true;
  for (int l = 0; l < 2 && ok; ++l) {
    const __nv_bfloat16* xin = l ? b.hbf[0] : b.xin0;
    ok = map2(&m->xin[l], xin, Hp, N1, 128) && map2(&m->xin64[l], xin, Hp, NB, 64) && map2(&m->hm[l], b.hm[l], Hp, N1, 128) &&
         map2(&m->hm64[l], b.hm[l], Hp, NB, 64) && map2(&m->Wih[l], b.Wih[l], Hp, G, 64) && map2(&m->Whh[l], b.Whh[l], Hp, G, 64) &&
         map2(&m->WihT[l], b.WihT[l], G, Hp, 64) && map2(&m->WhhT[l], b.WhhT[l], G, Hp, 64) && map2(&m->dg128[l], b.dgates[l], G, NB, 128) &&
         map2(&m->dg64[l], b.dgates[l], G, NB, 64);
  }
  return ok;
}

static inline int cdiv_(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// core f32 [N1][H], done u8 [N1], h0/c0 f32 [2][B][H], w8 = the 8 nn.LSTM tensors -> out f32 [N1][H], hT/cT f32 [2][B][H] (may be NULL)
static int lstm_forward_rows(const LstmDims& d, const LstmBuffers& b, const LstmMaps& m, const float* const* w8, const float* core,
                             const uint8_t* done, const float* h0, const float* c0, float* out, float* hT, float* cT, cudaStream_t st) {
  const int T1 = d.T1, B = d.B, H = d.H, Hp = d.Hp, G = d.G;
  const int64_t N1 = d.N1;
  lstm_pad_bf16_kernel<<<cdiv_(N1 * Hp, 256), 256, 0, st>>>(core, (int)N1, H, Hp, b.xin0);
  for (int l = 0; l < 2; ++l) {
    lstm_pack_w_kernel<<<cdiv_((int64_t)G * Hp, 256), 256, 0, st>>>(w8[4 * l], H, Hp, b.Wih[l], b.WihT[l]);
    lstm_pack_w_kernel<<<cdiv_((int64_t)G * Hp, 256), 256, 0, st>>>(w8[4 * l + 1], H, Hp, b.Whh[l], b.WhhT[l]);
  }
  CU(cudaGetLastError(), "lstm pack");
  const int cell_blocks = cdiv_((int64_t)B * Hp, 256);
  for (int l = 0; l < 2; ++l) {
    // padded copy of this layer's initial cell state
    CU(cudaMemcpy2DAsync(b.c_init + (size_t)l * B * Hp, Hp * 4, c0 + (size_t)l * B * H, H * 4, H * 4, B, cudaMemcpyDeviceToDevice, st), "c0 copy");
    lstm_init_hm_kernel<<<cell_blocks, 256, 0, st>>>(h0 + (size_t)l * B * H, done, B, H, Hp, b.hm[l]);
    { LGemmK::Params q{m.xin[l], m.Wih[l], b.gx, (int)N1, Hp / 64, G, 0, 0};      // input projection of every step
      CU(igemm_tma_launch<LGemmK>(q, dim3(cdiv_(N1, 128), G / 64), st), "lstm gx gemm"); }
    for (int t = 0; t < T1; ++t) {
      { LGemmK::Params q{m.hm[l], m.Whh[l], b.r, B, Hp / 64, G, t * B, 0};
        CU(igemm_tma_launch<LGemmK>(q, dim3(cdiv_(B, 128), G / 64), st), "lstm recurrent gemm"); }
      const float* cprev = t == 0 ? b.c_init + (size_t)l * B * Hp : b.cseq[l] + (size_t)(t - 1) * B * Hp;
      lstm_cell_fwd_kernel<<<cell_blocks, 256, 0, st>>>(
          b.gx + (size_t)t * B * G, b.r, w8[4 * l + 2], w8[4 * l + 3], cprev, done + (size_t)t * B, t + 1 < T1 ? done + (size_t)(t + 1) * B : nullptr, B,
          H, Hp, b.gates[l] + (size_t)t * B * G, b.cseq[l] + (size_t)t * B * Hp, b.hseq[l] + (size_t)t * B * Hp, b.hbf[l] + (size_t)t * B * Hp,
          t + 1 < T1 ? b.hm[l] + (size_t)(t + 1) * B * Hp : nullptr);
    }
    CU(cudaGetLastError(), "lstm cell");
  }
  lstm_unpad_rows_kernel<<<cdiv_(N1 * H, 256), 256, 0, st>>>(b.hseq[1], (int)N1, H, Hp, out);
  for (int l = 0; l < 2; ++l) {
    if (hT) CU(cudaMemcpy2DAsync(hT + (size_t)l * B * H, H * 4, b.hseq[l] + (size_t)(T1 - 1) * B * Hp, Hp * 4, H * 4, B, cudaMemcpyDeviceToDevice, st), "hT");
    if (cT) CU(cudaMemcpy2DAsync(cT + (size_t)l * B * H, H * 4, b.cseq[l] + (size_t)(T1 - 1) * B * Hp, Hp * 4, H * 4, B, cudaMemcpyDeviceToDevice, st), "cT");
  }
  CU(cudaGetLastError(), "lstm forward");
  return 0;
}

// BPTT over the first d.NB rows (steps 0 .. NB/B - 1) of the forward that filled b: dout f32 [NB][H] -> dcore f32 [NB][H]; the weight and
// bias gradients are ACCUMULATED into g8.  dhT / dcT f32 [2][B][H] (NULL: zero) seed the last step: dhT[l] is added to that step's dh
// unmasked, dcT[l] is its incoming cell-state carry.  dh0 / dc0 f32 [2][B][H] (NULL: not wanted) receive the gradient of the initial state.
static int lstm_backward_rows(const LstmDims& d, const LstmBuffers& b, const LstmMaps& m, float* const* g8, const uint8_t* done, const float* dout,
                              const float* dhT, const float* dcT, float* dcore, float* dh0, float* dc0, cudaStream_t st) {
  const int B = d.B, H = d.H, Hp = d.Hp, G = d.G;
  const int64_t NB = d.NB;
  const int steps = (int)(NB / B);
  const int cell_blocks = cdiv_((int64_t)B * Hp, 256);
  // dh_out of the top layer, padded to Hp (dx is the padded buffer)
  CU(cudaMemsetAsync(b.dx, 0, NB * Hp * 4, st), "zero dx");
  CU(cudaMemcpy2DAsync(b.dx, Hp * 4, dout, H * 4, H * 4, NB, cudaMemcpyDeviceToDevice, st), "pad dout");
  for (int l = 1; l >= 0; --l) {
    if (dcT) CU(cudaMemcpy2DAsync(b.dc, Hp * 4, dcT + (size_t)l * B * H, H * 4, H * 4, B, cudaMemcpyDeviceToDevice, st), "dcT copy");
    else CU(cudaMemsetAsync(b.dc, 0, (size_t)B * Hp * 4, st), "zero dc");
    if (dhT) CU(cudaMemcpy2DAsync(b.dhm, Hp * 4, dhT + (size_t)l * B * H, H * 4, H * 4, B, cudaMemcpyDeviceToDevice, st), "dhT copy");
    for (int t = steps - 1; t >= 0; --t) {
      const bool last = t + 1 == steps;
      const float* cprev = t == 0 ? b.c_init + (size_t)l * B * Hp : b.cseq[l] + (size_t)(t - 1) * B * Hp;
      lstm_cell_bwd_kernel<<<cell_blocks, 256, 0, st>>>(
          b.dx + (size_t)t * B * Hp, last && !dhT ? nullptr : b.dhm, last ? nullptr : done + (size_t)(t + 1) * B, b.gates[l] + (size_t)t * B * G,
          b.cseq[l] + (size_t)t * B * Hp, cprev, done + (size_t)t * B, b.dc, B, H, Hp, b.dgates[l] + (size_t)t * B * G);
      if (t > 0 || dh0) {   // dhm_t = dgates_t . Whh  (gradient w.r.t. m_t . h_{t-1})
        LGemmK::Params q{m.dg128[l], m.WhhT[l], b.dhm, B, G / 64, Hp, t * B, 0};
        CU(igemm_tma_launch<LGemmK>(q, dim3(cdiv_(B, 128), Hp / 64), st), "lstm bwd recurrent gemm");
      }
    }
    CU(cudaGetLastError(), "lstm cell bwd");
    if (dh0) lstm_unpad_masked_kernel<<<cdiv_((int64_t)B * H, 256), 256, 0, st>>>(b.dhm, done, B, H, Hp, dh0 + (size_t)l * B * H);
    if (dc0) lstm_unpad_rows_kernel<<<cdiv_((int64_t)B * H, 256), 256, 0, st>>>(b.dc, B, H, Hp, dc0 + (size_t)l * B * H);
    // weight gradients over all NB rows (MN-major operands), then un-pad + accumulate
    { LGemmMN::Params q{m.dg64[l], m.xin64[l], b.dwpad, (int)NB, Hp};
      CU(igemm_tma_launch<LGemmMN>(q, dim3(G / 128, Hp / 64), st), "lstm dWih gemm");
      lstm_unpad_w_kernel<<<cdiv_((int64_t)4 * H * H, 256), 256, 0, st>>>(b.dwpad, H, Hp, g8[4 * l]); }
    { LGemmMN::Params q{m.dg64[l], m.hm64[l], b.dwpad, (int)NB, Hp};
      CU(igemm_tma_launch<LGemmMN>(q, dim3(G / 128, Hp / 64), st), "lstm dWhh gemm");
      lstm_unpad_w_kernel<<<cdiv_((int64_t)4 * H * H, 256), 256, 0, st>>>(b.dwpad, H, Hp, g8[4 * l + 1]); }
    { const int chunks = cdiv_(NB, LSTM_BIAS_CHUNK);
      lstm_bias_part_kernel<<<dim3(cdiv_(G, 128), chunks), 128, 0, st>>>(b.dgates[l], (int)NB, G, b.bias_part);
      lstm_bias_sum_kernel<<<cdiv_((int64_t)4 * H, 256), 256, 0, st>>>(b.bias_part, chunks, H, Hp, g8[4 * l + 2], g8[4 * l + 3]); }
    // gradient w.r.t. this layer's input = dh_out of the layer below (or dcore)
    { LGemmK::Params q{m.dg128[l], m.WihT[l], b.dx, (int)NB, G / 64, Hp, 0, 0};
      CU(igemm_tma_launch<LGemmK>(q, dim3(cdiv_(NB, 128), Hp / 64), st), "lstm dx gemm"); }
  }
  lstm_unpad_rows_kernel<<<cdiv_(NB * H, 256), 256, 0, st>>>(b.dx, (int)NB, H, Hp, dcore);
  CU(cudaGetLastError(), "lstm backward");
  return 0;
}
}  // namespace srl

// ------------------------------------------------------------------------------------------------ learner context
struct srl_lstm {
  LstmDims d;                // backward over the first T = T1 - 1 steps
  const float* w[8];         // weight_ih, weight_hh, bias_ih, bias_hh per layer (fp32, PyTorch layouts, caller-owned)
  float* g[8];               // gradients (same layouts), accumulated
  char* arena;               // every row of lstm_rows
  LstmBuffers b;
  LstmMaps m;
};

extern "C" int srl_lstm_create(int T1, int B, int H, const float* const* weights8, float* const* grads8, srl_lstm_t** out) {
  REQ(T1 >= 2 && B >= 1 && H >= 1 && weights8 && grads8 && out, "lstm_create: bad argument");
  srl_lstm* L = new (std::nothrow) srl_lstm();
  REQ(L, "out of memory");
  L->d = lstm_dims(T1, B, H, (int64_t)(T1 - 1) * B);
  for (int i = 0; i < 8; ++i) { L->w[i] = weights8[i]; L->g[i] = grads8[i]; }
  WsRow t[LSTM_ROWS];
  lstm_rows(L->b, L->d, t);
  const int64_t total = rows_bytes(t, LSTM_ROWS, false);
  if (cudaMalloc(&L->arena, total) != cudaSuccess || cudaMemset(L->arena, 0, total) != cudaSuccess) { delete L; return fail(SRL_EINVAL, "lstm_create: cudaMalloc failed"); }
  carve_rows(t, LSTM_ROWS, false, L->arena);
  if (!lstm_maps(L->b, L->d, &L->m)) { cudaFree(L->arena); delete L; return fail(SRL_EINVAL, "lstm_create: tensor map creation failed"); }
  *out = L;
  return 0;
}
extern "C" int srl_lstm_destroy(srl_lstm_t* L) { if (L) { cudaFree(L->arena); delete L; } return 0; }

extern "C" int srl_lstm_forward(srl_lstm_t* L, const float* core, const uint8_t* done, const float* h0, const float* c0, float* out,
                                float* hT, float* cT, void* stream) {
  REQ(L && core && done && h0 && c0 && out, "lstm_forward: NULL pointer");
  return lstm_forward_rows(L->d, L->b, L->m, L->w, core, done, h0, c0, out, hT, cT, (cudaStream_t)stream);
}

extern "C" int srl_lstm_backward(srl_lstm_t* L, const float* dout, const uint8_t* done, float* dcore, void* stream) {
  REQ(L && dout && done && dcore, "lstm_backward: NULL pointer");
  return lstm_backward_rows(L->d, L->b, L->m, L->g, done, dout, nullptr, nullptr, dcore, nullptr, nullptr, (cudaStream_t)stream);
}

extern "C" int srl_lstm_debug_buffer(srl_lstm_t* L, const char* name, int layer, void** ptr, int64_t* count) {
  REQ(L && name && ptr && count, "lstm_debug_buffer: NULL argument");
  LstmBuffers b = {};
  WsRow t[LSTM_ROWS];
  lstm_rows(b, L->d, t);
  carve_rows(t, LSTM_ROWS, false, L->arena);          // the same table and arena as srl_lstm_create: the same addresses
  return lstm_find_row(t, name, layer, ptr, count, "lstm_debug_buffer");
}

// ------------------------------------------------------------------------------------------------ stand-alone core on caller-owned blocks
static int check_core_shape(int T1, int B, int A, const char* what) {
  REQ(T1 >= 1 && B >= 1 && (int64_t)T1 * B <= MAX_FRAMES, "%s: T1=%d B=%d: need T1 >= 1, B >= 1 and T1*B <= %d", what, T1, B, MAX_FRAMES);
  REQ(A >= 1 && A <= 31, "%s: A=%d must be in [1, 31]", what, A);
  return 0;
}

extern "C" int srl_lstm_core_sizes(int T1, int B, int A, int64_t* saved_bytes, int64_t* scratch_bytes) {
  REQ(saved_bytes && scratch_bytes, "lstm_core_sizes: NULL argument");
  int rc = check_core_shape(T1, B, A, "lstm_core_sizes");
  if (rc) return rc;
  LstmBuffers b = {};
  WsRow t[LSTM_ROWS];
  lstm_rows(b, lstm_dims(T1, B, 513 + A, (int64_t)T1 * B), t);
  block_bytes(t, LSTM_ROWS, LSTM_SAVED_ROWS, false, saved_bytes, scratch_bytes);
  return 0;
}

static int64_t lstm_tensor_bytes(int i, int H) { return (i % 4 < 2 ? (int64_t)4 * H * H : (int64_t)4 * H) * 4; }

// the checks both calls share: shape, the blocks' alignment and sizes
static int check_core_call(int T1, int B, int A, const void* saved, const void* scratch, int64_t* sb, int64_t* kb, const char* what) {
  int rc = check_core_shape(T1, B, A, what);
  if (rc) return rc;
  REQ(!misaligned(saved, 256) && !misaligned(scratch, 256), "%s: saved and scratch must be 256-byte aligned", what);
  return srl_lstm_core_sizes(T1, B, A, sb, kb);
}

// host arithmetic only (no CUDA call): the blocks are carved as core_call_setup carves them
extern "C" int srl_lstm_core_debug_buffer(int T1, int B, int A, void* saved, void* scratch, const char* name, int layer, void** ptr,
                                          int64_t* count) {
  REQ(saved && scratch && name && ptr && count, "lstm_core_debug_buffer: NULL argument");
  int64_t sb = 0, kb = 0;
  const int rc = check_core_call(T1, B, A, saved, scratch, &sb, &kb, "lstm_core_debug_buffer");
  if (rc) return rc;
  LstmBuffers b = {};
  WsRow t[LSTM_ROWS];
  lstm_rows(b, lstm_dims(T1, B, 513 + A, (int64_t)T1 * B), t);
  carve_rows(t, LSTM_SAVED_ROWS, false, static_cast<char*>(saved));
  carve_rows(t + LSTM_SAVED_ROWS, LSTM_ROWS - LSTM_SAVED_ROWS, false, static_cast<char*>(scratch));
  return lstm_find_row(t, name, layer, ptr, count, "lstm_core_debug_buffer");
}

// the blocks of one call -> the buffers and their tensor maps, encoded on the host for this call (legal under stream capture)
static int core_call_setup(const LstmDims& d, void* saved, void* scratch, LstmBuffers* b, LstmMaps* m, const char* what) {
  WsRow t[LSTM_ROWS];
  *b = LstmBuffers{};
  lstm_rows(*b, d, t);
  CU(carve_blocks(t, LSTM_ROWS, LSTM_SAVED_ROWS, false, saved, scratch), "cudaSetDevice");
  if (!lstm_maps(*b, d, m)) return fail(SRL_ESTATE, "%s: tensor map creation failed (driver without cuTensorMapEncodeTiled?)", what);
  pdl_set_active(true);
  return 0;
}

extern "C" int srl_lstm_core_forward(const float* core, const uint8_t* done, const float* h0, const float* c0, int A, int T1, int B,
                                     const float* const* weights8, void* saved, void* scratch, float* out, float* hT, float* cT, void* stream) {
  REQ(core && done && h0 && c0 && weights8 && saved && scratch && out && hT && cT, "lstm_core_forward: NULL pointer");
  for (int i = 0; i < 8; ++i) REQ(weights8[i], "lstm_core_forward: weights8[%d] is NULL", i);
  int64_t sb = 0, kb = 0;
  int rc = check_core_call(T1, B, A, saved, scratch, &sb, &kb, "lstm_core_forward");
  if (rc) return rc;
  const int H = 513 + A;
  const int64_t N1 = (int64_t)T1 * B, rows = N1 * H * 4, state = (int64_t)2 * B * H * 4;
  Span s[17] = {{core, rows, false, "core"}, {done, N1, false, "done"}, {h0, state, false, "h0"}, {c0, state, false, "c0"}};
  int n = 4;
  for (int i = 0; i < 8; ++i) s[n++] = {weights8[i], lstm_tensor_bytes(i, H), false, kW8[i]};
  s[n++] = {saved, sb, true, "saved"}; s[n++] = {scratch, kb, true, "scratch"};
  s[n++] = {out, rows, true, "out"}; s[n++] = {hT, state, true, "hT"}; s[n++] = {cT, state, true, "cT"};
  rc = check_spans(s, n, "lstm_core_forward");
  if (rc) return rc;
  const LstmDims d = lstm_dims(T1, B, H, N1);
  LstmBuffers b;
  LstmMaps m;
  rc = core_call_setup(d, saved, scratch, &b, &m, "lstm_core_forward");
  if (rc) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  CU(cudaMemcpyAsync(b.done, done, N1, cudaMemcpyDeviceToDevice, st), "done copy");
  return lstm_forward_rows(d, b, m, weights8, core, b.done, h0, c0, out, hT, cT, st);
}

extern "C" int srl_lstm_core_backward(const float* dout, const float* dhT, const float* dcT, int A, int T1, int B, void* saved, void* scratch,
                                      float* const* grads8, float* dcore, float* dh0, float* dc0, void* stream) {
  REQ(dout && saved && scratch && grads8 && dcore, "lstm_core_backward: NULL pointer");
  for (int i = 0; i < 8; ++i) REQ(grads8[i], "lstm_core_backward: grads8[%d] is NULL", i);
  int64_t sb = 0, kb = 0;
  int rc = check_core_call(T1, B, A, saved, scratch, &sb, &kb, "lstm_core_backward");
  if (rc) return rc;
  const int H = 513 + A;
  const int64_t N1 = (int64_t)T1 * B, rows = N1 * H * 4, state = (int64_t)2 * B * H * 4;
  Span s[16] = {{dout, rows, false, "dout"}, {dhT, state, false, "dhT"}, {dcT, state, false, "dcT"}, {saved, sb, false, "saved"},
                {scratch, kb, true, "scratch"}};
  int n = 5;
  for (int i = 0; i < 8; ++i) s[n++] = {grads8[i], lstm_tensor_bytes(i, H), true, kG8[i]};
  s[n++] = {dcore, rows, true, "dcore"}; s[n++] = {dh0, state, true, "dh0"}; s[n++] = {dc0, state, true, "dc0"};
  rc = check_spans(s, n, "lstm_core_backward");
  if (rc) return rc;
  const LstmDims d = lstm_dims(T1, B, H, N1);
  LstmBuffers b;
  LstmMaps m;
  rc = core_call_setup(d, saved, scratch, &b, &m, "lstm_core_backward");
  if (rc) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  for (int i = 0; i < 8; ++i) CU(cudaMemsetAsync(grads8[i], 0, lstm_tensor_bytes(i, H), st), "zero grads8");     // overwritten, not accumulated
  return lstm_backward_rows(d, b, m, grads8, b.done, dout, dhT, dcT, dcore, dh0, dc0, st);
}

// ------------------------------------------------------------------------------------------------ actor step: host side
namespace srl {
struct LstmStep {
  int B, H;
  const float* w[2][4];               // weight_ih, weight_hh, bias_ih, bias_hh per layer (fp32, caller-owned)
  __nv_bfloat16 *wp, *xh;             // packed weights [2][4Hp][2Hp]; operands [2][B][2Hp]
  alignas(64) CUtensorMap m_w, m_xh[2];
};

int lstm_step_create(int B, int H, const float* const* weights8, LstmStep** out) {
  *out = nullptr;
  REQ(B >= 1 && H >= 1 && (H + 63) / 64 * 64 == LS_HP, "lstm_step: H must be 513 + A with A in [1, 31]");
  LstmStep* S = new (std::nothrow) LstmStep();
  REQ(S, "out of host memory");
  S->B = B; S->H = H;
  for (int l = 0; l < 2; ++l) for (int k = 0; k < 4; ++k) S->w[l][k] = weights8[4 * l + k];
  const size_t wbytes = (size_t)2 * LS_G * LS_K * 2, xbytes = (size_t)2 * B * LS_K * 2;
  char* a = nullptr;
  cudaError_t e = cudaMalloc(&a, wbytes + xbytes);
  if (e == cudaSuccess) e = cudaMemset(a, 0, wbytes + xbytes);      // the operands' padding columns stay zero from here on
  if (e != cudaSuccess) { if (a) cudaFree(a); delete S; return cuda_fail(e, "lstm_step: cudaMalloc"); }
  S->wp = (__nv_bfloat16*)a; S->xh = (__nv_bfloat16*)(a + wbytes);
  const uint64_t dw[2] = {LS_K, 2 * LS_G}, dx[2] = {LS_K, (uint64_t)B}, st[1] = {LS_K};
  const uint32_t box[2] = {64, 128};
  if (!make_map(&S->m_w, S->wp, 2, dw, st, box) || !make_map(&S->m_xh[0], S->xh, 2, dx, st, box) ||
      !make_map(&S->m_xh[1], S->xh + (size_t)B * LS_K, 2, dx, st, box)) {
    cudaFree(a); delete S; return fail(SRL_ESTATE, "lstm_step: tensor map creation failed");
  }
  *out = S;
  return 0;
}
void lstm_step_destroy(LstmStep* S) { if (S) { cudaFree(S->wp); delete S; } }

cudaError_t lstm_step_pack(LstmStep* S, cudaStream_t st) {
  lstm_step_pack_kernel<<<cdiv_((int64_t)2 * LS_G * LS_K, 256), 256, 0, st>>>(S->w[0][0], S->w[0][1], S->w[1][0], S->w[1][1], S->H, S->wp);
  return cudaGetLastError();
}

template <int KS>
static cudaError_t launch_step_layer(const LstmStepParams& p, int ntiles, cudaStream_t st) {
  static PerDeviceOnce once;
  cudaError_t e = ensure_max_dynamic_smem(once, lstm_step_kernel<KS>, LS_SMEM);
  if (e != cudaSuccess) return e;
  return launch_chain(lstm_step_kernel<KS>, dim3(LS_G / 128, ntiles, KS), dim3(LS_THREADS), LS_SMEM, st, p);
}

bool lstm_step_ksplit_supported(int ks) { return ks == 1 || ks == 2 || ks == 3 || ks == 6; }

cudaError_t lstm_step_forward(LstmStep* S, const float* core, const uint8_t* done, const float* h_in, const float* c_in, float* h_out,
                              float* c_out, int ksplit, cudaStream_t st) {
  const int B = S->B, H = S->H;
  lstm_step_prep_kernel<<<cdiv_((int64_t)B * LS_HP, 256), 256, 0, st>>>(core, done, h_in, B, H, S->xh);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  for (int l = 0; l < 2; ++l) {
    LstmStepParams p;
    p.w = S->m_w; p.xh = S->m_xh[l];
    p.b_ih = S->w[l][2]; p.b_hh = S->w[l][3];
    p.c_in = c_in + (size_t)l * B * H; p.done = done;
    p.c_out = c_out + (size_t)l * B * H; p.h_out = h_out + (size_t)l * B * H;
    p.x_next = l == 0 ? S->xh + (size_t)B * LS_K : nullptr;
    p.N = B; p.H = H; p.w_row0 = l * LS_G;
    const int nt = cdiv_(B, LS_BN);
    switch (ksplit) {
      case 1: e = launch_step_layer<1>(p, nt, st); break;
      case 2: e = launch_step_layer<2>(p, nt, st); break;
      case 3: e = launch_step_layer<3>(p, nt, st); break;
      case 6: e = launch_step_layer<6>(p, nt, st); break;
      default: e = cudaErrorInvalidValue;
    }
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

void lstm_step_buffers(const LstmStep* S, void** xh, int64_t* nxh, void** w, int64_t* nw) {
  *xh = S ? S->xh : nullptr; *nxh = S ? (int64_t)2 * S->B * LS_K : 0;
  *w = S ? S->wp : nullptr; *nw = (int64_t)2 * LS_G * LS_K;
}
}  // namespace srl
