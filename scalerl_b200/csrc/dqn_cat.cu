// The categorical (C51) Q head of the Ape-X learner step, fp32 on the CUDA cores (Bellemare et al. 2017; the arithmetic per atom is
// dqn_cat.cuh's, shared with the Ape-X actor):
//   cat_gemm_kernel<false>  the logits [N][A K] = h W^T + b: a tiled, register-blocked SIMT GEMM (a head of up to 31 x 64 = 1,984 rows
//                           is read once per tile, not once per transition)
//   cat_gemm_kernel<true>   the head gradients gW = dlogits^T h, gb = dlogits^T 1: the same GEMM with each CTA running over every
//                           transition in order, so the sum over transitions has a fixed order and needs no partial buffers
//   cat_tail_kernel         per transition: Q of the target (or, double DQN, the online) network at s', a*, the projection of
//                           p_target(s')[a*], the cross-entropy, the KL priority, the loss through the ticket reduction, the dense
//                           dlogits row and the dcore row of the encoder backward
// dqn.cu's launchers call these for the categorical head (its q values: dqn.cu's q_values_kernel on the logits).
// Every logit is one fmaf chain over j = 0 .. 511 from 0, then + bias rounded once; every other sum has a fixed order: eager, captured
// and repeated runs compute the same bits, and no float atomics are used.
#include "common.cuh"
#include "dqn_cat.cuh"
#include "kernels.h"

namespace srl {

// C[m][c] = sum_k A(m, k) B(k, c), one fmaf chain per output over ascending k, 64 x 64 tiles, 16 k per stage, 256 threads of 4 x 4
// outputs each.  WGRAD = false: m = frame (core rows, stride ENC_CORE, h = columns < 512), c = logit row of W [R][512], k = j < 512;
// out [M][R] = C + b.  WGRAD = true: m = logit row r < R, c = column j of [h | 1] (j = 512: the bias), k = transition n < Kdim;
// out = gW [R][512], gb [R].
constexpr int CG_BM = 64, CG_BN = 64, CG_BK = 16, CG_PAD = 4;
struct CatGemm {
  const float *core, *W, *b, *dl;
  int M, Ncol, Kdim;
  float *out, *gb;
};
template <bool WGRAD>
__global__ void __launch_bounds__(256) cat_gemm_kernel(const CatGemm g) {
  __shared__ __align__(16) float As[CG_BK][CG_BM + CG_PAD];
  __shared__ __align__(16) float Bs[CG_BK][CG_BN + CG_PAD];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * CG_BM, c0 = blockIdx.x * CG_BN;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < g.Kdim; k0 += CG_BK) {
    if constexpr (!WGRAD) {
      // 64 core rows and 64 weight rows, 16 columns each, stored k-major: 4 consecutive k per thread (two 8-byte loads: core rows
      // are 8-byte aligned only)
      const int r = tid >> 2, kq = (tid & 3) * 4;
      float2 a0 = make_float2(0.f, 0.f), a1 = a0, b0 = a0, b1 = a0;
      if (m0 + r < g.M) {
        const float2* p = reinterpret_cast<const float2*>(g.core + (size_t)(m0 + r) * ENC_CORE + k0 + kq);
        a0 = __ldg(p); a1 = __ldg(p + 1);
      }
      if (c0 + r < g.Ncol) {
        const float2* p = reinterpret_cast<const float2*>(g.W + (size_t)(c0 + r) * 512 + k0 + kq);
        b0 = __ldg(p); b1 = __ldg(p + 1);
      }
      As[kq][r] = a0.x; As[kq + 1][r] = a0.y; As[kq + 2][r] = a1.x; As[kq + 3][r] = a1.y;
      Bs[kq][r] = b0.x; Bs[kq + 1][r] = b0.y; Bs[kq + 2][r] = b1.x; Bs[kq + 3][r] = b1.y;
    } else {
      // transition n = k0 + k: 4 consecutive logit rows of its dlogits row and 4 consecutive columns of [h | 1]; zero past the ends
      const int k = tid >> 4, q = (tid & 15) * 4, n = k0 + k;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = m0 + q + i, j = c0 + q + i;
        As[k][q + i] = n < g.Kdim && r < g.M ? __ldg(g.dl + (size_t)n * g.M + r) : 0.f;
        Bs[k][q + i] = n < g.Kdim ? (j < 512 ? __ldg(g.core + (size_t)n * ENC_CORE + j) : (j == 512 ? 1.f : 0.f)) : 0.f;
      }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < CG_BK; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= g.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = c0 + tx * 4 + j;
      if (c >= g.Ncol) continue;
      if constexpr (!WGRAD) g.out[(size_t)m * g.Ncol + c] = __fadd_rn(acc[i][j], __ldg(g.b + c));
      else if (c < 512) g.out[(size_t)m * 512 + c] = acc[i][j];
      else g.gb[m] = acc[i][j];
    }
  }
}

// One warp per transition, 4 per block: on = the online head.  scratch: [0] the ticket, [4 + k] block k's partial of sum_n w_n ce_n
// (dqn_head.cuh's tail_loss).
__global__ void __launch_bounds__(128) cat_tail_kernel(const QHead on, const QTail t, float inv_B) {
  __shared__ float sm[4][CAT_MAX_ATOMS], sd[4][CAT_MAX_ATOMS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = blockIdx.x * 4 + warp;
  float l = 0.f;
  if (n < t.B) {
    const int K = on.c.K, R = on.R;
    const int act = ld_action(t.action + n, on.A);
    const float w = t.weight ? __ldg(t.weight + n) : 1.f;
    float *m = sm[warp], *d = sd[warp];
    const CatLoss r = cat_transition(t.logits_s + (size_t)n * R + (size_t)act * K, t.core_n ? t.logits_n + (size_t)n * R : nullptr,
                                     t.logits_nt + (size_t)n * R, on.A, __ldg(t.reward + n), t.done[n] ? 0.f : t.gamma, on.c, lane, m,
                                     __fmul_rn(w, inv_B), d);
    if (lane == 0) {
      l = __fmul_rn(w, r.ce);
      t.q[n] = r.q; t.y[n] = r.y; t.ce[n] = r.ce;
      t.prio[n] = cat_priority(r.kl, t.priority_eps);
    }
    for (int k = lane; k < K; k += 32) t.m[(size_t)n * K + k] = m[k];
    float* dl = t.dlogits + (size_t)n * R;
    for (int c = lane; c < R; c += 32) {
      const int k = c - act * K;
      dl[c] = k >= 0 && k < K ? d[k] : 0.f;
    }
    // dL/dh = sum_k dlogit_k W[act K + k], k ascending
    float acc[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = 0.f;
    for (int k = 0; k < K; ++k) {
      const float dk = d[k];
      const float* wr = on.W + (size_t)(act * K + k) * 512;
#pragma unroll
      for (int i = 0; i < 16; ++i) acc[i] = fmaf(dk, __ldg(wr + lane + 32 * i), acc[i]);
    }
    float* dc = t.dcore + (size_t)n * ENC_CORE;
#pragma unroll
    for (int i = 0; i < 16; ++i) dc[lane + 32 * i] = acc[i];
    if (lane < ENC_CORE - 512) dc[512 + lane] = 0.f;
  }
  tail_loss(l, t.B, t.scratch, t.loss);
}

cudaError_t launch_cat_logits(const float* core, const float* W, const float* b, int N, int R, float* logits, cudaStream_t st) {
  CatGemm g = {core, W, b, nullptr, N, R, 512, logits, nullptr};
  cat_gemm_kernel<false><<<dim3((R + CG_BN - 1) / CG_BN, (N + CG_BM - 1) / CG_BM), 256, 0, st>>>(g);
  return cudaGetLastError();
}
cudaError_t launch_cat_wgrad(const float* dlogits, const float* core, int N, int R, float* gW, float* gb, cudaStream_t st) {
  CatGemm g = {core, nullptr, nullptr, dlogits, R, 513, N, gW, gb};
  cat_gemm_kernel<true><<<dim3((513 + CG_BN - 1) / CG_BN, (R + CG_BM - 1) / CG_BM), 256, 0, st>>>(g);
  return cudaGetLastError();
}
// the three logit sets (s and s' under the online head, s' under the target head), then the projection / cross-entropy tail
cudaError_t launch_cat_tail(const QHead& on, const QHead& tg, const QTail& t, cudaStream_t st) {
  cudaError_t e = launch_cat_logits(t.core_s, on.W, on.b, t.B, on.R, t.logits_s, st);
  if (e == cudaSuccess && t.core_n) e = launch_cat_logits(t.core_n, on.W, on.b, t.B, on.R, t.logits_n, st);
  if (e == cudaSuccess) e = launch_cat_logits(t.core_nt, tg.W, tg.b, t.B, tg.R, t.logits_nt, st);
  if (e != cudaSuccess) return e;
  cat_tail_kernel<<<dqn_tail_blocks(t.B), 128, 0, st>>>(on, t, 1.f / (float)t.B);
  return cudaGetLastError();
}

}  // namespace srl
