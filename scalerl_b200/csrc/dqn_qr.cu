// The quantile (QR-DQN) Q head of the Ape-X learner step, fp32 on the CUDA cores (Dabney et al. 2018; the arithmetic per transition
// is dqn_qr.cuh's, shared with the Ape-X actor):
//   dqn_cat.cu's cat_gemm_kernel<false>  the quantiles [N][A K] = h W^T + b of s, of s' under the target network and (double DQN) of s'
//                                        under the online network: generic in the head's rows R = A K
//   dqn_cat.cu's cat_gemm_kernel<true>   the head gradients gW = dtheta^T h, gb = dtheta^T 1 (launch_cat_wgrad)
//   qr_tail_kernel                       per transition: a*, the target quantiles, the quantile Huber loss, the priority, the loss
//                                        through the ticket reduction, the dense dtheta row and the dcore row of the encoder backward
// dqn.cu's launchers call these for the quantile head (its q values: dqn.cu's q_values_kernel on the quantiles).
// Every sum has a fixed order (dqn_qr.cuh): eager, captured and repeated runs compute the same bits, and no float atomics are used.
#include "common.cuh"
#include "dqn_qr.cuh"
#include "kernels.h"

namespace srl {

// One warp per transition, 4 per block: on = the online head.  scratch: [0] the ticket, [4 + k] block k's partial of sum_n w_n loss_n
// (dqn_head.cuh's tail_loss).  The per-warp target quantiles and dtheta live in shared memory (2 x 4 x 1 KB).
__global__ void __launch_bounds__(128) qr_tail_kernel(const QHead on, const QTail t, float inv_B) {
  __shared__ float st[4][QR_MAX_QUANTILES], sd[4][QR_MAX_QUANTILES];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = blockIdx.x * 4 + warp;
  float l = 0.f;
  if (n < t.B) {
    const int N = on.qr.N, R = on.R;
    const int act = ld_action(t.action + n, on.A);
    const float w = t.weight ? __ldg(t.weight + n) : 1.f;
    float *tq = st[warp], *d = sd[warp];
    const QrLoss r = qr_transition<true>(t.logits_s + (size_t)n * R + (size_t)act * N, t.core_n ? t.logits_n + (size_t)n * R : nullptr,
                                         t.logits_nt + (size_t)n * R, on.A, N, __ldg(t.reward + n), t.done[n] ? 0.f : t.gamma,
                                         on.qr.kappa, lane, tq, __fmul_rn(w, inv_B), d);
    if (lane == 0) {
      l = __fmul_rn(w, r.loss);
      t.q[n] = r.q; t.y[n] = r.y; t.ce[n] = r.loss;
      t.prio[n] = qr_priority(r.loss, t.priority_eps);
    }
    for (int j = lane; j < N; j += 32) t.m[(size_t)n * N + j] = tq[j];
    float* dl = t.dlogits + (size_t)n * R;
    for (int c = lane; c < R; c += 32) {
      const int i = c - act * N;
      dl[c] = i >= 0 && i < N ? d[i] : 0.f;
    }
    // dL/dh = sum_i dtheta_i W[act N + i], i ascending
    float acc[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) acc[k] = 0.f;
    for (int i = 0; i < N; ++i) {
      const float di = d[i];
      const float* wr = on.W + (size_t)(act * N + i) * 512;
#pragma unroll
      for (int k = 0; k < 16; ++k) acc[k] = fmaf(di, __ldg(wr + lane + 32 * k), acc[k]);
    }
    float* dc = t.dcore + (size_t)n * ENC_CORE;
#pragma unroll
    for (int k = 0; k < 16; ++k) dc[lane + 32 * k] = acc[k];
    if (lane < ENC_CORE - 512) dc[512 + lane] = 0.f;
  }
  tail_loss(l, t.B, t.scratch, t.loss);
}

// the three quantile sets (s and s' under the online head, s' under the target head), then the quantile Huber tail
cudaError_t launch_qr_tail(const QHead& on, const QHead& tg, const QTail& t, cudaStream_t st) {
  cudaError_t e = launch_cat_logits(t.core_s, on.W, on.b, t.B, on.R, t.logits_s, st);
  if (e == cudaSuccess && t.core_n) e = launch_cat_logits(t.core_n, on.W, on.b, t.B, on.R, t.logits_n, st);
  if (e == cudaSuccess) e = launch_cat_logits(t.core_nt, tg.W, tg.b, t.B, tg.R, t.logits_nt, st);
  if (e != cudaSuccess) return e;
  qr_tail_kernel<<<dqn_tail_blocks(t.B), 128, 0, st>>>(on, t, 1.f / (float)t.B);
  return cudaGetLastError();
}

}  // namespace srl
