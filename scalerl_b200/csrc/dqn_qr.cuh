// The quantile (QR-DQN) Q head's device arithmetic (Dabney et al. 2018, "Distributional Reinforcement Learning with Quantile
// Regression"), shared by the learner's tail (dqn_qr.cu) and the Ape-X actor (apex_actor.cu), so that an actor's Q values, greedy
// actions and initial priorities are the learner's bits for the same weights and quantiles.
// The head q = Linear(512, A N) writes N quantiles per action: row a N + i of a frame's row is theta_{a,i}, quantile i of action a at
// the midpoint tau^_i = (2 i + 1) / (2 N).  For one transition with the taken action a and the target action a*:
//   Q(s, a)   = (sum_i theta_{a,i}) / N
//   T_j       = r + g theta'_{a*,j}   (g = gamma (1 - d); g = 0: T_j = r and s' is not read)
//   u_ij      = T_j - theta_{a,i},  L(u) = u^2 / 2 if |u| <= kappa, else kappa (|u| - kappa / 2)
//   loss      = (1 / N) sum_i sum_j |tau^_i - 1{u_ij < 0}| L(u_ij) / kappa
//   dtheta_i  = -(w / B) (1 / N) sum_j |tau^_i - 1{u_ij < 0}| clamp(u_ij, -kappa, kappa) / kappa
// The order of every sum, the same in the learner and the actor (no contraction, no float atomics):
//   Q and y = (sum_j T_j) / N: ascending index from 0, then one IEEE division by N;
//   per online quantile i: S_i = sum_j |tau^_i - 1{u_ij < 0}| L(u_ij) and G_i = sum_j |tau^_i - 1{u_ij < 0}| clamp(u_ij), j ascending;
//   loss: lane l adds S_i for i = l, l + 32, ... in that order, then warp_sum's xor butterfly; then / kappa, then / N;
//   dtheta_i = -(wB (G_i / (kappa N))), kappa N rounded once.
#pragma once
#include "common.cuh"
#include "dqn_head.cuh"
#include "kernels.h"

namespace srl {

constexpr int QR_PER_LANE = QR_MAX_QUANTILES / 32;     // online quantiles per lane

SRL_DEVINL float qr_tau(int i, int N) { return __fdiv_rn((float)(2 * i + 1), (float)(2 * N)); }

// Q = (sum_i x_i) / N of one action's N quantiles
SRL_DEVINL float qr_q(const float* __restrict__ x, int N) {
  float s = 0.f;
  for (int i = 0; i < N; ++i) s = __fadd_rn(s, __ldg(x + i));
  return __fdiv_rn(s, (float)N);
}
// the Q row of one frame's A N quantiles, one action per lane (lane a < A: Q_a; other lanes 0): q_row_max takes its first argmax
SRL_DEVINL float qr_q_lane(const float* __restrict__ row, int A, int N, int lane) {
  return lane < A ? qr_q(row + (size_t)lane * N, N) : 0.f;
}

// loss + eps in double (the loss is a sum of non-negative terms: no clamp); a NaN loss stays NaN (the replay add counts it)
SRL_DEVINL double qr_priority(float loss, float eps) { return (double)loss + (double)eps; }

struct QrLoss {
  float loss;    // (1 / N) sum_i sum_j rho_ij
  float q;       // Q(s, a)
  float y;       // (sum_j T_j) / N
};
// One transition on one warp; every lane calls it.  xs: the online quantiles of s at the taken action (N floats); xt: the target
// network's A N quantiles of s'; a* = the first argmax of Q_target(s') or, with xn (double DQN: the online network's quantiles of s'),
// of Q_online(s').  tq (N floats of shared memory) <- the target quantiles T_j.  GRAD: d (N floats of shared memory) <- dtheta of wB
// loss.  loss is on every lane, q and y on lane 0; tq and d are visible to the warp on return.
template <bool GRAD>
SRL_DEVINL QrLoss qr_transition(const float* __restrict__ xs, const float* __restrict__ xn, const float* __restrict__ xt, int A, int N,
                                float reward, float g, float kappa, int lane, float* tq, float wB, float* d) {
  if (g != 0.f) {      // warp-uniform: one transition per warp
    int a_star;
    q_row_max(qr_q_lane(xn ? xn : xt, A, N, lane), A, &a_star);
    const float* t = xt + (size_t)a_star * N;
    for (int j = lane; j < N; j += 32) tq[j] = __fadd_rn(reward, __fmul_rn(g, __ldg(t + j)));
  } else {
    for (int j = lane; j < N; j += 32) tq[j] = reward;
  }
  __syncwarp();
  float th[QR_PER_LANE], tau[QR_PER_LANE], S[QR_PER_LANE], G[QR_PER_LANE];
#pragma unroll
  for (int k = 0; k < QR_PER_LANE; ++k) {
    const int i = lane + 32 * k;
    th[k] = i < N ? __ldg(xs + i) : 0.f;
    tau[k] = qr_tau(i, N);
    S[k] = 0.f;
    G[k] = 0.f;
  }
  const float half_kappa = __fmul_rn(0.5f, kappa);
  const int kn = (N - lane + 31) >> 5;      // this lane's quantiles
  for (int j = 0; j < N; ++j) {
    const float t = tq[j];
#pragma unroll
    for (int k = 0; k < QR_PER_LANE; ++k) {
      if (k >= kn) break;
      const float u = __fsub_rn(t, th[k]);
      const float wt = fabsf(__fsub_rn(tau[k], u < 0.f ? 1.f : 0.f));
      const float au = fabsf(u);
      const float L = au <= kappa ? __fmul_rn(0.5f, __fmul_rn(u, u)) : __fmul_rn(kappa, __fsub_rn(au, half_kappa));
      S[k] = __fadd_rn(S[k], __fmul_rn(wt, L));
      if (GRAD) G[k] = __fadd_rn(G[k], __fmul_rn(wt, fminf(fmaxf(u, -kappa), kappa)));
    }
  }
  float p = 0.f;
#pragma unroll
  for (int k = 0; k < QR_PER_LANE; ++k) p = __fadd_rn(p, S[k]);
  QrLoss r;
  r.loss = __fdiv_rn(__fdiv_rn(warp_sum(p), kappa), (float)N);
  if (GRAD) {
    const float kN = __fmul_rn(kappa, (float)N);
#pragma unroll
    for (int k = 0; k < QR_PER_LANE; ++k)
      if (k < kn) d[lane + 32 * k] = -__fmul_rn(wB, __fdiv_rn(G[k], kN));
  }
  r.q = 0.f;
  r.y = 0.f;
  if (lane == 0) {
    r.q = qr_q(xs, N);
    float s = 0.f;
    for (int j = 0; j < N; ++j) s = __fadd_rn(s, tq[j]);
    r.y = __fdiv_rn(s, (float)N);
  }
  __syncwarp();
  return r;
}

}  // namespace srl
