// The Q-learning tail of the Ape-X / DQN learner step, fp32 on the CUDA cores (the Q head is 512 x A: no tensor-core work):
//   dqn_tail_kernel           q(s,a), the bootstrapped target y, priorities |q - y| + eps, the loss mean(w (q - y)^2) through the
//                             ticket reduction of the IMPALA tail, dq and the dcore rows of the encoder backward
//                             (apex/worker.py:148-157; dqn/dqn_agent.py:155-171)
//   dqn_wgrad_kernel /        the Q head's weight and bias gradients: slab-group partials added in group order (the order of
//   dqn_wgrad_reduce_kernel   heads.cu's head_wgrad kernels), so every run computes the same bits
//   q_values_kernel           the forward-only Q head (predict / get_action)
//   apex_soft_update_kernel   theta_t <- tau theta + (1 - tau) theta_t (dqn_agent.py:185-190, utils/model_utils.py:29-32)
// The Q head arithmetic (q_dot, q_max, dueling_q, q_row_max, the target and the priority) is dqn_head.cuh's, shared with the Ape-X actor.
// The tail and the head gradients are templates on the scalar heads: DUELING = the dueling head V + Adv - mean(Adv) on the shared fc
// output (Wang et al. 2016, eq. 9), whose A + 1 rows (the value row first) lie as one [(A + 1)][512] block.  launch_q_tail,
// launch_q_wgrad and launch_q_values are the one place that picks the kernels of a head; the categorical head's are dqn_cat.cu's, the
// quantile head's dqn_qr.cu's tail on dqn_cat.cu's GEMMs.
#include "common.cuh"
#include "dqn_cat.cuh"
#include "dqn_head.cuh"
#include "kernels.h"

namespace srl {

// One warp per transition, 4 per block: on, tg = the online and target heads.  scratch: [0] the ticket, [4 + k] block k's partial of
// sum_n w_n (q_n - y_n)^2.  DUELING: the dueling head (dqn_head.cuh's dueling_q) in place of q = Linear(512, A); the target, loss and
// priority are the same.
template <bool DUELING>
__global__ void __launch_bounds__(128) dqn_tail_kernel(const QHead on, const QHead tg, const QTail t, float two_over_B) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = blockIdx.x * 4 + warp;
  float l = 0.f;
  if (n < t.B) {
    const int act = ld_action(t.action + n, on.A);
    const float* hs = t.core_s + (size_t)n * ENC_CORE;
    float q, nx;
    float wsum[16];     // dueling: the advantage rows' column sums (lane + 32 i)
    if constexpr (!DUELING) {
      q = q_dot(hs, on.W + (size_t)act * 512, lane) + __ldg(on.b + act);
      const float* hn = t.core_nt + (size_t)n * ENC_CORE;
      int a_star;
      if (t.core_n) {     // double DQN: the online network picks a*, the target network values it (dqn_agent.py:155-160)
        q_max<2>(t.core_n + (size_t)n * ENC_CORE, on.W, on.b, on.A, lane, &a_star);
        nx = q_dot(hn, tg.W + (size_t)a_star * 512, lane) + __ldg(tg.b + a_star);
      } else {            // max_a Q_target(s', a) (apex/worker.py:149, dqn_agent.py:162-163)
        nx = q_max<2>(hn, tg.W, tg.b, on.A, lane, &a_star);
      }
    } else {            // the same statements on the dueling Q rows (lane a holds Q_a)
      q = __shfl_sync(0xffffffffu, dueling_q<true>(hs, on.W, on.b, on.ba, on.A, lane, wsum), act);
      const float qt = dueling_q<false>(t.core_nt + (size_t)n * ENC_CORE, tg.W, tg.b, tg.ba, on.A, lane, nullptr);
      int a_star;
      if (t.core_n) {
        q_row_max(dueling_q<false>(t.core_n + (size_t)n * ENC_CORE, on.W, on.b, on.ba, on.A, lane, nullptr), on.A, &a_star);
        nx = __shfl_sync(0xffffffffu, qt, a_star);
      } else {
        nx = q_row_max(qt, on.A, &a_star);
      }
    }
    const float y = td_target(__ldg(t.reward + n), t.gamma, nx, t.done[n] != 0);
    const float w = t.weight ? __ldg(t.weight + n) : 1.f;
    const float delta = __fsub_rn(q, y);
    l = __fmul_rn(w, __fmul_rn(delta, delta));
    // d loss / d q of mean(w (q - y)^2): the gradient flows through q only (y is detached)
    const float dq = two_over_B * w * delta;
    if (lane == 0) {
      t.q[n] = q; t.y[n] = y; t.dq[n] = dq;
      t.prio[n] = td_priority(delta, t.priority_eps);
    }
    if constexpr (!DUELING) {
      const float* wa = on.W + (size_t)act * 512;
      float* dc = t.dcore + (size_t)n * ENC_CORE;
      for (int j = lane; j < ENC_CORE; j += 32) dc[j] = j < 512 ? dq * __ldg(wa + j) : 0.f;
    } else {            // dL/dV = dq, dL/dAdv_a = dq (1[a = act] - 1/A): dL/dh = dq (w_v + W_adv[act] - mean_a W_adv[a])
      const float* wa = on.W + (size_t)(act + 1) * 512;
      float* dc = t.dcore + (size_t)n * ENC_CORE;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int j = lane + 32 * i;
        dc[j] = dq * __fsub_rn(__fadd_rn(__ldg(on.W + j), __ldg(wa + j)), __fdiv_rn(wsum[i], (float)on.A));
      }
      if (lane < ENC_CORE - 512) dc[512 + lane] = 0.f;
    }
  }
  tail_loss(l, t.B, t.scratch, t.loss);
}

// Q head weight/bias gradients: thread = one column j of h (j == 512 is the bias "ones" column), blockIdx.y = a group of consecutive
// slabs of transitions.  Plain head: row a of a slab carries dq only for the transition's action.  Dueling head (A + 1 rows, the
// value row first): row 0 carries dq, row 1 + a carries dq (1[a = act] - 1/A).  Each group writes part[group][row][j].
constexpr int DQN_SLAB = 16, DQN_MAX_A = 32;
template <bool DUELING>
__global__ void __launch_bounds__(128) dqn_wgrad_kernel(const float* __restrict__ dq, const int64_t* __restrict__ action,
                                                        const float* __restrict__ core, int N, int A, int slabs_per_group,
                                                        float* __restrict__ part) {
  __shared__ float sd[DQN_SLAB][DQN_MAX_A];
  const int R = DUELING ? A + 1 : A;          // head rows
  const int j = blockIdx.x * 128 + threadIdx.x;
  const int nslab = (N + DQN_SLAB - 1) / DQN_SLAB;
  const int s0 = blockIdx.y * slabs_per_group, s1 = min(nslab, s0 + slabs_per_group);
  float acc[DQN_MAX_A];
#pragma unroll
  for (int a = 0; a < DQN_MAX_A; ++a) acc[a] = 0.f;
  for (int sl = s0; sl < s1; ++sl) {
    const int n0 = sl * DQN_SLAB, cnt = min(DQN_SLAB, N - n0);
    __syncthreads();                 // the previous slab's shared rows have been read
    for (int i = threadIdx.x; i < DQN_SLAB * R; i += 128) {     // rows past the ragged end are zero
      const int r = i / R, a = i - r * R;
      if constexpr (!DUELING) {
        sd[r][a] = (r < cnt && ld_action(action + n0 + r, A) == a) ? __ldg(dq + n0 + r) : 0.f;
      } else {
        float g = 0.f;
        if (r < cnt) {
          const float d = __ldg(dq + n0 + r);
          g = a == 0 ? d : d * ((ld_action(action + n0 + r, A) == a - 1 ? 1.f : 0.f) - __fdiv_rn(1.f, (float)A));
        }
        sd[r][a] = g;
      }
    }
    __syncthreads();
    if (j > 512) continue;
    float c[DQN_SLAB];
#pragma unroll
    for (int r = 0; r < DQN_SLAB; ++r) c[r] = r < cnt ? (j < 512 ? __ldg(core + (size_t)(n0 + r) * ENC_CORE + j) : 1.f) : 0.f;
#pragma unroll
    for (int a = 0; a < DQN_MAX_A; ++a) {
      if (a >= R) break;
#pragma unroll
      for (int r = 0; r < DQN_SLAB; ++r) acc[a] = fmaf(sd[r][a], c[r], acc[a]);
    }
  }
  if (j > 512) return;
#pragma unroll
  for (int a = 0; a < DQN_MAX_A; ++a)
    if (a < R) part[((size_t)blockIdx.y * R + a) * 513 + j] = acc[a];
}
// sums the groups' partials in group order into the Q head gradients (stored, not accumulated); dueling: row 0's bias -> gb[0], row
// 1 + a's -> gba[a]
template <bool DUELING>
__global__ void __launch_bounds__(256) dqn_wgrad_reduce_kernel(const float* __restrict__ part, int groups, int A, float* __restrict__ gW,
                                                               float* __restrict__ gb, float* __restrict__ gba) {
  const int n = (DUELING ? A + 1 : A) * 513, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = 0.f;
  for (int g = 0; g < groups; ++g) s += __ldg(part + (size_t)g * n + i);
  const int a = i / 513, j = i - a * 513;
  if (j < 512) gW[(size_t)a * 512 + j] = s; else if (!DUELING || a == 0) gb[a] = s; else gba[a - 1] = s;
}

// q_out[n][a] = Q(rows[n])[a] (q_lane: core rows, or the categorical / quantile head's logits), one warp per frame
template <QKind KIND>
__global__ void __launch_bounds__(128) q_values_kernel(const QHead h, const float* __restrict__ rows, int N, float* __restrict__ q_out) {
  const int lane = threadIdx.x & 31, n = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (n >= N) return;
  const float q = q_lane<KIND>(h, rows, n, lane);
  if (lane < h.A) q_out[(size_t)n * h.A + lane] = q;
}

// theta_t = tau * theta + one_minus_tau * theta_t, each product and the sum rounded separately as torch computes it
__global__ void __launch_bounds__(256) apex_soft_update_kernel(const float* __restrict__ p, float* __restrict__ pt, int64_t n, float tau,
                                                               float one_minus_tau) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    pt[i] = __fadd_rn(__fmul_rn(tau, p[i]), __fmul_rn(one_minus_tau, pt[i]));
}

cudaError_t launch_q_tail(const QHead& on, const QHead& tg, const QTail& t, cudaStream_t st) {
  switch (on.kind) {
    case Q_PLAIN: dqn_tail_kernel<false><<<dqn_tail_blocks(t.B), 128, 0, st>>>(on, tg, t, 2.f / (float)t.B); break;
    case Q_DUELING: dqn_tail_kernel<true><<<dqn_tail_blocks(t.B), 128, 0, st>>>(on, tg, t, 2.f / (float)t.B); break;
    case Q_CATEGORICAL: return launch_cat_tail(on, tg, t, st);
    case Q_QUANTILE: return launch_qr_tail(on, tg, t, st);
  }
  return cudaGetLastError();
}
cudaError_t launch_q_wgrad(const QHead& h, const QHeadGrad& g, const QTail& t, cudaStream_t st) {
  if (head_has_logits(h)) return launch_cat_wgrad(t.dlogits, t.core_s, t.B, h.R, g.gW, g.gb, st);
  const int nslab = (t.B + DQN_SLAB - 1) / DQN_SLAB, spg = (nslab + HEAD_GROUPS - 1) / HEAD_GROUPS, groups = (nslab + spg - 1) / spg;
  const dim3 grid((513 + 127) / 128, groups);
  if (h.kind == Q_DUELING) {
    dqn_wgrad_kernel<true><<<grid, 128, 0, st>>>(t.dq, t.action, t.core_s, t.B, h.A, spg, t.head_part);
    dqn_wgrad_reduce_kernel<true><<<(h.R * 513 + 255) / 256, 256, 0, st>>>(t.head_part, groups, h.A, g.gW, g.gb, g.gba);
  } else {
    dqn_wgrad_kernel<false><<<grid, 128, 0, st>>>(t.dq, t.action, t.core_s, t.B, h.A, spg, t.head_part);
    dqn_wgrad_reduce_kernel<false><<<(h.R * 513 + 255) / 256, 256, 0, st>>>(t.head_part, groups, h.A, g.gW, g.gb, nullptr);
  }
  return cudaGetLastError();
}
cudaError_t launch_q_values(const QHead& h, const float* core, int N, float* logits, float* q_out, cudaStream_t st) {
  const int blocks = (N + 3) / 4;
  switch (h.kind) {
    case Q_PLAIN: q_values_kernel<Q_PLAIN><<<blocks, 128, 0, st>>>(h, core, N, q_out); break;
    case Q_DUELING: q_values_kernel<Q_DUELING><<<blocks, 128, 0, st>>>(h, core, N, q_out); break;
    case Q_CATEGORICAL: {
      const cudaError_t e = launch_cat_logits(core, h.W, h.b, N, h.R, logits, st);
      if (e != cudaSuccess) return e;
      q_values_kernel<Q_CATEGORICAL><<<blocks, 128, 0, st>>>(h, logits, N, q_out);
      break;
    }
    case Q_QUANTILE: {
      const cudaError_t e = launch_cat_logits(core, h.W, h.b, N, h.R, logits, st);
      if (e != cudaSuccess) return e;
      q_values_kernel<Q_QUANTILE><<<blocks, 128, 0, st>>>(h, logits, N, q_out);
      break;
    }
  }
  return cudaGetLastError();
}
cudaError_t launch_apex_soft_update(const float* p, float* pt, int64_t n, float tau, float one_minus_tau, cudaStream_t st) {
  const int64_t blocks = (n + 255) / 256;
  apex_soft_update_kernel<<<(int)(blocks < 1024 ? blocks : 1024), 256, 0, st>>>(p, pt, n, tau, one_minus_tau);
  return cudaGetLastError();
}

}  // namespace srl
