// The Q head's device arithmetic, shared by the learner's tail (dqn.cu) and the Ape-X actor (apex_actor.cu), so that an actor's Q
// values, greedy actions and initial priorities are the same bits as the learner's for the same weights.
// The Q head reads the encoder's core rows [h (512), clamp(reward), one-hot] (ENC_CORE floats per row) and only their h columns.
// Two heads: the plain q = Linear(512, A) (q_dot / q_max) and the dueling V + Adv - mean(Adv) (dueling_q / q_row_max), both on h.
#pragma once
#include "common.cuh"

namespace srl {

// q = h . W[a] + b[a] for one 512-float row h of a core row and one 512-float weight row: lane-strided products, then the warp sum
SRL_DEVINL float q_dot(const float* __restrict__ h, const float* __restrict__ w, int lane) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) s = fmaf(__ldg(h + lane + 32 * i), __ldg(w + lane + 32 * i), s);
  return warp_sum(s);
}
// max_a Q(h)[a] and its first argmax (torch.max(dim=1) returns the first maximal index).  UNROLL rows in flight: the learner's tail
// takes 2, since its loop is bound by the weight rows' load latency
template <int UNROLL = 1>
SRL_DEVINL float q_max(const float* h, const float* W, const float* b, int A, int lane, int* arg) {
  float best = -INFINITY;
  int ib = 0;
#pragma unroll UNROLL
  for (int a = 0; a < A; ++a) {
    const float v = q_dot(h, W + (size_t)a * 512, lane) + __ldg(b + a);
    if (v > best) { best = v; ib = a; }
  }
  *arg = ib;
  return best;
}

// The dueling head (Wang et al. 2016, eq. 9) on the shared fc output: W = [(A + 1)][512] with the value row first, then the A
// advantage rows; bv = [1] the value bias, ba = [A] the advantage biases.
//   V = h . W[0] + bv,  Adv_a = h . W[1 + a] + ba[a],  Q_a = (V + Adv_a) - mean_a Adv_a
// The mean is the sum over a = 0 .. A-1 in that order, divided by A (IEEE division: nothing is contracted).  Returns Q_lane on
// lanes < A (every lane of the warp takes part).  With WSUM, wsum[i] = sum_a W[1 + a][lane + 32 i] in the same order, the column
// sums of the advantage rows that the tail's dcore needs, from the loads the dot products make anyway.
template <bool WSUM>
SRL_DEVINL float dueling_q(const float* __restrict__ h, const float* __restrict__ W, const float* __restrict__ bv,
                           const float* __restrict__ ba, int A, int lane, float* wsum) {
  const float v = q_dot(h, W, lane) + __ldg(bv);
  if (WSUM) {
#pragma unroll
    for (int i = 0; i < 16; ++i) wsum[i] = 0.f;
  }
  float s = 0.f, mine = 0.f;
  for (int a = 0; a < A; ++a) {
    const float* w = W + (size_t)(a + 1) * 512;
    const float adv = q_dot(h, w, lane) + __ldg(ba + a);
    if (WSUM) {
#pragma unroll
      for (int i = 0; i < 16; ++i) wsum[i] += __ldg(w + lane + 32 * i);
    }
    s += adv;
    if (lane == a) mine = adv;
  }
  return __fsub_rn(__fadd_rn(v, mine), __fdiv_rn(s, (float)A));
}
// max_a and the first argmax of a Q row held one action per lane (lane a: Q_a, a < A), in q_max's order and comparison
SRL_DEVINL float q_row_max(float q, int A, int* arg) {
  float best = -INFINITY;
  int ib = 0;
  for (int a = 0; a < A; ++a) {
    const float v = __shfl_sync(0xffffffffu, q, a);
    if (v > best) { best = v; ib = a; }
  }
  *arg = ib;
  return best;
}
// y = r + gamma * Q' * (1 - d), the products and the add rounded one by one as torch evaluates them (no FMA contraction)
SRL_DEVINL float td_target(float reward, float gamma, float next_q, bool done) {
  return __fadd_rn(reward, __fmul_rn(__fmul_rn(gamma, next_q), done ? 0.f : 1.f));
}
// |q - y| + eps in double (apex/worker.py:152-154; + eps > 0 keeps the tree's assert), from delta = q - y
SRL_DEVINL double td_priority(float delta, float eps) { return (double)fabsf(delta) + (double)eps; }

// The learner tails' loss (one warp per transition, 4 per block; every thread of every block calls it with l = its warp's weighted loss
// on lane 0): the block partial (l0 + l1) + (l2 + l3) goes to scratch[4 + block], then the ticket scratch[0]; the last block adds the
// partials lane-strided in block order, then the warp sum, and writes loss[0] = sum / B and re-arms the ticket.
SRL_DEVINL void tail_loss(float l, int B, float* scratch, float* loss) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __shared__ float red[4];
  __shared__ bool is_last;
  if (lane == 0) red[warp] = l;
  __syncthreads();
  if (threadIdx.x == 0) {
    scratch[4 + blockIdx.x] = (red[0] + red[1]) + (red[2] + red[3]);
    is_last = take_ticket(scratch);
  }
  __syncthreads();
  if (is_last && warp == 0) {
    __threadfence();
    float s = 0.f;
    for (unsigned k = lane; k < gridDim.x; k += 32) s += reinterpret_cast<volatile float*>(scratch)[4 + k];
    s = warp_sum(s);
    if (lane == 0) {
      loss[0] = s / (float)B;
      *reinterpret_cast<unsigned*>(scratch) = 0u;      // re-arm the ticket
    }
  }
}

}  // namespace srl
