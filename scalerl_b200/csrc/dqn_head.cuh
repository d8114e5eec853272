// The Q head's device arithmetic, shared by the learner's tail (dqn.cu) and the Ape-X actor (apex_actor.cu), so that an actor's Q
// values, greedy actions and initial priorities are the same bits as the learner's for the same weights.
// The Q head reads the encoder's core rows [h (512), clamp(reward), one-hot] (ENC_CORE floats per row) and only their h columns.
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
// max_a Q(h)[a] and its first argmax (torch.max(dim=1) returns the first maximal index)
SRL_DEVINL float q_max(const float* h, const float* W, const float* b, int A, int lane, int* arg) {
  float best = -INFINITY;
  int ib = 0;
  for (int a = 0; a < A; ++a) {
    const float v = q_dot(h, W + (size_t)a * 512, lane) + __ldg(b + a);
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

}  // namespace srl
