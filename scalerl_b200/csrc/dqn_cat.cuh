// The categorical (C51) Q head's device arithmetic (Bellemare et al. 2017, "A Distributional Perspective on Reinforcement Learning"),
// shared by the learner's tail (dqn_cat.cu) and the Ape-X actor (apex_actor.cu), so that an actor's Q values, greedy actions and
// initial priorities are the learner's bits for the same weights and logits.
// The head q = Linear(512, A K) writes K logits per action: row a K + k of a frame's logit row is atom k of action a.  p = softmax over
// an action's K logits, Q = sum_k z_k p_k on the support z_k = v_min + k dz.  Every sum runs in atom order, every rounding is
// explicit (no contraction), so the bits depend on the logits alone.
#pragma once
#include "common.cuh"
#include "dqn_head.cuh"
#include "dqn_qr.cuh"
#include "kernels.h"

namespace srl {

SRL_DEVINL float cat_z(const CatSupport& c, int k) { return __fadd_rn(c.v_min, __fmul_rn((float)k, c.dz)); }

// the softmax statistics of one row of K logits: mx = max_k x_k, se = sum_k exp(x_k - mx)
SRL_DEVINL void cat_row_stats(const float* __restrict__ x, int K, float* mx, float* se) {
  float m = -INFINITY;
  for (int k = 0; k < K; ++k) m = fmaxf(m, __ldg(x + k));
  float s = 0.f;
  for (int k = 0; k < K; ++k) s = __fadd_rn(s, expf(__fsub_rn(__ldg(x + k), m)));
  *mx = m;
  *se = s;
}
// p_k = exp(x_k - mx) / se; log p_k in the log-softmax form (x_k - mx) - log se, never log(p_k)
SRL_DEVINL float cat_p(float x, float mx, float se) { return __fdiv_rn(expf(__fsub_rn(x, mx)), se); }
SRL_DEVINL float cat_logp(float x, float mx, float lse) { return __fsub_rn(__fsub_rn(x, mx), lse); }

// Q = sum_k z_k p_k of one action's K logits
SRL_DEVINL float cat_q(const float* __restrict__ x, const CatSupport& c) {
  float mx, se;
  cat_row_stats(x, c.K, &mx, &se);
  float q = 0.f;
  for (int k = 0; k < c.K; ++k) q = __fmaf_rn(cat_z(c, k), cat_p(__ldg(x + k), mx, se), q);
  return q;
}
// the Q row of one frame's A K logits, one action per lane (lane a < A: Q_a; other lanes 0): q_row_max takes its first argmax
SRL_DEVINL float cat_q_lane(const float* __restrict__ row, int A, const CatSupport& c, int lane) {
  return lane < A ? cat_q(row + (size_t)lane * c.K, c) : 0.f;
}
// the Q row of frame n, one action per lane (lane a < A: Q_a), for every head: rows = the core rows [N][ENC_CORE] (scalar heads) or the
// logits [N][R] (categorical, quantile: dqn_qr.cuh).  The plain head's dot products end in warp_sum, whose xor butterfly leaves the
// same sum on every lane, so lane a holds the value q_max compares at a.
template <QKind KIND>
SRL_DEVINL float q_lane(const QHead& h, const float* rows, size_t n, int lane) {
  if constexpr (KIND == Q_CATEGORICAL) {
    return cat_q_lane(rows + n * h.R, h.A, h.c, lane);
  } else if constexpr (KIND == Q_QUANTILE) {
    return qr_q_lane(rows + n * h.R, h.A, h.qr.N, lane);
  } else if constexpr (KIND == Q_DUELING) {
    return dueling_q<false>(rows + n * ENC_CORE, h.W, h.b, h.ba, h.A, lane, nullptr);
  } else {
    float mine = 0.f;
    for (int a = 0; a < h.A; ++a) {
      const float v = q_dot(rows + n * ENC_CORE, h.W + (size_t)a * 512, lane) + __ldg(h.b + a);
      if (lane == a) mine = v;
    }
    return mine;
  }
}

// Algorithm 1 of Bellemare et al. 2017 on one lane: m[0 .. K-1] <- the projection onto the support of the target distribution p' (the
// softmax of x's K logits) moved to Tz_j = clamp(r + g z_j, v_min, v_max), g = gamma (1 - d).  b_j = (Tz_j - v_min) / dz, l = floor(b_j)
// and u = ceil(b_j) clamped to [0, K - 1]; m_l += p'_j (u - b_j), m_u += p'_j (b_j - l), or m_l += p'_j when l == u; j ascending.
// With g = 0 (done, or gamma = 0) every Tz_j is clamp(r): the whole mass, sum_j p'_j = 1, goes there exactly, so the target does not
// depend on s' (whose rows an actor's prioritized add may hold from a later step than the learner's after a done).
SRL_DEVINL void cat_project(const float* __restrict__ x, float reward, float g, const CatSupport& c, float* m) {
  for (int k = 0; k < c.K; ++k) m[k] = 0.f;
  if (g == 0.f) {
    const float b = __fdiv_rn(__fsub_rn(fminf(fmaxf(reward, c.v_min), c.v_max), c.v_min), c.dz);
    const int l = min(max((int)floorf(b), 0), c.K - 1), u = min(max((int)ceilf(b), 0), c.K - 1);
    if (l == u) {
      m[l] = 1.f;
    } else {
      m[l] = __fsub_rn((float)u, b);
      m[u] = __fsub_rn(b, (float)l);
    }
    return;
  }
  float mx, se;
  cat_row_stats(x, c.K, &mx, &se);
  for (int j = 0; j < c.K; ++j) {
    const float p = cat_p(__ldg(x + j), mx, se);
    const float tz = fminf(fmaxf(__fadd_rn(reward, __fmul_rn(g, cat_z(c, j))), c.v_min), c.v_max);
    const float b = __fdiv_rn(__fsub_rn(tz, c.v_min), c.dz);
    const int l = min(max((int)floorf(b), 0), c.K - 1), u = min(max((int)ceilf(b), 0), c.K - 1);
    if (l == u) {
      m[l] = __fadd_rn(m[l], p);
    } else {
      m[l] = __fadd_rn(m[l], __fmul_rn(p, __fsub_rn((float)u, b)));
      m[u] = __fadd_rn(m[u], __fmul_rn(p, __fsub_rn(b, (float)l)));
    }
  }
}

// max(KL, 0) + eps in double (Hessel et al. 2018 prioritise by the KL loss); a NaN KL stays NaN (the replay add counts it)
SRL_DEVINL double cat_priority(float kl, float eps) { return (double)(kl < 0.f ? 0.f : kl) + (double)eps; }

struct CatLoss {
  float ce;      // -sum_k m_k log p_k
  float kl;      // sum_k m_k (log m_k - log p_k), 0 log 0 = 0
  float q;       // Q(s, a) = sum_k z_k p_k
  float y;       // sum_k z_k m_k: the expectation of the projected target
};
// One transition on one warp; every lane calls it, lane 0 returns the result.  xt: the target network's A K logits of s'; a* = the
// first argmax of Q_target(s') or, with xn (double DQN: the online network's logits of s'), of Q_online(s'); m (K floats of shared
// memory) <- the projection of p_target(s')[a*]; then CE, KL, Q and y of xs (the online logits of s at the taken action) against m.
// d (NULL: not wanted) <- the logit gradient wB (p_k sum_k' m_k' - m_k) of wB CE.  m and d are visible to the warp on return.
SRL_DEVINL CatLoss cat_transition(const float* __restrict__ xs, const float* __restrict__ xn, const float* __restrict__ xt, int A,
                                  float reward, float g, const CatSupport& c, int lane, float* m, float wB, float* d) {
  int a_star;
  const float qt = cat_q_lane(xt, A, c, lane);
  if (xn) q_row_max(cat_q_lane(xn, A, c, lane), A, &a_star);
  else q_row_max(qt, A, &a_star);
  CatLoss r = {0.f, 0.f, 0.f, 0.f};
  if (lane == 0) {
    const int K = c.K;
    cat_project(xt + (size_t)a_star * K, reward, g, c, m);
    float mx, se;
    cat_row_stats(xs, K, &mx, &se);
    const float lse = logf(se);
    float s = 0.f, msum = 0.f;
    for (int k = 0; k < K; ++k) {
      const float x = __ldg(xs + k), mk = m[k], lp = cat_logp(x, mx, lse);
      s = __fmaf_rn(mk, lp, s);
      if (mk > 0.f) r.kl = __fmaf_rn(mk, __fsub_rn(logf(mk), lp), r.kl);
      r.q = __fmaf_rn(cat_z(c, k), cat_p(x, mx, se), r.q);
      r.y = __fmaf_rn(cat_z(c, k), mk, r.y);
      msum = __fadd_rn(msum, mk);
    }
    r.ce = -s;
    if (d)
      for (int k = 0; k < K; ++k) d[k] = __fmul_rn(wB, __fsub_rn(__fmul_rn(cat_p(__ldg(xs + k), mx, se), msum), m[k]));
  }
  __syncwarp();
  return r;
}

}  // namespace srl
