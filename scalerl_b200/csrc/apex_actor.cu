// The Ape-X actor: per-env epsilon-greedy acting and the initial priorities of new transitions, forward-only on a parameter snapshot.
// Restates the reference's
//   scalerl/algorithms/apex/worker.py:14-30 (Actor: one eps per actor), :59-79 (compute_prior: |Q(s)[a] - (r + mask gamma^steps max Q(s'))|)
//   scalerl/algorithms/apex/memory.py:43-64 (PrioritizedReplayBuffer.add: each transition enters with its actor's priority)
// with one encoder forward (srl_encoder_forward) per frame set and the Q head of the learner (dqn_head.cuh, dqn_cat.cuh, dqn_qr.cuh), so that a
// priority computed here has the bits of the learner's for the same weights.  fp32 on the CUDA cores: the Q head is 512 x A, no
// tensor-core work.
//   apex_act_kernel       the Q row, its first argmax and the epsilon-greedy draw (one warp per env), a template on the head kind
//   apex_priority_kernel  q(s, a), the n-step target from max_a Q(s') and the priority (one warp per transition), plain or dueling
//   apex_cat_priority_kernel  the same on the categorical head: the learner tail's cat_transition
//   apex_qr_priority_kernel   the same on the quantile head: the learner tail's qr_transition
// The categorical and quantile heads run the learner's logits GEMM (dqn_cat.cu) first.  launch_apex_act and launch_apex_priorities are the one
// place that picks the kernels of a head.  The distributional dueling head composes its rows from the snapshot first (dueling_rows.cu), as
// the learner does, and then is the categorical or quantile head on them.
#include <math.h>
#include <string.h>
#include <new>
#include "common.cuh"
#include "dqn_cat.cuh"
#include "dqn_head.cuh"
#include "errors.h"
#include "kernels.h"
#include "../../include/scalerl_b200.h"

namespace srl {

constexpr int64_t ACTOR_OBS_BYTES = 4 * 84 * 84;

// env e's action of draw d: with probability eps[e] a uniform action, else `greedy`
SRL_DEVINL int64_t eps_greedy(unsigned long long d, int e, uint2 key, int A, const float* __restrict__ eps, int greedy) {
  const uint4 r = philox4x32_10(make_uint4((uint32_t)d, (uint32_t)(d >> 32), (uint32_t)e, 0u), key);
  const float u = (float)(r.x >> 8) * 0x1p-24f;                            // uniform in [0, 1)
  const int random_action = (int)(((unsigned long long)r.y * (unsigned)A) >> 32);   // uniform in [0, A)
  return u < __ldg(eps + e) ? random_action : greedy;
}
// the end of an act launch: the block that finishes last advances the draw counter d and re-arms the ticket
SRL_DEVINL void advance_draws(unsigned long long* draws, unsigned long long d) {
  __shared__ bool is_last;
  __syncthreads();                 // every warp of the block has read the counter
  if (threadIdx.x == 0) is_last = take_ticket(reinterpret_cast<float*>(draws + 1));
  __syncthreads();
  if (is_last && threadIdx.x == 0) {
    draws[0] = d + 1;
    *reinterpret_cast<unsigned*>(draws + 1) = 0u;
  }
}

// One warp per env, 4 per block.  draws[0]: the draw counter (u64), read by every block and advanced by the block that finishes
// last (draws[1] low word: the ticket, re-armed by that block), so every env of one launch uses the same draw.  rows: q_lane's (the
// core rows, or the categorical head's logits).
template <QKind KIND>
__global__ void __launch_bounds__(128) apex_act_kernel(const QHead h, const float* __restrict__ rows, int E, const float* __restrict__ eps,
                                                       uint2 key, unsigned long long* draws, int64_t* __restrict__ actions) {
  const int lane = threadIdx.x & 31, e = blockIdx.x * 4 + (threadIdx.x >> 5);
  const unsigned long long d = *reinterpret_cast<volatile unsigned long long*>(draws);
  if (e < E) {
    int greedy;
    q_row_max(q_lane<KIND>(h, rows, e, lane), h.A, &greedy);
    if (lane == 0) actions[e] = eps_greedy(d, e, key, h.A, eps, greedy);
  }
  advance_draws(draws, d);
}

// One warp per transition e in ring slot (ptr + e) mod M, 4 per block: q = Q(s)[a], y = R + gamma_n (1 - d) max_a Q(s'), the
// learner tail's arithmetic (dqn_tail_kernel with the snapshot as online and target network, no double DQN)
template <bool DUELING>
__global__ void __launch_bounds__(128) apex_priority_kernel(const QHead h, const float* __restrict__ core_s, const float* __restrict__ core_n,
                                                            int E, const int64_t* __restrict__ action, const float* __restrict__ reward,
                                                            const uint8_t* __restrict__ done, int64_t ptr, int64_t M, float gamma_n, float eps,
                                                            double* __restrict__ prio) {
  const int lane = threadIdx.x & 31, e = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (e >= E) return;
  const int64_t slot = (ptr + e) % M;
  const int act = ld_action(action + slot, h.A);
  float q, nx;
  int a_star;
  if constexpr (DUELING) {
    q = __shfl_sync(0xffffffffu, dueling_q<false>(core_s + (size_t)e * ENC_CORE, h.W, h.b, h.ba, h.A, lane, nullptr), act);
    nx = q_row_max(dueling_q<false>(core_n + (size_t)e * ENC_CORE, h.W, h.b, h.ba, h.A, lane, nullptr), h.A, &a_star);
  } else {
    q = q_dot(core_s + (size_t)e * ENC_CORE, h.W + (size_t)act * 512, lane) + __ldg(h.b + act);
    nx = q_max(core_n + (size_t)e * ENC_CORE, h.W, h.b, h.A, lane, &a_star);
  }
  const float y = td_target(__ldg(reward + slot), gamma_n, nx, done[slot] != 0);
  if (lane == 0) prio[e] = td_priority(__fsub_rn(q, y), eps);
}
// the categorical head: the learner tail's cat_transition with the snapshot's logits of s (logits_s) and s' (logits_n) as the online and
// target network's, no double DQN -> max(KL(m || p(s)[a]), 0) + eps
__global__ void __launch_bounds__(128) apex_cat_priority_kernel(const QHead h, const float* __restrict__ logits_s, const float* __restrict__ logits_n,
                                                                int E, const int64_t* __restrict__ action, const float* __restrict__ reward,
                                                                const uint8_t* __restrict__ done, int64_t ptr, int64_t M, float gamma_n, float eps,
                                                                double* __restrict__ prio) {
  __shared__ float sm[4][CAT_MAX_ATOMS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, e = blockIdx.x * 4 + warp;
  if (e >= E) return;
  const int64_t slot = (ptr + e) % M;
  const int act = ld_action(action + slot, h.A);
  const CatLoss r = cat_transition(logits_s + (size_t)e * h.R + (size_t)act * h.c.K, nullptr, logits_n + (size_t)e * h.R, h.A,
                                   __ldg(reward + slot), done[slot] ? 0.f : gamma_n, h.c, lane, sm[warp], 0.f, nullptr);
  if (lane == 0) prio[e] = cat_priority(r.kl, eps);
}

// the quantile head: the learner tail's qr_transition with the snapshot's quantiles of s (theta_s) and s' (theta_n) as the online and
// target network's, no double DQN -> the quantile Huber loss + eps
__global__ void __launch_bounds__(128) apex_qr_priority_kernel(const QHead h, const float* __restrict__ theta_s, const float* __restrict__ theta_n,
                                                               int E, const int64_t* __restrict__ action, const float* __restrict__ reward,
                                                               const uint8_t* __restrict__ done, int64_t ptr, int64_t M, float gamma_n, float eps,
                                                               double* __restrict__ prio) {
  __shared__ float st[4][QR_MAX_QUANTILES];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, e = blockIdx.x * 4 + warp;
  if (e >= E) return;
  const int64_t slot = (ptr + e) % M;
  const int act = ld_action(action + slot, h.A);
  const QrLoss r = qr_transition<false>(theta_s + (size_t)e * h.R + (size_t)act * h.qr.N, nullptr, theta_n + (size_t)e * h.R, h.A, h.qr.N,
                                        __ldg(reward + slot), done[slot] ? 0.f : gamma_n, h.qr.kappa, lane, st[warp], 0.f, nullptr);
  if (lane == 0) prio[e] = qr_priority(r.loss, eps);
}

// the act kernel of head h over the E core rows (the categorical and quantile heads: through logits [E][R])
cudaError_t launch_apex_act(const QHead& h, const float* core, float* logits, int E, const float* eps, uint2 key, unsigned long long* draws,
                            int64_t* actions, cudaStream_t st) {
  const int blocks = (E + 3) / 4;
  switch (h.kind) {
    case Q_PLAIN: apex_act_kernel<Q_PLAIN><<<blocks, 128, 0, st>>>(h, core, E, eps, key, draws, actions); break;
    case Q_DUELING: apex_act_kernel<Q_DUELING><<<blocks, 128, 0, st>>>(h, core, E, eps, key, draws, actions); break;
    case Q_CATEGORICAL: {
      const cudaError_t e = launch_cat_logits(core, h.W, h.b, E, h.R, logits, st);
      if (e != cudaSuccess) return e;
      apex_act_kernel<Q_CATEGORICAL><<<blocks, 128, 0, st>>>(h, logits, E, eps, key, draws, actions);
      break;
    }
    case Q_QUANTILE: {
      const cudaError_t e = launch_cat_logits(core, h.W, h.b, E, h.R, logits, st);
      if (e != cudaSuccess) return e;
      apex_act_kernel<Q_QUANTILE><<<blocks, 128, 0, st>>>(h, logits, E, eps, key, draws, actions);
      break;
    }
  }
  return cudaGetLastError();
}
// the priority kernel of head h over the core rows of s (core) and s' (core + E rows); the categorical and quantile heads: through
// logits [2E][R]
cudaError_t launch_apex_priorities(const QHead& h, const float* core, float* logits, int E, const int64_t* action, const float* reward,
                                   const uint8_t* done, int64_t ptr, int64_t M, float gamma_n, float eps, double* prio, cudaStream_t st) {
  const int blocks = (E + 3) / 4;
  const float* core_n = core + (size_t)E * ENC_CORE;
  switch (h.kind) {
    case Q_PLAIN:
      apex_priority_kernel<false><<<blocks, 128, 0, st>>>(h, core, core_n, E, action, reward, done, ptr, M, gamma_n, eps, prio);
      break;
    case Q_DUELING:
      apex_priority_kernel<true><<<blocks, 128, 0, st>>>(h, core, core_n, E, action, reward, done, ptr, M, gamma_n, eps, prio);
      break;
    case Q_CATEGORICAL: {
      const cudaError_t e = launch_cat_logits(core, h.W, h.b, 2 * E, h.R, logits, st);      // s and s' rows in one GEMM
      if (e != cudaSuccess) return e;
      apex_cat_priority_kernel<<<blocks, 128, 0, st>>>(h, logits, logits + (size_t)E * h.R, E, action, reward, done, ptr, M, gamma_n, eps, prio);
      break;
    }
    case Q_QUANTILE: {
      const cudaError_t e = launch_cat_logits(core, h.W, h.b, 2 * E, h.R, logits, st);      // s and s' rows in one GEMM
      if (e != cudaSuccess) return e;
      apex_qr_priority_kernel<<<blocks, 128, 0, st>>>(h, logits, logits + (size_t)E * h.R, E, action, reward, done, ptr, M, gamma_n, eps, prio);
      break;
    }
  }
  return cudaGetLastError();
}

}  // namespace srl
using namespace srl;

struct srl_apex_actor {
  int E, precision;
  uint2 key;
  ApexNetDesc desc;
  ApexNet snap;                    // the snapshot on its flat buffer (noisy: the mu tensors)
  ApexNet run;                     // what the forwards run on: noisy, the kept draw's composed weights (apex_forward_net); else snap
  float* logits;                   // categorical / quantile: [2E][R], the logits (quantiles) of the core rows
  srl_encoder_t* enc;
  char *saved, *scratch;           // encoder blocks for E frames: the two forwards of an add run one after the other
  float* core;                     // [2E][ENC_CORE]: the forward over s (and act's), then the one over s'
  float* zero_reward;              // the reward / action columns of the forwards (the Q head reads h only)
  int64_t* zero_action;
  double* prio;                    // [E] the priorities of the last add
  unsigned long long* draws;       // [0] draw counter, [1] the act kernel's ticket
  // noisy networks: the kept draw, its counter and the composed weights
  float *normals, *noise;
  unsigned long long* noise_draws;
  NoisyWeights cw;
  HeadRows rows;                   // the distributional dueling head: the rows the last call composed
  char* arena;
};

namespace {
int actor_rows(srl_apex_actor* X, int64_t saved, int64_t scratch, WsRow* t) {
  const int64_t E = X->E;
  int n = 0;
  t[n++] = ws_row<char>(nullptr, saved, &X->saved);
  t[n++] = ws_row<char>(nullptr, scratch, &X->scratch);
  t[n++] = ws_row(nullptr, 2 * E * ENC_CORE, &X->core);
  t[n++] = ws_row(nullptr, E, &X->zero_reward);
  t[n++] = ws_row(nullptr, E, &X->zero_action);
  t[n++] = ws_row(nullptr, E, &X->prio);
  t[n++] = ws_row(nullptr, 2, &X->draws);
  t[n++] = ws_row(nullptr, head_has_logits(X->desc.head) ? 2 * E * X->desc.head.R : 0, &X->logits);
  t[n++] = ws_row(nullptr, X->desc.noisy, &X->noise_draws);
  n += noise_rows(X->desc, 0, &X->normals, &X->noise, &X->cw, t + n);
  const int64_t DR = dist_dueling(X->desc) ? X->desc.head.R : 0;
  t[n++] = ws_row("rows_weight", DR * 512, &X->rows.W);
  t[n++] = ws_row("rows_bias", DR, &X->rows.b);
  return n;
}
constexpr int ACTOR_ROWS = 18;

// the head of the actor's next forwards, from the snapshot as it is now: a noisy actor draws new noise first when `draw` (act) and
// composes the kept draw with the snapshot; the distributional dueling head composes its rows from those weights -> *h
cudaError_t actor_head(srl_apex_actor* X, bool draw, cudaStream_t st, QHead* h) {
  *h = X->run.q;
  if (X->desc.noisy) {
    if (draw) {
      const cudaError_t e = launch_noisy_draw(X->key, nullptr, X->noise_draws, 1, noise_count(X->desc), &X->normals, &X->noise, st);
      if (e != cudaSuccess) return e;
    }
    const float* noise = X->noise;
    const cudaError_t e = launch_noisy_compose(&X->snap.nz, &X->cw, &noise, 1, X->desc, st);
    if (e != cudaSuccess) return e;
  }
  if (!dist_dueling(X->desc)) return cudaSuccess;
  *h = on_rows(*h, X->rows);
  return launch_dist_dueling_compose(&X->run.q, &X->rows, 1, X->desc.vrows, st);
}

// Q head rows of `frames` frames of obs into core (f <= E frames per call)
int actor_forward(srl_apex_actor* X, const uint8_t* obs, int frames, float* core, cudaStream_t st) {
  return srl_encoder_forward(X->enc, obs, X->zero_reward, X->zero_action, frames, 1, X->run.w8, X->saved, X->scratch, core, st);
}
}  // namespace

extern "C" int srl_apex_actor_create(int A, int num_envs, int precision, uint64_t seed, const float* params, srl_apex_actor_t** out) {
  return srl_apex_actor_create_quantile(A, num_envs, precision, 0, 0, 0.f, 0.f, 0, 0.f, 0, seed, params, out);
}

extern "C" int srl_apex_actor_create_ex(int A, int num_envs, int precision, int dueling, uint64_t seed, const float* params,
                                        srl_apex_actor_t** out) {
  return srl_apex_actor_create_quantile(A, num_envs, precision, dueling, 0, 0.f, 0.f, 0, 0.f, 0, seed, params, out);
}

extern "C" int srl_apex_actor_create_cat(int A, int num_envs, int precision, int num_atoms, float v_min, float v_max, uint64_t seed,
                                         const float* params, srl_apex_actor_t** out) {
  return srl_apex_actor_create_quantile(A, num_envs, precision, 0, num_atoms, v_min, v_max, 0, 0.f, 0, seed, params, out);
}

extern "C" int srl_apex_actor_create_noisy(int A, int num_envs, int precision, int dueling, int num_atoms, float v_min, float v_max, int noisy,
                                           uint64_t seed, const float* params, srl_apex_actor_t** out) {
  return srl_apex_actor_create_quantile(A, num_envs, precision, dueling, num_atoms, v_min, v_max, 0, 0.f, noisy, seed, params, out);
}

extern "C" int srl_apex_actor_create_quantile(int A, int num_envs, int precision, int dueling, int num_atoms, float v_min, float v_max,
                                              int num_quantiles, float kappa, int noisy, uint64_t seed, const float* params,
                                              srl_apex_actor_t** out) {
  return srl_apex_actor_create_dist_dueling(A, num_envs, precision, dueling, num_atoms, v_min, v_max, num_quantiles, kappa, 0, noisy, seed,
                                            params, out);
}

extern "C" int srl_apex_actor_create_dist_dueling(int A, int num_envs, int precision, int dueling, int num_atoms, float v_min, float v_max,
                                                  int num_quantiles, float kappa, int dist_dueling, int noisy, uint64_t seed,
                                                  const float* params, srl_apex_actor_t** out) {
  REQ(params && out, "apex_actor_create: NULL argument");
  REQ(num_envs >= 1 && num_envs <= MAX_FRAMES, "apex_actor_create: num_envs=%d must be in [1, %d]", num_envs, MAX_FRAMES);
  REQ(precision == 0 || precision == 1, "apex_actor_create: precision=%d must be 0 (bf16 operands) or 1 (fp32-accurate split operands)", precision);
  ApexNetDesc d;
  int rc = make_apex_desc("apex_actor_create", A, dueling, num_atoms, v_min, v_max, num_quantiles, kappa, dist_dueling, noisy, &d);
  if (rc) return rc;
  REQ(!misaligned(params, 16), "apex_actor_create: params must be 16-byte aligned");
  int64_t sb = 0, kb = 0;
  rc = srl_encoder_sizes(num_envs, precision, &sb, &kb);
  if (rc) return rc;
  srl_apex_actor* X = new (std::nothrow) srl_apex_actor();
  REQ(X, "out of host memory");
  auto undo = [X](int code) { srl_apex_actor_destroy(X); return code; };
  X->E = num_envs;
  X->precision = precision;
  X->key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  X->desc = d;
  X->snap = bind_apex(d, const_cast<float*>(params));
  rc = srl_encoder_create(precision, &X->enc);
  if (rc) return undo(rc);
  WsRow t[ACTOR_ROWS];
  const int n = actor_rows(X, sb, kb, t);
  const int64_t total = rows_bytes(t, n, false);
  cudaError_t e = cudaMalloc(&X->arena, total);
  if (e != cudaSuccess) return undo(cuda_fail(e, "apex_actor_create: cudaMalloc"));
  e = cudaMemset(X->arena, 0, total);          // the zero columns, the draw counters and the ticket
  if (e != cudaSuccess) return undo(cuda_fail(e, "apex_actor_create: cudaMemset"));
  carve_rows(t, n, false, X->arena);
  X->run = apex_forward_net(d, X->snap, X->cw);
  if (noisy) {      // the first draw, kept until the first act
    e = launch_noisy_draw(X->key, nullptr, X->noise_draws, 1, noise_count(d), &X->normals, &X->noise, nullptr);
    if (e == cudaSuccess) e = cudaStreamSynchronize(nullptr);
    if (e != cudaSuccess) return undo(cuda_fail(e, "apex_actor_create: first noise draw"));
  }
  *out = X;
  return 0;
}

extern "C" int srl_apex_actor_destroy(srl_apex_actor_t* X) {
  if (!X) return 0;
  srl_encoder_destroy(X->enc);
  cudaFree(X->arena);
  delete X;
  return 0;
}

extern "C" int srl_apex_actor_act(srl_apex_actor_t* X, const uint8_t* obs, const float* epsilons, int64_t* actions, void* stream) {
  REQ(X && obs && epsilons && actions, "apex_actor_act: NULL pointer");
  const int E = X->E;
  const Span s[3] = {{obs, E * ACTOR_OBS_BYTES, false, "obs"}, {epsilons, (int64_t)E * 4, false, "epsilons"}, {actions, (int64_t)E * 8, true, "actions"}};
  int rc = check_spans(s, 3, "apex_actor_act");
  if (rc) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  QHead h;
  CU(actor_head(X, true, st, &h), "apex_actor_act: head");
  rc = actor_forward(X, obs, E, X->core, st);
  if (rc) return rc;
  CU(launch_apex_act(h, X->core, X->logits, E, epsilons, X->key, X->draws, actions, st), "apex_act");
  return 0;
}

extern "C" int srl_apex_actor_q_values(srl_apex_actor_t* X, const uint8_t* obs, int n, float* q_out, void* stream) {
  REQ(X && obs && q_out, "apex_actor_q_values: NULL pointer");
  REQ(n >= 1, "apex_actor_q_values: n=%d must be >= 1", n);
  const int A = X->desc.head.A;
  const Span s[2] = {{obs, n * ACTOR_OBS_BYTES, false, "obs"}, {q_out, (int64_t)n * A * 4, true, "q_out"}};
  int rc = check_spans(s, 2, "apex_actor_q_values");
  if (rc) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  QHead h;
  CU(actor_head(X, false, st, &h), "apex_actor_q_values: head");
  for (int f0 = 0; f0 < n; f0 += X->E) {        // chunks of at most E frames: the blocks' size
    const int f = n - f0 < X->E ? n - f0 : X->E;
    rc = actor_forward(X, obs + (size_t)f0 * ACTOR_OBS_BYTES, f, X->core, st);
    if (rc) return rc;
    CU(launch_q_values(h, X->core, f, X->logits, q_out + (size_t)f0 * A, st), "q_values");
  }
  return 0;
}

extern "C" int srl_apex_actor_debug_buffer(srl_apex_actor_t* X, const char* name, void** ptr, int64_t* count) {
  REQ(X && name && ptr && count, "apex_actor_debug_buffer: NULL argument");
  const int64_t rows = 2 * (int64_t)X->E;
  if (strcmp(name, "core") == 0) { *ptr = X->core; *count = rows * ENC_CORE; return 0; }
  if (strcmp(name, X->desc.head.kind == Q_QUANTILE ? "theta" : "logits") == 0 && head_has_logits(X->desc.head)) {
    *ptr = X->logits; *count = rows * X->desc.head.R; return 0;
  }
  int64_t sb = 0, kb = 0;
  int rc = srl_encoder_sizes(X->E, X->precision, &sb, &kb);
  if (rc) return rc;
  srl_apex_actor shadow = *X;          // the table's rows re-derived on a copy: the same sizes give the same addresses
  WsRow t[ACTOR_ROWS];
  const int n = actor_rows(&shadow, sb, kb, t);
  carve_rows(t, n, false, X->arena);
  for (int i = 0; i < n; ++i)
    if (t[i].name && strcmp(t[i].name, name) == 0 && t[i].count > 0) { *ptr = *t[i].hi; *count = t[i].count; return 0; }
  return fail(SRL_EINVAL, "apex_actor_debug_buffer: unknown buffer '%s'", name);
}

namespace srl {
int apex_actor_num_envs(const srl_apex_actor* X) { return X->E; }

int apex_actor_priorities(srl_apex_actor* X, const uint8_t* s, const uint8_t* s_next, const int64_t* action, const float* reward,
                          const uint8_t* done, int64_t ptr, int64_t M, float gamma_n, float eps, const double** prio, cudaStream_t st) {
  const int E = X->E;
  QHead h;
  CU(actor_head(X, false, st, &h), "apex_actor_priorities: head");
  int rc = actor_forward(X, s, E, X->core, st);
  if (!rc) rc = actor_forward(X, s_next, E, X->core + (size_t)E * ENC_CORE, st);
  if (rc) return rc;
  CU(launch_apex_priorities(h, X->core, X->logits, E, action, reward, done, ptr, M, gamma_n, eps, X->prio, st), "apex_priorities");
  *prio = X->prio;
  return 0;
}
}  // namespace srl
