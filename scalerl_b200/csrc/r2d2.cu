// The R2D2 learner step (Kapturowski et al. 2019, "Recurrent Experience Replay in Distributed Reinforcement Learning"): the encoder
// (srl_encoder_*) and the 2-layer LSTM core (srl_lstm_core_*) of AtariNet(use_lstm=True), a Q head on the core output, and the
// sequence tail.  The kernels here are fp32 on the CUDA cores (the head is H x A with H = 513 + A: no tensor-core work):
//   r2d2_head_fwd_kernel          Q rows [N][A] of core output rows [N][H]: q = Linear(H, A), or the dueling head V + Adv - mean(Adv)
//                                 with the advantage mean summed in action order (dqn_head.cuh's dueling_q on K = H columns)
//   r2d2_tail_kernel              per sequence: a* (double Q), the n-step return, the value-rescaled target, the TD errors, the
//                                 priority eta max|d| + (1 - eta) mean|d| + eps, the dense dQ rows and the loss through tail_loss's
//                                 ticket reduction
//   r2d2_head_dcore_kernel        dout = dQ W (the dueling composition folded in), zero on the bootstrap rows
//   r2d2_head_wgrad_kernel /      the head's weight and bias gradients: slab-group partials, then the groups added in group order
//   r2d2_head_wgrad_reduce_kernel (dqn_wgrad_kernel's scheme on K = H columns; no atomics, the same bits on every run)
// The entry points srl_r2d2_* compose these with the encoder, the LSTM core, the fused clip + Adam step and the sampler's priority
// update on one stream, so a step can be captured as one CUDA graph.
#include <string.h>
#include <cmath>
#include <new>

#include "../../include/scalerl_b200.h"
#include "common.cuh"
#include "dqn_head.cuh"
#include "errors.h"
#include "kernels.h"

namespace srl {
namespace {

constexpr int R2_MAX_K = 544;                 // H = 513 + A, A <= 31
constexpr int R2_KI = R2_MAX_K / 32;          // columns per lane
constexpr int R2_SLAB = 16, R2_MAX_R = 32;    // wgrad: rows per slab, head rows (A or A + 1)
constexpr int R2_QF = 2048;                   // most frames of one q-value chunk

// The Q head on the core output: plain, W = q.weight [A][K], b = q.bias [A]; dueling, W = value.weight [1][K], b = value.bias [1],
// Wa = advantage.weight [A][K], ba = advantage.bias [A].  Head row r: plain, q row r; dueling, row 0 the value and row 1 + a the
// advantage of action a.
struct R2Head {
  const float *W, *b, *Wa, *ba;
  int A, K;
};
struct R2HeadGrad {
  float *gW, *gb, *gWa, *gba;
};

SRL_DEVINL double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
SRL_DEVINL double warp_max_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// x . w over the K columns, lane-strided: lane holds x[lane + 32 i]; one fmaf chain per lane, then the warp sum
SRL_DEVINL float row_dot(const float (&x)[R2_KI], const float* __restrict__ w, int K, int lane) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < R2_KI; ++i) {
    const int j = lane + 32 * i;
    if (j < K) s = fmaf(x[i], __ldg(w + j), s);
  }
  return warp_sum(s);
}

// one warp per row: q[n][a] = Q(X[n])[a]
template <bool DUELING>
__global__ void __launch_bounds__(128) r2d2_head_fwd_kernel(const R2Head h, const float* __restrict__ X, int N, float* __restrict__ q) {
  const int lane = threadIdx.x & 31, n = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (n >= N) return;
  const int K = h.K, A = h.A;
  float x[R2_KI];
#pragma unroll
  for (int i = 0; i < R2_KI; ++i) {
    const int j = lane + 32 * i;
    x[i] = j < K ? __ldg(X + (size_t)n * K + j) : 0.f;
  }
  float mine = 0.f;
  if constexpr (!DUELING) {
    for (int a = 0; a < A; ++a) {
      const float v = row_dot(x, h.W + (size_t)a * K, K, lane) + __ldg(h.b + a);
      if (lane == a) mine = v;
    }
  } else {            // (V + Adv_a) - (sum_a Adv_a) / A, the sum in action order
    const float v = row_dot(x, h.W, K, lane) + __ldg(h.b);
    float s = 0.f, adv_mine = 0.f;
    for (int a = 0; a < A; ++a) {
      const float adv = row_dot(x, h.Wa + (size_t)a * K, K, lane) + __ldg(h.ba + a);
      s = __fadd_rn(s, adv);
      if (lane == a) adv_mine = adv;
    }
    mine = __fsub_rn(__fadd_rn(v, adv_mine), __fdiv_rn(s, (float)A));
  }
  if (lane < A) q[(size_t)n * A + lane] = mine;
}

// value rescaling (Pohlen et al. 2018; R2D2 section 2): h(x) = sign(x)(sqrt(|x| + 1) - 1) + eps x and its inverse, in double
SRL_DEVINL double rescale_h(double x, double eps) {
  const double s = x > 0.0 ? 1.0 : (x < 0.0 ? -1.0 : 0.0);
  return s * (sqrt(fabs(x) + 1.0) - 1.0) + eps * x;
}
SRL_DEVINL double rescale_h_inv(double x, double eps) {
  const double s = x > 0.0 ? 1.0 : (x < 0.0 ? -1.0 : 0.0);
  const double r = (sqrt(1.0 + 4.0 * eps * (fabs(x) + 1.0 + eps)) - 1.0) / (2.0 * eps);
  return s * (r * r - 1.0);
}

// One batch of B sequences of L = burn_in + T + n rows (time-major [L][B] columns).  q_on [(T + n)][B][A]: the online Q rows of batch
// rows burn_in .. L - 1; q_tg [T][B][A]: the target Q rows of batch rows burn_in + n .. L - 1.  Outputs per trained row i (batch row
// burn_in + i), [T][B]: q_taken, y, delta and dq [T][B][A]; per sequence the priority (f64 [B]); the loss [1].
struct R2Tail {
  const float *q_on, *q_tg;
  const int64_t* last_action;
  const float* reward;
  const uint8_t* done;
  const float* weight;
  int B, A, burn_in, T, n;
  float gamma;
  int rescale;
  double rescale_eps, eta, priority_eps;
  float two_over_BT;
  float *q_taken, *y, *delta, *dq, *loss, *scratch;
  double* prio;
};

// One warp per sequence, 4 per block; lane l takes the trained rows i = l, l + 32, ...  For row t = burn_in + i: a_t =
// last_action[t + 1], m = the first k in 1..n with done[t + k], G = sum_{k=1}^{min(n, m)} gamma^{k-1} reward[t + k] (in double, in
// k order), a* = the first argmax of Q_online(s_{t+n}), y = h(G + [no m] gamma^n h^-1(Q_target(s_{t+n}, a*))) rounded once to fp32,
// delta = Q_online(s_t, a_t) - y.  loss = (1 / (B T)) sum_b w_b sum_t delta^2 (tail_loss over the blocks' partials).
__global__ void __launch_bounds__(128) r2d2_tail_kernel(const R2Tail t) {
  const int lane = threadIdx.x & 31, b = blockIdx.x * 4 + (threadIdx.x >> 5);
  float l = 0.f;
  if (b < t.B) {
    const int B = t.B, A = t.A;
    const float w = t.weight ? __ldg(t.weight + b) : 1.f;
    double dmax = 0.0, dsum = 0.0;
    float d2 = 0.f;
    for (int i = lane; i < t.T; i += 32) {
      const int r = t.burn_in + i;                       // the batch row of s_t
      const int act = ld_action(t.last_action + (size_t)(r + 1) * B + b, A);
      const float q = __ldg(t.q_on + ((size_t)i * B + b) * A + act);
      const float* qn = t.q_on + ((size_t)(i + t.n) * B + b) * A;
      float best = -INFINITY;
      int a_star = 0;
      for (int a = 0; a < A; ++a) {
        const float v = __ldg(qn + a);
        if (v > best) { best = v; a_star = a; }
      }
      double G = 0.0, g = 1.0;
      bool terminal = false;
      for (int k = 1; k <= t.n; ++k) {
        const size_t o = (size_t)(r + k) * B + b;
        G += g * (double)__ldg(t.reward + o);
        if (t.done[o]) { terminal = true; break; }
        g *= (double)t.gamma;
      }
      if (!terminal) {
        const double qt = (double)__ldg(t.q_tg + ((size_t)i * B + b) * A + a_star);
        G += g * (t.rescale ? rescale_h_inv(qt, t.rescale_eps) : qt);
      }
      const float y = (float)(t.rescale ? rescale_h(G, t.rescale_eps) : G);
      const float d = __fsub_rn(q, y);
      const size_t row = (size_t)i * B + b;
      t.q_taken[row] = q; t.y[row] = y; t.delta[row] = d;
      const float dq = t.two_over_BT * w * d;       // d loss / d Q_online(s_t, a_t): y is detached
      for (int a = 0; a < A; ++a) t.dq[row * A + a] = a == act ? dq : 0.f;
      dmax = fmax(dmax, (double)fabsf(d));
      dsum += (double)fabsf(d);
      d2 = __fadd_rn(d2, __fmul_rn(d, d));
    }
    dmax = warp_max_d(dmax);
    dsum = warp_sum_d(dsum);
    d2 = warp_sum(d2);
    if (lane == 0) t.prio[b] = t.eta * dmax + (1.0 - t.eta) * (dsum / (double)t.T) + t.priority_eps;
    l = __fmul_rn(w, d2);
  }
  tail_loss(l, t.B * t.T, t.scratch, t.loss);
}

// the head rows' gradients of one dQ row (lane a holds dQ_a, a < A), uniform over the warp: plain, G_r = dQ_r; dueling, G_0 = s =
// sum_a dQ_a (in action order) and G_{1+a} = dQ_a - s / A
template <bool DUELING>
SRL_DEVINL float head_row_grad(float g, float s, int A, int r) {
  if constexpr (!DUELING) return __shfl_sync(0xffffffffu, g, r);
  const float ga = __shfl_sync(0xffffffffu, g, r > 0 ? r - 1 : 0);
  return r == 0 ? s : __fsub_rn(ga, __fdiv_rn(s, (float)A));
}

// one warp per row n < N_all: dout[n] = sum_r G_r W_r (one fmaf chain per column in r order); rows >= N_train (the bootstrap rows) are 0
template <bool DUELING>
__global__ void __launch_bounds__(128) r2d2_head_dcore_kernel(const R2Head h, const float* __restrict__ dq, int N_train, int N_all,
                                                              float* __restrict__ dout) {
  const int lane = threadIdx.x & 31, n = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (n >= N_all) return;
  const int K = h.K, A = h.A, R = DUELING ? A + 1 : A;
  float* o = dout + (size_t)n * K;
  if (n >= N_train) {
    for (int j = lane; j < K; j += 32) o[j] = 0.f;
    return;
  }
  const float g = lane < A ? __ldg(dq + (size_t)n * A + lane) : 0.f;
  float s = 0.f;
  if (DUELING)
    for (int a = 0; a < A; ++a) s = __fadd_rn(s, __shfl_sync(0xffffffffu, g, a));
  float acc[R2_KI];
#pragma unroll
  for (int i = 0; i < R2_KI; ++i) acc[i] = 0.f;
  for (int r = 0; r < R; ++r) {
    const float G = head_row_grad<DUELING>(g, s, A, r);
    const float* w = DUELING ? (r == 0 ? h.W : h.Wa + (size_t)(r - 1) * K) : h.W + (size_t)r * K;
#pragma unroll
    for (int i = 0; i < R2_KI; ++i) {
      const int j = lane + 32 * i;
      if (j < K) acc[i] = fmaf(G, __ldg(w + j), acc[i]);
    }
  }
#pragma unroll
  for (int i = 0; i < R2_KI; ++i) {
    const int j = lane + 32 * i;
    if (j < K) o[j] = acc[i];
  }
}

// head weight / bias gradients: thread = one column j of X (j == K: the bias "ones" column), blockIdx.y = a group of consecutive slabs
// of R2_SLAB rows; group g writes part[g][r][j] = sum over its rows of G_r x_j, one fmaf chain in row order
template <bool DUELING>
__global__ void __launch_bounds__(128) r2d2_head_wgrad_kernel(const float* __restrict__ dq, const float* __restrict__ X, int N, int A, int K,
                                                              int slabs_per_group, float* __restrict__ part) {
  __shared__ float sd[R2_SLAB][R2_MAX_R];
  __shared__ float ssum[R2_SLAB];
  const int R = DUELING ? A + 1 : A;
  const int j = blockIdx.x * 128 + threadIdx.x;
  const int nslab = (N + R2_SLAB - 1) / R2_SLAB;
  const int s0 = blockIdx.y * slabs_per_group, s1 = min(nslab, s0 + slabs_per_group);
  float acc[R2_MAX_R];
#pragma unroll
  for (int a = 0; a < R2_MAX_R; ++a) acc[a] = 0.f;
  for (int sl = s0; sl < s1; ++sl) {
    const int n0 = sl * R2_SLAB, cnt = min(R2_SLAB, N - n0);
    __syncthreads();                 // the previous slab's shared rows have been read
    if (DUELING && threadIdx.x < R2_SLAB) {
      float s = 0.f;
      if ((int)threadIdx.x < cnt)
        for (int a = 0; a < A; ++a) s = __fadd_rn(s, __ldg(dq + (size_t)(n0 + threadIdx.x) * A + a));
      ssum[threadIdx.x] = s;
    }
    if (DUELING) __syncthreads();
    for (int i = threadIdx.x; i < R2_SLAB * R; i += 128) {     // rows past the ragged end are zero
      const int r = i / R, a = i - r * R;
      float g = 0.f;
      if (r < cnt) {
        if constexpr (!DUELING) g = __ldg(dq + (size_t)(n0 + r) * A + a);
        else g = a == 0 ? ssum[r] : __fsub_rn(__ldg(dq + (size_t)(n0 + r) * A + a - 1), __fdiv_rn(ssum[r], (float)A));
      }
      sd[r][a] = g;
    }
    __syncthreads();
    if (j > K) continue;
    float c[R2_SLAB];
#pragma unroll
    for (int r = 0; r < R2_SLAB; ++r) c[r] = r < cnt ? (j < K ? __ldg(X + (size_t)(n0 + r) * K + j) : 1.f) : 0.f;
#pragma unroll
    for (int a = 0; a < R2_MAX_R; ++a) {
      if (a >= R) break;
#pragma unroll
      for (int r = 0; r < R2_SLAB; ++r) acc[a] = fmaf(sd[r][a], c[r], acc[a]);
    }
  }
  if (j > K) return;
#pragma unroll
  for (int a = 0; a < R2_MAX_R; ++a)
    if (a < R) part[((size_t)blockIdx.y * R + a) * (K + 1) + j] = acc[a];
}
// the groups' partials added in group order into the head gradients (stored); dueling: row 0 -> value, row 1 + a -> advantage row a
template <bool DUELING>
__global__ void __launch_bounds__(256) r2d2_head_wgrad_reduce_kernel(const float* __restrict__ part, int groups, int A, int K, R2HeadGrad g) {
  const int R = DUELING ? A + 1 : A, C = K + 1, n = R * C, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = 0.f;
  for (int k = 0; k < groups; ++k) s += __ldg(part + (size_t)k * n + i);
  const int r = i / C, j = i - r * C;
  if (DUELING && r > 0) {
    if (j < K) g.gWa[(size_t)(r - 1) * K + j] = s; else g.gba[r - 1] = s;
  } else {
    if (j < K) g.gW[(size_t)r * K + j] = s; else g.gb[r] = s;
  }
}

bool is_dueling(const R2Head& h) { return h.Wa != nullptr; }

cudaError_t r2d2_head_fwd(const R2Head& h, const float* X, int N, float* q, cudaStream_t st) {
  const int blocks = (N + 3) / 4;
  if (is_dueling(h)) r2d2_head_fwd_kernel<true><<<blocks, 128, 0, st>>>(h, X, N, q);
  else r2d2_head_fwd_kernel<false><<<blocks, 128, 0, st>>>(h, X, N, q);
  return cudaGetLastError();
}
cudaError_t r2d2_head_bwd(const R2Head& h, const R2HeadGrad& g, const float* dq, const float* X, int N_train, int N_all, float* dout,
                            float* part, cudaStream_t st) {
  const int blocks = (N_all + 3) / 4, A = h.A, K = h.K, R = is_dueling(h) ? A + 1 : A;
  const int nslab = (N_train + R2_SLAB - 1) / R2_SLAB, spg = (nslab + HEAD_GROUPS - 1) / HEAD_GROUPS, groups = (nslab + spg - 1) / spg;
  const dim3 grid((K + 1 + 127) / 128, groups);
  if (is_dueling(h)) {
    r2d2_head_dcore_kernel<true><<<blocks, 128, 0, st>>>(h, dq, N_train, N_all, dout);
    r2d2_head_wgrad_kernel<true><<<grid, 128, 0, st>>>(dq, X, N_train, A, K, spg, part);
    r2d2_head_wgrad_reduce_kernel<true><<<(R * (K + 1) + 255) / 256, 256, 0, st>>>(part, groups, A, K, g);
  } else {
    r2d2_head_dcore_kernel<false><<<blocks, 128, 0, st>>>(h, dq, N_train, N_all, dout);
    r2d2_head_wgrad_kernel<false><<<grid, 128, 0, st>>>(dq, X, N_train, A, K, spg, part);
    r2d2_head_wgrad_reduce_kernel<false><<<(R * (K + 1) + 255) / 256, 256, 0, st>>>(part, groups, A, K, g);
  }
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------- host side
// The tensors in state_dict order: conv1..3 and fc {weight, bias} (8), rnn_layer {weight_ih, weight_hh, bias_ih, bias_hh} x 2 layers
// (8), then q {weight [A][H], bias [A]} or value {weight [1][H], bias [1]} and advantage {weight [A][H], bias [A]}; in memory in that
// order, each segment padded to 4 floats.
int64_t r2d2_layout(int A, int dueling, int64_t* off, int64_t* cnt) {
  const int64_t H = 513 + A, G = 4 * H;
  int64_t c[20] = {32 * 4 * 8 * 8, 32, 64 * 32 * 4 * 4, 64, 64 * 64 * 3 * 3, 64, 512 * 3136, 512,
                   G * H, G * H, G, G, G * H, G * H, G, G};
  int n = 16;
  if (dueling) { c[n++] = H; c[n++] = 1; c[n++] = A * H; c[n++] = A; }
  else { c[n++] = A * H; c[n++] = A; }
  int64_t o = 0;
  for (int i = 0; i < n; ++i) {
    if (off) off[i] = o;
    if (cnt) cnt[i] = c[i];
    o += (c[i] + 3) & ~int64_t(3);
  }
  return o;
}

// one network on a flat buffer (parameters or gradients)
struct R2Net {
  float* enc[8];
  float* lstm[8];
  R2Head head;
  R2HeadGrad grad;
};
R2Net bind_r2d2(int A, int dueling, float* base) {
  int64_t off[20];
  r2d2_layout(A, dueling, off, nullptr);
  R2Net n = {};
  for (int i = 0; i < 8; ++i) { n.enc[i] = base + off[i]; n.lstm[i] = base + off[8 + i]; }
  float* h[4] = {base + off[16], base + off[17], dueling ? base + off[18] : nullptr, dueling ? base + off[19] : nullptr};
  n.head = R2Head{h[0], h[1], h[2], h[3], A, 513 + A};
  n.grad = R2HeadGrad{h[0], h[1], h[2], h[3]};
  return n;
}

}  // namespace
}  // namespace srl

using namespace srl;

struct srl_r2d2_learner {
  srl_r2d2_config_t cfg;
  float *params, *grads, *m, *v, *target;
  int64_t nparams;
  R2Net net[3];                   // online, target, gradients
  srl_encoder_t *E, *Eq;          // the step's encoder context and the q-value forwards' own
  int QF;                         // frames of one q-value chunk
  // encoder and LSTM blocks: *_keep = the online forward over rows burn_in .. L - 1 (read by the backward), *_tmp = the burn-in and
  // target forwards; *_q = the q-value forwards'
  char *enc_keep, *enc_tmp, *enc_scratch, *lstm_keep, *lstm_tmp, *lstm_scratch;
  char *enc_q, *enc_scratch_q, *lstm_q, *lstm_scratch_q;
  float *core, *out_on, *out_tg, *hb, *cb, *hx, *cx, *q_on, *q_tg, *dq, *dout, *dcore;
  float *q_taken, *y, *delta, *loss, *tail_scratch, *head_part, *coef, *opt_scratch;
  float *core_q, *out_q, *state_q;
  double* prio;
  int* dstep;
  char* arena;
};

namespace {
struct R2Blocks {
  int64_t enc_keep, enc_tmp, enc_scratch, lstm_keep, lstm_tmp, lstm_scratch, enc_q, enc_scratch_q, lstm_q, lstm_scratch_q;
};
int r2d2_blocks(const srl_r2d2_config_t& c, int QF, R2Blocks* k) {
  const int B = c.B, L = c.burn_in + c.T + c.n_step, M = c.T + c.n_step;
  int64_t dummy;
  int rc = srl_encoder_sizes(M * B, 0, &k->enc_keep, &dummy);
  if (!rc) rc = srl_encoder_sizes(L * B, 0, &k->enc_tmp, &k->enc_scratch);
  if (!rc) rc = srl_lstm_core_sizes(M, B, c.A, &k->lstm_keep, &dummy);
  if (!rc) rc = srl_lstm_core_sizes(L, B, c.A, &k->lstm_tmp, &k->lstm_scratch);
  if (!rc) rc = srl_encoder_sizes(QF, 0, &k->enc_q, &k->enc_scratch_q);
  if (!rc) rc = srl_lstm_core_sizes(1, QF, c.A, &k->lstm_q, &k->lstm_scratch_q);     // covers every rows x N <= QF chunk
  return rc;
}
// the context's device buffers in carving order; rows with a name are what srl_r2d2_learner_debug_buffer lends
int r2d2_rows(srl_r2d2_learner* L, const R2Blocks& k, WsRow* t) {
  const srl_r2d2_config_t& c = L->cfg;
  const int64_t B = c.B, A = c.A, H = 513 + A, T = c.T, M = c.T + c.n_step, Lr = c.burn_in + M, QF = L->QF;
  const int64_t R = c.dueling ? A + 1 : A;
  int n = 0;
  t[n++] = ws_row<char>(nullptr, k.enc_keep, &L->enc_keep);
  t[n++] = ws_row<char>(nullptr, k.enc_tmp, &L->enc_tmp);
  t[n++] = ws_row<char>(nullptr, k.enc_scratch, &L->enc_scratch);
  t[n++] = ws_row<char>(nullptr, k.lstm_keep, &L->lstm_keep);
  t[n++] = ws_row<char>(nullptr, k.lstm_tmp, &L->lstm_tmp);
  t[n++] = ws_row<char>(nullptr, k.lstm_scratch, &L->lstm_scratch);
  t[n++] = ws_row<char>(nullptr, k.enc_q, &L->enc_q);
  t[n++] = ws_row<char>(nullptr, k.enc_scratch_q, &L->enc_scratch_q);
  t[n++] = ws_row<char>(nullptr, k.lstm_q, &L->lstm_q);
  t[n++] = ws_row<char>(nullptr, k.lstm_scratch_q, &L->lstm_scratch_q);
  t[n++] = ws_row("core", Lr * B * H, &L->core);
  t[n++] = ws_row("out_online", M * B * H, &L->out_on);
  t[n++] = ws_row("out_target", Lr * B * H, &L->out_tg);
  t[n++] = ws_row("h_burn_in", 2 * B * H, &L->hb);
  t[n++] = ws_row("c_burn_in", 2 * B * H, &L->cb);
  t[n++] = ws_row(nullptr, 2 * B * H, &L->hx);
  t[n++] = ws_row(nullptr, 2 * B * H, &L->cx);
  t[n++] = ws_row("q_online", M * B * A, &L->q_on);
  t[n++] = ws_row("q_target", T * B * A, &L->q_tg);
  t[n++] = ws_row("dq", T * B * A, &L->dq);
  t[n++] = ws_row("dout", M * B * H, &L->dout);
  t[n++] = ws_row("dcore", M * B * H, &L->dcore);
  t[n++] = ws_row("q_taken", T * B, &L->q_taken);
  t[n++] = ws_row("y", T * B, &L->y);
  t[n++] = ws_row("delta", T * B, &L->delta);
  t[n++] = ws_row("priorities", B, &L->prio);
  t[n++] = ws_row("loss", 4, &L->loss);
  t[n++] = ws_row("step", 4, &L->dstep);
  t[n++] = ws_row(nullptr, 4 + dqn_tail_blocks((int)B), &L->tail_scratch);
  t[n++] = ws_row(nullptr, HEAD_GROUPS * R * (H + 1), &L->head_part);
  t[n++] = ws_row(nullptr, 4, &L->coef);
  t[n++] = ws_row(nullptr, 2048, &L->opt_scratch);
  t[n++] = ws_row(nullptr, QF * H, &L->core_q);
  t[n++] = ws_row(nullptr, QF * H, &L->out_q);
  t[n++] = ws_row(nullptr, 4 * 2 * QF * H, &L->state_q);     // two (h, c) pairs the q-value chunks pass the state through
  return n;
}
constexpr int R2_ROWS = 35;

int check_r2d2_cfg(const srl_r2d2_config_t* c) {
  REQ(c, "r2d2_learner: config is NULL");
  REQ(c->A >= 1 && c->A <= 31, "r2d2_learner: A=%d must be in [1,31]", c->A);
  REQ(c->B >= 1 && c->burn_in >= 0 && c->T >= 1 && c->n_step >= 1, "r2d2_learner: need B >= 1, burn_in >= 0, T >= 1 and n_step >= 1 "
      "(B=%d, burn_in=%d, T=%d, n_step=%d)", c->B, c->burn_in, c->T, c->n_step);
  const int64_t L = (int64_t)c->burn_in + c->T + c->n_step;
  REQ(L * c->B <= MAX_FRAMES, "r2d2_learner: (burn_in + T + n_step) * B = %lld frames must be <= %d", (long long)(L * c->B), MAX_FRAMES);
  REQ(std::isfinite(c->gamma) && c->gamma >= 0.f && c->gamma <= 1.f, "r2d2_learner: gamma=%g must be in [0, 1]", (double)c->gamma);
  REQ(c->dueling == 0 || c->dueling == 1, "r2d2_learner: dueling must be 0 or 1");
  REQ(c->value_rescaling == 0 || c->value_rescaling == 1, "r2d2_learner: value_rescaling must be 0 or 1");
  REQ(!c->value_rescaling || (std::isfinite(c->rescale_eps) && c->rescale_eps > 0.f), "r2d2_learner: rescale_eps=%g must be finite and > 0",
      (double)c->rescale_eps);
  REQ(c->priority_eta >= 0.f && c->priority_eta <= 1.f, "r2d2_learner: priority_eta=%g must be in [0, 1]", (double)c->priority_eta);
  REQ(std::isfinite(c->priority_eps) && c->priority_eps >= 0.f, "r2d2_learner: priority_eps=%g must be finite and >= 0", (double)c->priority_eps);
  REQ(c->max_grad_norm > 0.f, "r2d2_learner: max_grad_norm=%g must be > 0 (+inf: no clipping)", (double)c->max_grad_norm);
  REQ(std::isfinite(c->learning_rate) && c->learning_rate > 0.f, "r2d2_learner: learning_rate=%g must be finite and > 0", (double)c->learning_rate);
  REQ(c->adam_beta1 >= 0.f && c->adam_beta1 < 1.f && c->adam_beta2 >= 0.f && c->adam_beta2 < 1.f, "r2d2_learner: Adam betas must be in [0, 1)");
  REQ(std::isfinite(c->adam_eps) && c->adam_eps >= 0.f, "r2d2_learner: adam_eps=%g must be finite and >= 0", (double)c->adam_eps);
  return 0;
}
}  // namespace

extern "C" int64_t srl_r2d2_param_layout(int A, int dueling, int64_t* offsets20, int64_t* counts20) {
  REQ(A >= 1 && A <= 31, "r2d2_param_layout: A=%d must be in [1,31]", A);
  REQ(dueling == 0 || dueling == 1, "r2d2_param_layout: dueling=%d must be 0 or 1", dueling);
  return r2d2_layout(A, dueling, offsets20, counts20);
}

extern "C" int srl_r2d2_learner_create(const srl_r2d2_config_t* cfg, float* params, float* grads, float* exp_avg, float* exp_avg_sq,
                                       float* target_params, srl_r2d2_learner_t** out) {
  int rc = check_r2d2_cfg(cfg);
  if (rc) return rc;
  REQ(params && grads && exp_avg && exp_avg_sq && target_params && out, "r2d2_learner_create: NULL argument");
  REQ(!misaligned(params, 16) && !misaligned(grads, 16) && !misaligned(exp_avg, 16) && !misaligned(exp_avg_sq, 16) &&
      !misaligned(target_params, 16), "r2d2_learner_create: flat buffers must be 16-byte aligned");
  const int64_t np = r2d2_layout(cfg->A, cfg->dueling, nullptr, nullptr);
  const Span s[5] = {{params, np * 4, true, "params"}, {grads, np * 4, true, "grads"}, {exp_avg, np * 4, true, "exp_avg"},
                     {exp_avg_sq, np * 4, true, "exp_avg_sq"}, {target_params, np * 4, true, "target_params"}};
  rc = check_spans(s, 5, "r2d2_learner_create");
  if (rc) return rc;
  srl_r2d2_learner* L = new (std::nothrow) srl_r2d2_learner();
  REQ(L, "out of host memory");
  auto undo = [L](int code) { srl_r2d2_learner_destroy(L); return code; };
  L->cfg = *cfg; L->params = params; L->grads = grads; L->m = exp_avg; L->v = exp_avg_sq; L->target = target_params; L->nparams = np;
  L->net[0] = bind_r2d2(cfg->A, cfg->dueling, params);
  L->net[1] = bind_r2d2(cfg->A, cfg->dueling, target_params);
  L->net[2] = bind_r2d2(cfg->A, cfg->dueling, grads);
  const int frames = (cfg->burn_in + cfg->T + cfg->n_step) * cfg->B;
  L->QF = frames < R2_QF ? frames : R2_QF;
  rc = srl_encoder_create(0, &L->E);
  if (!rc) rc = srl_encoder_create(0, &L->Eq);
  if (rc) return undo(rc);
  R2Blocks k;
  rc = r2d2_blocks(*cfg, L->QF, &k);
  if (rc) return undo(rc);
  WsRow t[R2_ROWS];
  const int n = r2d2_rows(L, k, t);
  const int64_t total = rows_bytes(t, n, false);
  cudaError_t e = cudaMalloc(&L->arena, total);
  if (e != cudaSuccess) return undo(cuda_fail(e, "r2d2_learner_create: cudaMalloc workspace"));
  e = cudaMemset(L->arena, 0, total);        // the tail's ticket and the step count
  if (e == cudaSuccess) e = cudaMemset(grads, 0, np * 4);      // the padding between the segments enters the gradient norm
  if (e != cudaSuccess) return undo(cuda_fail(e, "r2d2_learner_create: cudaMemset"));
  carve_rows(t, n, false, L->arena);
  *out = L;
  return 0;
}

extern "C" int srl_r2d2_learner_destroy(srl_r2d2_learner_t* L) {
  if (!L) return 0;
  srl_encoder_destroy(L->E);
  srl_encoder_destroy(L->Eq);
  cudaFree(L->arena);
  delete L;
  return 0;
}

extern "C" int srl_r2d2_learner_step(srl_r2d2_learner_t* L, const uint8_t* frame, const int64_t* last_action, const float* reward,
                                     const uint8_t* done, const float* h0, const float* c0, const float* weights, const int64_t* idxs,
                                     srl_per_t* per, float* stats_out, void* stream) {
  REQ(L && frame && last_action && reward && done && h0 && c0, "r2d2_learner_step: NULL pointer");
  REQ(!idxs == !per, "r2d2_learner_step: idxs and per go together (both NULL or both set)");
  const srl_r2d2_config_t& c = L->cfg;
  const int B = c.B, A = c.A, H = 513 + A, bi = c.burn_in, T = c.T, n = c.n_step, M = T + n, Lr = bi + M;
  const int64_t F = 28224;          // bytes of one 4 x 84 x 84 frame stack
  const cudaStream_t st = (cudaStream_t)stream;
  const R2Net &on = L->net[0], &tg = L->net[1], &gr = L->net[2];
  int rc = 0;
  // the burn-in: rows 0 .. burn_in - 1 through the online network from the stored state, no gradient
  const float *hs = h0, *cs = c0;
  if (bi > 0) {
    rc = srl_encoder_forward(L->E, frame, reward, last_action, bi * B, A, on.enc, L->enc_tmp, L->enc_scratch, L->core, stream);
    if (!rc) rc = srl_lstm_core_forward(L->core, done, h0, c0, A, bi, B, on.lstm, L->lstm_tmp, L->lstm_scratch, L->out_tg, L->hb, L->cb,
                                        stream);
    if (rc) return rc;
    hs = L->hb; cs = L->cb;
  }
  // the online forward over rows burn_in .. L - 1 (trained rows and bootstrap rows), its blocks kept for the backward
  const size_t o = (size_t)bi * B;
  rc = srl_encoder_forward(L->E, frame + o * F, reward + o, last_action + o, M * B, A, on.enc, L->enc_keep, L->enc_scratch, L->core, stream);
  if (!rc) rc = srl_lstm_core_forward(L->core, done + o, hs, cs, A, M, B, on.lstm, L->lstm_keep, L->lstm_scratch, L->out_on, L->hx, L->cx,
                                      stream);
  // the target network over all L rows from the stored state
  if (!rc) rc = srl_encoder_forward(L->E, frame, reward, last_action, Lr * B, A, tg.enc, L->enc_tmp, L->enc_scratch, L->core, stream);
  if (!rc) rc = srl_lstm_core_forward(L->core, done, h0, c0, A, Lr, B, tg.lstm, L->lstm_tmp, L->lstm_scratch, L->out_tg, L->hx, L->cx,
                                      stream);
  if (rc) return rc;
  CU(r2d2_head_fwd(on.head, L->out_on, M * B, L->q_on, st), "r2d2_head_fwd online");
  CU(r2d2_head_fwd(tg.head, L->out_tg + (size_t)(bi + n) * B * H, T * B, L->q_tg, st), "r2d2_head_fwd target");
  const R2Tail tail = {L->q_on, L->q_tg, last_action, reward, done, weights, B, A, bi, T, n, c.gamma, c.value_rescaling,
                       (double)c.rescale_eps, (double)c.priority_eta, (double)c.priority_eps, 2.f / (float)(B * T),
                       L->q_taken, L->y, L->delta, L->dq, L->loss, L->tail_scratch, L->prio};
  r2d2_tail_kernel<<<dqn_tail_blocks(B), 128, 0, st>>>(tail);
  CU(cudaGetLastError(), "r2d2_tail");
  CU(r2d2_head_bwd(on.head, gr.grad, L->dq, L->out_on, T * B, M * B, L->dout, L->head_part, st), "r2d2_head_bwd");
  // BPTT over the kept rows (dout is zero on the bootstrap rows; no gradient reaches the stored or burnt-in state), then the encoder
  rc = srl_lstm_core_backward(L->dout, nullptr, nullptr, A, M, B, L->lstm_keep, L->lstm_scratch, gr.lstm, L->dcore, nullptr, nullptr, stream);
  if (!rc) rc = srl_encoder_backward(L->E, L->dcore, M * B, A, L->enc_keep, L->enc_scratch, gr.enc, stream);
  if (rc) return rc;
  const OptStep opt = {1, L->params, L->grads, L->m, L->v, L->nparams, c.max_grad_norm, L->coef, L->opt_scratch, c.learning_rate,
                       c.adam_beta1, c.adam_beta2, c.adam_eps, 0, L->dstep, OptExtra{}};
  CU(launch_clip_optim(opt, st), "clip+adam");
  if (per) {
    rc = srl_per_update_priorities(per, idxs, L->prio, B, stream);
    if (rc) return rc;
  }
  if (stats_out) {
    CU(cudaMemcpyAsync(stats_out, L->loss, sizeof(float), cudaMemcpyDeviceToDevice, st), "copy loss");
    CU(cudaMemcpyAsync(stats_out + 1, L->coef, 2 * sizeof(float), cudaMemcpyDeviceToDevice, st), "copy coef");
  }
  return 0;
}

extern "C" int srl_r2d2_learner_q_values(srl_r2d2_learner_t* L, const uint8_t* frame, const int64_t* last_action, const float* reward,
                                         const uint8_t* done, int T1, int N, const float* h0, const float* c0, float* q_out, float* hT,
                                         float* cT, void* stream) {
  REQ(L && frame && last_action && reward && done && h0 && c0 && q_out && hT && cT, "r2d2_learner_q_values: NULL pointer");
  REQ(T1 >= 1 && N >= 1 && N <= L->QF, "r2d2_learner_q_values: T1=%d, N=%d: need T1 >= 1 and 1 <= N <= %d", T1, N, L->QF);
  const int A = L->cfg.A, H = 513 + A;
  const int64_t rows = (int64_t)T1 * N, state = (int64_t)2 * N * H * 4;
  const Span s[9] = {{frame, rows * 28224, false, "frame"}, {last_action, rows * 8, false, "last_action"}, {reward, rows * 4, false, "reward"},
                      {done, rows, false, "done"}, {h0, state, false, "h0"}, {c0, state, false, "c0"},
                      {q_out, rows * A * 4, true, "q_out"}, {hT, state, true, "hT"}, {cT, state, true, "cT"}};
  int rc = check_spans(s, 9, "r2d2_learner_q_values");
  if (rc) return rc;
  const R2Net& on = L->net[0];
  const int per_chunk = L->QF / N;
  const size_t sq = (size_t)2 * N * H;
  const float *hs = h0, *cs = c0;
  for (int r0 = 0, k = 0; r0 < T1; r0 += per_chunk, ++k) {
    const int r = T1 - r0 < per_chunk ? T1 - r0 : per_chunk;
    const bool last = r0 + r >= T1;
    float* ho = last ? hT : L->state_q + (size_t)(k & 1) * 2 * sq;       // ping-pong between the two internal (h, c) pairs
    float* co = last ? cT : ho + sq;
    const size_t f = (size_t)r0 * N;
    rc = srl_encoder_forward(L->Eq, frame + f * 28224, reward + f, last_action + f, r * N, A, on.enc, L->enc_q, L->enc_scratch_q, L->core_q,
                             stream);
    if (!rc) rc = srl_lstm_core_forward(L->core_q, done + f, hs, cs, A, r, N, on.lstm, L->lstm_q, L->lstm_scratch_q, L->out_q, ho, co, stream);
    if (rc) return rc;
    CU(r2d2_head_fwd(on.head, L->out_q, r * N, q_out + f * A, (cudaStream_t)stream), "r2d2_head_fwd");
    hs = ho; cs = co;
  }
  return 0;
}

extern "C" int srl_r2d2_learner_update_target(srl_r2d2_learner_t* L, float tau, void* stream) {
  REQ(L, "r2d2_learner_update_target: learner is NULL");
  REQ(tau >= 0.f && tau <= 1.f, "r2d2_learner_update_target: tau=%g must be in [0, 1]", (double)tau);
  CU(launch_apex_soft_update(L->params, L->target, L->nparams, tau, (float)(1.0 - (double)tau), (cudaStream_t)stream), "apex_soft_update");
  return 0;
}

extern "C" int srl_r2d2_learner_set_step(srl_r2d2_learner_t* L, int64_t step, void* stream) {
  REQ(L && step >= 0 && step < (int64_t(1) << 31), "r2d2_learner_set_step: bad argument");
  const int v = (int)step;
  CU(cudaMemcpyAsync(L->dstep, &v, sizeof(int), cudaMemcpyHostToDevice, (cudaStream_t)stream), "r2d2_learner_set_step");
  CU(cudaStreamSynchronize((cudaStream_t)stream), "r2d2_learner_set_step");      // `v` is a stack variable
  return 0;
}

extern "C" int srl_r2d2_learner_debug_buffer(srl_r2d2_learner_t* L, const char* name, void** ptr, int64_t* count) {
  REQ(L && name && ptr && count, "r2d2_learner_debug_buffer: NULL argument");
  R2Blocks k;
  int rc = r2d2_blocks(L->cfg, L->QF, &k);
  if (rc) return rc;
  srl_r2d2_learner shadow = *L;        // the table's rows re-derived on a copy: the same sizes give the same addresses
  WsRow t[R2_ROWS];
  const int n = r2d2_rows(&shadow, k, t);
  carve_rows(t, n, false, L->arena);
  for (int i = 0; i < n; ++i)
    if (t[i].name && strcmp(t[i].name, name) == 0 && t[i].count > 0) { *ptr = *t[i].hi; *count = t[i].count; return 0; }
  return fail(SRL_EINVAL, "r2d2_learner_debug_buffer: unknown buffer '%s'", name);
}
