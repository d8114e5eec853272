// V-trace kernels (reference: scalerl/algorithms/impala/vtrace.py) and the fused learner tail
// (impala_atari.py:293-330 + loss_fn.py:5-23 + head gradients).  All fp32, HBM/latency bound.
//
//   vtrace_iw_seq_kernel<VEC>  column-sequential reverse recursion, lanes along B (coalesced; float4 when VEC=4)
//   vtrace_iw_scan_kernel      [T x 32] tile staged through shared memory, lane = t, Kogge-Stone scan of the
//                              affine maps x -> delta_t + (gamma_t c_t) x with warp shuffles, 32-step chunks + carry
//   vtrace_logits_kernel       from_logits (log-softmax gather for both policies, then the recursion)
//   impala_tail_kernel         one pass over the [T+1,B] batch rows: shifts, reward clip, discounts, V-trace,
//                              pg/baseline/entropy losses (deterministic two-level reduction), dlogits, dbaseline
//   impala_tail_warp_kernel    the same tail with one warp per column (tail_column_warp), for B <= 2048
// Shared device pieces (a copy that stays written out says why at the copy: through the helper, that kernel compiles differently):
//   row_lse / row_logp / row_entropy   log-softmax and sum_a p log p of one row: impala_tail_kernel, policy row operators
//   scan_compose                       the warp's Kogge-Stone suffix composition: vtrace_iw_scan_kernel, tail_column_warp
//   tail_reward_discount               the tail's per-step reward clip and discount: impala_tail_kernel, tail_column_warp
//   publish_block_partials             a 4-warp block's loss partials and its ticket: both tail kernels
//   take_ticket / write_losses         the reduction's ticket, and the losses with the re-armed ticket: also column_step_kernel
// Each reducing kernel keeps its own final summation order.  The sequential V-trace step stays written out in its three kernels.
#include "common.cuh"
#include "kernels.h"

namespace srl {

template <int VEC>
SRL_DEVINL void ldv(const float* p, float (&o)[VEC]) {
  if (VEC == 4) { float4 t = __ldg(reinterpret_cast<const float4*>(p)); o[0] = t.x; o[1 % VEC] = t.y; o[2 % VEC] = t.z; o[3 % VEC] = t.w; }
  else o[0] = __ldg(p);
}
template <int VEC>
SRL_DEVINL void stv(float* p, const float (&o)[VEC]) {
  if (VEC == 4) *reinterpret_cast<float4*>(p) = make_float4(o[0], o[1 % VEC], o[2 % VEC], o[3 % VEC]);
  else *p = o[0];
}

// Element loads of the row helpers: NC = true reads global memory through the read-only path (ld.global.nc), NC = false is a plain
// load (the shared-memory copies of the column kernel).
template <bool NC>
SRL_DEVINL float ldf(const float* p) { return NC ? __ldg(p) : *p; }
// log_softmax of one row of A logits (vtrace.py:31-40): log p[a] = (x[a] - mx) - lse
struct RowLse { float mx, lse; };
template <bool NC>
SRL_DEVINL RowLse row_lse(const float* row, int A) {
  float mx = -INFINITY;
  for (int a = 0; a < A; ++a) mx = fmaxf(mx, ldf<NC>(row + a));
  float se = 0.f;
  for (int a = 0; a < A; ++a) se += expf(ldf<NC>(row + a) - mx);
  return {mx, logf(se)};
}
template <bool NC>
SRL_DEVINL float row_logp(const float* row, RowLse s, int a) { return (ldf<NC>(row + a) - s.mx) - s.lse; }
template <bool NC>
SRL_DEVINL float row_entropy(const float* row, RowLse s, int A) {   // sum_a p log p (loss_fn.py:9-13)
  float e = 0.f;
  for (int a = 0; a < A; ++a) { const float lp = row_logp<NC>(row, s, a); e += expf(lp) * lp; }
  return e;
}

// Kogge-Stone suffix composition over the warp (lane = step): (aa, bb) becomes F_t = f_t o f_{t+1} o ... o f_{31}
SRL_DEVINL void scan_compose(int lane, float& aa, float& bb) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const float a2 = __shfl_down_sync(0xffffffffu, aa, d);
    const float b2 = __shfl_down_sync(0xffffffffu, bb, d);
    if (lane + d < 32) { bb = fmaf(aa, b2, bb); aa = aa * a2; }
  }
}

// Deterministic loss reduction: scratch[0] counts the blocks that have published their partials (scratch[4 + 3 k ..] for block k).
// One thread per block calls take_ticket (common.cuh) after its stores: true in the block that published last, which sums the
// partials in its kernel's fixed order and calls write_losses.
SRL_DEVINL void write_losses(float* losses, float* scratch, float s_pg, float s_bl, float s_ent, float baseline_cost, float entropy_cost) {
  const float a = s_pg, c = baseline_cost * s_bl, e = entropy_cost * s_ent;
  losses[0] = a; losses[1] = c; losses[2] = e; losses[3] = a + c + e;
  *reinterpret_cast<unsigned*>(scratch) = 0u;   // re-arm the ticket
}

// per-step tail input: the reward (clipped to [-1, 1] when clip_reward) and the discount of trajectory row o1
SRL_DEVINL void tail_reward_discount(const float* __restrict__ reward, const uint8_t* __restrict__ done, size_t o1, float discounting,
                                     int clip_reward, float& r, float& g) {
  r = __ldg(reward + o1);
  if (clip_reward) r = fminf(fmaxf(r, -1.f), 1.f);
  g = done[o1] ? 0.f : discounting;
}

// the loss partials of a block of 4 warps: warp sums, then (w0 + w1) + (w2 + w3) per loss into the block's slot, then the ticket.
// Returns true, in every thread, in the block that published last.
SRL_DEVINL bool publish_block_partials(float* scratch, float l_pg, float l_bl, float l_ent) {
  __shared__ float red[3][4];
  __shared__ bool is_last;
  l_pg = warp_sum(l_pg); l_bl = warp_sum(l_bl); l_ent = warp_sum(l_ent);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { red[0][warp] = l_pg; red[1][warp] = l_bl; red[2][warp] = l_ent; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 0; i < 3; ++i) scratch[4 + blockIdx.x * 3 + i] = (red[i][0] + red[i][1]) + (red[i][2] + red[i][3]);
    is_last = take_ticket(scratch);
  }
  __syncthreads();
  return is_last;
}

// vtrace.py:135-169.  Each thread owns VEC adjacent columns; the reverse loop carries acc and vs_{t+1}.
template <int VEC>
__global__ void __launch_bounds__(128) vtrace_iw_seq_kernel(const float* __restrict__ log_rhos, const float* __restrict__ discounts,
                                                            const float* __restrict__ rewards, const float* __restrict__ values,
                                                            const float* __restrict__ bootstrap, int T, int B, float clip_rho,
                                                            float clip_pg, float* __restrict__ vs, float* __restrict__ pg) {
  const int b = (blockIdx.x * blockDim.x + threadIdx.x) * VEC;
  if (b >= B) return;
  float acc[VEC], vnext[VEC], vsnext[VEC];
  ldv<VEC>(bootstrap + b, vnext);
#pragma unroll
  for (int i = 0; i < VEC; ++i) { acc[i] = 0.f; vsnext[i] = vnext[i]; }
#pragma unroll 4
  for (int t = T - 1; t >= 0; --t) {
    const size_t o = (size_t)t * B + b;
    float lr[VEC], g[VEC], r[VEC], v[VEC], ovs[VEC], opg[VEC];
    ldv<VEC>(log_rhos + o, lr); ldv<VEC>(discounts + o, g); ldv<VEC>(rewards + o, r); ldv<VEC>(values + o, v);
#pragma unroll
    for (int i = 0; i < VEC; ++i) {   // the sequential step, written out here, in vtrace_logits_kernel and in impala_tail_kernel:
                                      // through one shared helper this kernel and impala_tail_kernel compile differently
      const float rho = expf(lr[i]);
      const float crho = clip_rho >= 0.f ? fminf(rho, clip_rho) : rho;
      const float c = fminf(rho, 1.0f);
      const float delta = crho * (r[i] + g[i] * vnext[i] - v[i]);
      acc[i] = delta + g[i] * c * acc[i];
      const float prho = clip_pg >= 0.f ? fminf(rho, clip_pg) : rho;
      opg[i] = prho * (r[i] + g[i] * vsnext[i] - v[i]);
      ovs[i] = acc[i] + v[i];
      vsnext[i] = ovs[i];
      vnext[i] = v[i];
    }
    stv<VEC>(vs + o, ovs);
    stv<VEC>(pg + o, opg);
  }
}

// Warp-shuffle segmented scan variant.  Block = 32 columns x 8 warps (4 columns per warp).
constexpr int SCAN_MAX_T = 128;
__global__ void __launch_bounds__(256) vtrace_iw_scan_kernel(const float* __restrict__ log_rhos, const float* __restrict__ discounts,
                                                             const float* __restrict__ rewards, const float* __restrict__ values,
                                                             const float* __restrict__ bootstrap, int T, int B, float clip_rho,
                                                             float clip_pg, float* __restrict__ vs, float* __restrict__ pg) {
  extern __shared__ float sm[];   // 4 arrays [T][33]
  float* s_lr = sm;
  float* s_g = sm + (size_t)T * 33;
  float* s_r = sm + (size_t)2 * T * 33;
  float* s_v = sm + (size_t)3 * T * 33;
  const int b0 = blockIdx.x * 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // coalesced tile load: lanes along B
  for (int t = warp; t < T; t += 8) {
    const int b = b0 + lane;
    const size_t o = (size_t)t * B + b;
    const bool ok = b < B;
    s_lr[t * 33 + lane] = ok ? __ldg(log_rhos + o) : 0.f;
    s_g[t * 33 + lane] = ok ? __ldg(discounts + o) : 0.f;
    s_r[t * 33 + lane] = ok ? __ldg(rewards + o) : 0.f;
    s_v[t * 33 + lane] = ok ? __ldg(values + o) : 0.f;
  }
  __syncthreads();
  const int nchunk = (T + 31) / 32;
  for (int cc = 0; cc < 4; ++cc) {
    const int c = warp * 4 + cc;
    const int b = b0 + c;
    const float boot = b < B ? __ldg(bootstrap + b) : 0.f;
    float carry_acc = 0.f;        // acc_{t_end} entering the chunk from the future
    float carry_v = boot;         // V_{t_end}
    float carry_vs = boot;        // vs_{t_end}
    for (int ch = nchunk - 1; ch >= 0; --ch) {
      const int t = ch * 32 + lane;
      const bool ok = t < T;
      const float lr = ok ? s_lr[t * 33 + c] : 0.f;
      const float g = ok ? s_g[t * 33 + c] : 0.f;
      const float r = ok ? s_r[t * 33 + c] : 0.f;
      const float v = ok ? s_v[t * 33 + c] : 0.f;
      float vn = __shfl_down_sync(0xffffffffu, v, 1);
      if (lane == 31 || t + 1 >= T) vn = carry_v;
      const float rho = expf(lr);
      const float crho = clip_rho >= 0.f ? fminf(rho, clip_rho) : rho;
      // affine map of this step: x -> bb + aa * x ; identity for padding lanes
      float aa = ok ? g * fminf(rho, 1.0f) : 1.f;
      float bb = ok ? crho * (r + g * vn - v) : 0.f;
      scan_compose(lane, aa, bb);
      const float acc = fmaf(aa, carry_acc, bb);
      const float myvs = acc + v;
      float vsn = __shfl_down_sync(0xffffffffu, myvs, 1);
      if (lane == 31 || t + 1 >= T) vsn = carry_vs;
      const float prho = clip_pg >= 0.f ? fminf(rho, clip_pg) : rho;
      const float mypg = prho * (r + g * vsn - v);
      if (ok) { s_lr[t * 33 + c] = myvs; s_g[t * 33 + c] = mypg; }   // reuse the tiles for the outputs
      carry_acc = __shfl_sync(0xffffffffu, acc, 0);
      carry_v = __shfl_sync(0xffffffffu, v, 0);
      carry_vs = __shfl_sync(0xffffffffu, myvs, 0);
    }
  }
  __syncthreads();
  for (int t = warp; t < T; t += 8) {
    const int b = b0 + lane;
    if (b < B) {
      const size_t o = (size_t)t * B + b;
      vs[o] = s_lr[t * 33 + lane];
      pg[o] = s_g[t * 33 + lane];
    }
  }
}

// log_softmax(logits)[action] for one row of A logits (vtrace.py:31-40).  Written out: through row_lse, which takes the log before
// the gather, vtrace_logits_kernel and the tail kernels compile differently.
SRL_DEVINL float action_logp(const float* __restrict__ row, int A, int act) {
  float mx = -INFINITY;
  for (int a = 0; a < A; ++a) mx = fmaxf(mx, __ldg(row + a));
  float se = 0.f;
  for (int a = 0; a < A; ++a) se += expf(__ldg(row + a) - mx);
  return (__ldg(row + act) - mx) - logf(se);
}

__global__ void __launch_bounds__(128) vtrace_logits_kernel(const float* __restrict__ bl, const float* __restrict__ tl,
                                                            const int64_t* __restrict__ actions, const float* __restrict__ discounts,
                                                            const float* __restrict__ rewards, const float* __restrict__ values,
                                                            const float* __restrict__ bootstrap, int T, int B, int A, float clip_rho,
                                                            float clip_pg, float* __restrict__ vs, float* __restrict__ pg,
                                                            float* __restrict__ o_lr, float* __restrict__ o_balp, float* __restrict__ o_talp) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float acc = 0.f, vnext = __ldg(bootstrap + b), vsnext = vnext;
  for (int t = T - 1; t >= 0; --t) {
    const size_t o = (size_t)t * B + b;
    const int act = ld_action(actions + o, A);
    const float talp = action_logp(tl + o * A, A, act);
    const float balp = action_logp(bl + o * A, A, act);
    const float lr = talp - balp;
    const float g = __ldg(discounts + o), r = __ldg(rewards + o), v = __ldg(values + o);
    const float rho = expf(lr);   // the sequential step, also in vtrace_iw_seq_kernel and impala_tail_kernel (see there)
    const float crho = clip_rho >= 0.f ? fminf(rho, clip_rho) : rho;
    acc = crho * (r + g * vnext - v) + g * fminf(rho, 1.0f) * acc;
    const float prho = clip_pg >= 0.f ? fminf(rho, clip_pg) : rho;
    pg[o] = prho * (r + g * vsnext - v);
    vsnext = acc + v;
    vs[o] = vsnext;
    vnext = v;
    if (o_lr) o_lr[o] = lr;
    if (o_balp) o_balp[o] = balp;
    if (o_talp) o_talp[o] = talp;
  }
}

// Fused learner tail.  One thread per batch column; rows follow the reference's shifts:
//   model outputs (target logits, values) use row t, trajectory fields (behaviour logits, action, reward, done)
//   use row t+1 (impala_atari.py:296-300), bootstrap = baseline[T] (:293).
__global__ void __launch_bounds__(128) impala_tail_kernel(const float* __restrict__ bl, const float* __restrict__ tl,
                                                          const float* __restrict__ baseline, const int64_t* __restrict__ action,
                                                          const float* __restrict__ reward, const uint8_t* __restrict__ done, int T, int B,
                                                          int A, float discounting, int clip_reward, float clip_rho, float clip_pg,
                                                          float baseline_cost, float entropy_cost, float* __restrict__ vs,
                                                          float* __restrict__ pg, float* __restrict__ dlogits, float* __restrict__ dbaseline,
                                                          float* __restrict__ losses, float* __restrict__ scratch) {
  pdl_wait(44);    // launched with programmatic stream serialization: see common.cuh
  pdl_launch();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  float l_pg = 0.f, l_bl = 0.f, l_ent = 0.f;
  if (b < B) {
    float acc = 0.f;
    float vnext = __ldg(baseline + (size_t)T * B + b);
    float vsnext = vnext;
    for (int t = T - 1; t >= 0; --t) {
      const size_t o = (size_t)t * B + b;        // model row t
      const size_t o1 = o + B;                   // trajectory row t+1
      const int act = ld_action(action + o1, A);
      const float* trow = tl + o * A;
      const RowLse s = row_lse<true>(trow, A);
      const float ent = row_entropy<true>(trow, s, A);
      const float talp = row_logp<true>(trow, s, act);
      const float balp = action_logp(bl + o1 * A, A, act);
      const float rho = expf(talp - balp);
      float r, g;
      tail_reward_discount(reward, done, o1, discounting, clip_reward, r, g);
      const float v = __ldg(baseline + o);
      const float crho = clip_rho >= 0.f ? fminf(rho, clip_rho) : rho;
      acc = crho * (r + g * vnext - v) + g * fminf(rho, 1.0f) * acc;   // the sequential step: see vtrace_iw_seq_kernel
      const float prho = clip_pg >= 0.f ? fminf(rho, clip_pg) : rho;
      const float adv = prho * (r + g * vsnext - v);
      const float myvs = acc + v;
      // output stage, also in tail_column_warp: written out twice, as through one helper both tail kernels compile differently
      if (vs) vs[o] = myvs;
      if (pg) pg[o] = adv;
      l_pg += -talp * adv;                                   // loss_fn.py:16-23
      l_bl += 0.5f * (myvs - v) * (myvs - v);                // loss_fn.py:5-6
      l_ent += ent;                                          // loss_fn.py:9-13
      dbaseline[o] = -baseline_cost * (myvs - v);
      float* drow = dlogits + o * A;
      for (int a = 0; a < A; ++a) {
        const float lp = row_logp<true>(trow, s, a);
        const float p = expf(lp);
        drow[a] = adv * (p - (a == act ? 1.f : 0.f)) + entropy_cost * p * (lp - ent);
      }
      vsnext = myvs;
      vnext = v;
    }
  }
  if (publish_block_partials(scratch, l_pg, l_bl, l_ent) && threadIdx.x == 0) {
    __threadfence();
    double s[3] = {0, 0, 0};
    for (unsigned k = 0; k < gridDim.x; ++k)
      for (int i = 0; i < 3; ++i) s[i] += (double)reinterpret_cast<volatile float*>(scratch)[4 + k * 3 + i];
    write_losses(losses, scratch, (float)s[0], (float)s[1], (float)s[2], baseline_cost, entropy_cost);
  }
}


// One batch column handled by one warp: lanes = time steps (chunks of 32, walked backwards with an affine carry).
// Target logits / baseline are read through (row pointer, stride) so the same code serves global memory (NC = true: ld.nc)
// and the shared-memory copies of the fused column kernel (NC = false).  sdl (optional): [T][A+1] copy of
// (dlogits..., dbaseline) for the caller.  l_* are per-lane partial loss sums.
// The row arithmetic is written out here: through row_lse / row_entropy / row_logp the warp and column kernels compile differently.
template <bool NC>
SRL_DEVINL void tail_column_warp(const float* __restrict__ bl, const float* trow0, size_t tstride, const float* base0, size_t bstride,
                                 const int64_t* __restrict__ action, const float* __restrict__ reward, const uint8_t* __restrict__ done,
                                 int T, int B, int A, int b, int lane, float discounting, int clip_reward, float clip_rho, float clip_pg,
                                 float baseline_cost, float entropy_cost, float* __restrict__ vs, float* __restrict__ pg,
                                 float* __restrict__ dlogits, float* __restrict__ dbaseline, float* sdl, float& l_pg, float& l_bl,
                                 float& l_ent) {
  const float boot = ldf<NC>(base0 + (size_t)T * bstride);
  float carry_acc = 0.f, carry_vs = boot;
  const int nchunk = (T + 31) >> 5;
  for (int ch = nchunk - 1; ch >= 0; --ch) {
    const int t = ch * 32 + lane;
    const bool ok = t < T;
    const int tt = ok ? t : 0;
    const size_t o = (size_t)tt * B + b, o1 = o + B;
    const int act = ld_action(action + o1, A);
    const float* trow = trow0 + (size_t)tt * tstride;
    float mx = -INFINITY;
    for (int a = 0; a < A; ++a) mx = fmaxf(mx, ldf<NC>(trow + a));
    float se = 0.f;
    for (int a = 0; a < A; ++a) se += expf(ldf<NC>(trow + a) - mx);
    const float lse = logf(se);
    float ent = 0.f;
    for (int a = 0; a < A; ++a) { const float lp = (ldf<NC>(trow + a) - mx) - lse; ent += expf(lp) * lp; }
    const float talp = (ldf<NC>(trow + act) - mx) - lse;
    const float balp = action_logp(bl + o1 * A, A, act);
    const float rho = expf(talp - balp);
    float r, g;
    tail_reward_discount(reward, done, o1, discounting, clip_reward, r, g);
    const float v = ldf<NC>(base0 + (size_t)tt * bstride);
    const float vn = ldf<NC>(base0 + (size_t)(tt + 1) * bstride);     // V_{t+1}; row T is the bootstrap value
    const float crho = clip_rho >= 0.f ? fminf(rho, clip_rho) : rho;
    float aa = ok ? g * fminf(rho, 1.0f) : 1.f;          // x -> bb + aa x ; identity on padding lanes
    float bb = ok ? crho * (r + g * vn - v) : 0.f;
    scan_compose(lane, aa, bb);
    const float acc = fmaf(aa, carry_acc, bb);
    const float myvs = acc + v;
    float vsn = __shfl_down_sync(0xffffffffu, myvs, 1);
    if (lane == 31 || t + 1 >= T) vsn = carry_vs;
    const float prho = clip_pg >= 0.f ? fminf(rho, clip_pg) : rho;
    const float adv = prho * (r + g * vsn - v);
    if (ok) {   // output stage, also in impala_tail_kernel: written out twice, as through one helper both tail kernels compile differently
      if (vs) vs[o] = myvs;
      if (pg) pg[o] = adv;
      l_pg += -talp * adv;
      l_bl += 0.5f * (myvs - v) * (myvs - v);
      l_ent += ent;
      const float dv = -baseline_cost * (myvs - v);
      dbaseline[o] = dv;
      if (sdl) sdl[(size_t)t * (A + 1) + A] = dv;
      float* drow = dlogits + o * A;
      for (int a = 0; a < A; ++a) {
        const float lp = (ldf<NC>(trow + a) - mx) - lse;
        const float p = expf(lp);
        const float d = adv * (p - (a == act ? 1.f : 0.f)) + entropy_cost * p * (lp - ent);
        drow[a] = d;
        if (sdl) sdl[(size_t)t * (A + 1) + a] = d;
      }
    }
    carry_acc = __shfl_sync(0xffffffffu, acc, 0);
    carry_vs = __shfl_sync(0xffffffffu, myvs, 0);
  }
}


// Warp-per-column variant of the fused tail for small B (latency-bound regime): lane = t, the T-step
// recursion becomes a Kogge-Stone scan of affine maps with warp shuffles (32-step chunks + carry), and the
// softmax / log-prob work of all T steps of a column runs in parallel.  Block = 4 warps = 4 columns.
__global__ void __launch_bounds__(128) impala_tail_warp_kernel(const float* __restrict__ bl, const float* __restrict__ tl,
                                                               const float* __restrict__ baseline, const int64_t* __restrict__ action,
                                                               const float* __restrict__ reward, const uint8_t* __restrict__ done, int T,
                                                               int B, int A, float discounting, int clip_reward, float clip_rho,
                                                               float clip_pg, float baseline_cost, float entropy_cost,
                                                               float* __restrict__ vs, float* __restrict__ pg, float* __restrict__ dlogits,
                                                               float* __restrict__ dbaseline, float* __restrict__ losses,
                                                               float* __restrict__ scratch) {
  pdl_wait(45);    // launched with programmatic stream serialization: see common.cuh
  pdl_launch();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.x * 4 + warp;
  float l_pg = 0.f, l_bl = 0.f, l_ent = 0.f;
  if (b < B)
    tail_column_warp<true>(bl, tl + (size_t)b * A, (size_t)B * A, baseline + b, (size_t)B, action, reward, done, T, B, A, b, lane, discounting,
                           clip_reward, clip_rho, clip_pg, baseline_cost, entropy_cost, vs, pg, dlogits, dbaseline, nullptr, l_pg, l_bl,
                           l_ent);
  if (publish_block_partials(scratch, l_pg, l_bl, l_ent) && warp == 0) {   // fixed-order parallel sum of the block partials, also in column_step_kernel
    __threadfence();
    float s[3] = {0.f, 0.f, 0.f};
    for (unsigned k = lane; k < gridDim.x; k += 32)
      for (int i = 0; i < 3; ++i) s[i] += reinterpret_cast<volatile float*>(scratch)[4 + k * 3 + i];
    for (int i = 0; i < 3; ++i) s[i] = warp_sum(s[i]);
    if (lane == 0) write_losses(losses, scratch, s[0], s[1], s[2], baseline_cost, entropy_cost);
  }
}


// ------------------------------------------------------------------------------------------------
// Row-wise policy ops behind the differentiable drop-ins of loss_fn.py / vtrace.action_log_probs (host side:
// scalerl_b200/algorithms/impala/{loss_fn,vtrace}.py).  One thread per row of A logits.
//   forward : logp[n] = log_softmax(logits[n])[action[n]]   (vtrace.py:31-40; loss_fn.py:16-23 uses its negation)
//             ent[n]  = sum_a p log p                       (loss_fn.py:9-13)
//   backward: dlogits[n][a] = w_logp[n] * (onehot(a == action[n]) - p[a]) + w_ent[n] * p[a] * (log p[a] - ent[n])
//             (the autograd of  sum_n w_logp[n] * logp[n] + w_ent[n] * ent[n];  NULL weight array = zeros)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) policy_rows_fwd_kernel(const float* __restrict__ logits, const int64_t* __restrict__ actions, int64_t N,
                                                              int A, float* __restrict__ logp, float* __restrict__ ent) {
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const float* row = logits + n * A;
  const RowLse s = row_lse<true>(row, A);
  if (logp) logp[n] = row_logp<true>(row, s, ld_action(actions + n, A));
  if (ent) ent[n] = row_entropy<true>(row, s, A);
}
__global__ void __launch_bounds__(128) policy_rows_bwd_kernel(const float* __restrict__ logits, const int64_t* __restrict__ actions,
                                                              const float* __restrict__ w_logp, const float* __restrict__ w_ent, int64_t N,
                                                              int A, float* __restrict__ dlogits) {
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const float* row = logits + n * A;
  const RowLse s = row_lse<true>(row, A);
  const float wl = w_logp ? __ldg(w_logp + n) : 0.f, we = w_ent ? __ldg(w_ent + n) : 0.f;
  const float e = w_ent ? row_entropy<true>(row, s, A) : 0.f;
  const int act = actions ? ld_action(actions + n, A) : -1;
  for (int a = 0; a < A; ++a) {
    const float lp = row_logp<true>(row, s, a), p = expf(lp);
    dlogits[n * A + a] = wl * ((a == act ? 1.f : 0.f) - p) + we * p * (lp - e);
  }
}
// out[0] = scale * sum_i x[i]  or  scale * sum_i x[i]^2 (square != 0); ONE block, fixed order: deterministic
__global__ void __launch_bounds__(1024) reduce_sum_kernel(const float* __restrict__ x, int64_t n, int square, float scale, float* __restrict__ out) {
  __shared__ float part[32];
  float s = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += 1024) { const float v = __ldg(x + i); s += square ? v * v : v; }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = part[threadIdx.x];
    t = warp_sum(t);
    if (threadIdx.x == 0) out[0] = scale * t;
  }
}
// action[n] ~ softmax(logits[n]) by inverse CDF of the uniform u[n] in [0,1)  (AtariNet.forward's torch.multinomial in training mode,
// atari_model.py:130-132);  u == NULL: argmax (evaluation mode, :133-134).  One thread per row.
__global__ void __launch_bounds__(128) sample_actions_kernel(const float* __restrict__ logits, const float* __restrict__ u, int64_t N, int A,
                                                             int64_t* __restrict__ actions) {
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const float* row = logits + n * A;
  float mx = -INFINITY;
  int arg = 0;
  for (int a = 0; a < A; ++a) { const float v = __ldg(row + a); if (v > mx) { mx = v; arg = a; } }
  if (!u) { actions[n] = arg; return; }
  float se = 0.f;
  for (int a = 0; a < A; ++a) se += expf(__ldg(row + a) - mx);
  const float target = __ldg(u + n) * se;
  float c = 0.f;
  int pick = A - 1;
  for (int a = 0; a < A; ++a) {
    c += expf(__ldg(row + a) - mx);
    if (target < c) { pick = a; break; }
  }
  actions[n] = pick;
}
cudaError_t launch_sample_actions(const float* logits, const float* u, int64_t N, int A, int64_t* actions, cudaStream_t st) {
  if (N <= 0) return cudaSuccess;
  sample_actions_kernel<<<(unsigned)((N + 127) / 128), 128, 0, st>>>(logits, u, N, A, actions);
  return cudaGetLastError();
}
cudaError_t launch_policy_rows_fwd(const float* logits, const int64_t* actions, int64_t N, int A, float* logp, float* ent, cudaStream_t st) {
  if (N <= 0) return cudaSuccess;
  policy_rows_fwd_kernel<<<(unsigned)((N + 127) / 128), 128, 0, st>>>(logits, actions, N, A, logp, ent);
  return cudaGetLastError();
}
cudaError_t launch_policy_rows_bwd(const float* logits, const int64_t* actions, const float* w_logp, const float* w_ent, int64_t N, int A,
                                   float* dlogits, cudaStream_t st) {
  if (N <= 0) return cudaSuccess;
  policy_rows_bwd_kernel<<<(unsigned)((N + 127) / 128), 128, 0, st>>>(logits, actions, w_logp, w_ent, N, A, dlogits);
  return cudaGetLastError();
}
cudaError_t launch_reduce_sum(const float* x, int64_t n, int square, float scale, float* out, cudaStream_t st) {
  reduce_sum_kernel<<<1, 1024, 0, st>>>(x, n, square, scale, out);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
cudaError_t launch_vtrace_iw(const float* log_rhos, const float* discounts, const float* rewards, const float* values,
                             const float* bootstrap, int T, int B, float clip_rho, float clip_pg, float* vs, float* pg, int variant,
                             cudaStream_t st) {
  if (T <= 0 || B <= 0) return cudaSuccess;
  if (variant == 1 && T <= SCAN_MAX_T) {
    const size_t smem = (size_t)4 * T * 33 * sizeof(float);
    cudaError_t e = cudaFuncSetAttribute(vtrace_iw_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    vtrace_iw_scan_kernel<<<(B + 31) / 32, 256, smem, st>>>(log_rhos, discounts, rewards, values, bootstrap, T, B, clip_rho, clip_pg, vs, pg);
    return cudaGetLastError();
  }
  const bool al = ((reinterpret_cast<uintptr_t>(log_rhos) | reinterpret_cast<uintptr_t>(discounts) | reinterpret_cast<uintptr_t>(rewards) |
                    reinterpret_cast<uintptr_t>(values) | reinterpret_cast<uintptr_t>(bootstrap) | reinterpret_cast<uintptr_t>(vs) |
                    reinterpret_cast<uintptr_t>(pg)) & 15) == 0;
  if (B % 4 == 0 && al && B >= 4 * 128 * 132) {   // enough columns to fill the chip with 4-wide threads
    const int threads = B / 4;
    vtrace_iw_seq_kernel<4><<<(threads + 127) / 128, 128, 0, st>>>(log_rhos, discounts, rewards, values, bootstrap, T, B, clip_rho, clip_pg, vs, pg);
  } else {
    vtrace_iw_seq_kernel<1><<<(B + 127) / 128, 128, 0, st>>>(log_rhos, discounts, rewards, values, bootstrap, T, B, clip_rho, clip_pg, vs, pg);
  }
  return cudaGetLastError();
}

cudaError_t launch_vtrace_logits(const float* bl, const float* tl, const int64_t* actions, const float* discounts, const float* rewards,
                                 const float* values, const float* bootstrap, int T, int B, int A, float clip_rho, float clip_pg,
                                 float* vs, float* pg, float* lr, float* balp, float* talp, cudaStream_t st) {
  if (T <= 0 || B <= 0) return cudaSuccess;
  vtrace_logits_kernel<<<(B + 127) / 128, 128, 0, st>>>(bl, tl, actions, discounts, rewards, values, bootstrap, T, B, A, clip_rho, clip_pg,
                                                         vs, pg, lr, balp, talp);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// Fused column kernel (learner step only): one block per batch column b does, for its T+1 frames,
//   A. the fc epilogue (split-K partial sums + bias + ReLU -> h) and the policy / baseline heads (atari_model.py:100-113),
//   B. V-trace + the three losses + d(logits), d(baseline) for the column (vtrace.py:78-172, impala_atari.py:293-330),
//   C. dh = (dlogits . Wp + dbaseline Wb) * (h > 0) -> bf16, the operand of the fc backward GEMMs,
// with h, the logits and the head gradients kept in shared memory between the phases: three dependent launches of
// latency-bound kernels become one.  Needs (T+1) * 2 KB of shared memory: used when that fits, B <= 512, A <= 32.
// AMAX (8 or 32) bounds the unrolled per-action loops: their predicated-off iterations still cost issue slots.
// ------------------------------------------------------------------------------------------------
constexpr int COL_THREADS = 1024, COL_MAX_A = 31;      // lane a == A computes the baseline: A + 1 <= 32 lanes
//      // 32 warps: every frame of a T <= 31 column in one pass of phase A
template <int NSPLIT, int AMAX>
__global__ void __launch_bounds__(COL_THREADS) column_step_kernel(
    const float* __restrict__ hpart, const float* __restrict__ bfc, float* __restrict__ h, const float* __restrict__ reward,
    const int64_t* __restrict__ action, const uint8_t* __restrict__ done, const float* __restrict__ bl, const float* __restrict__ Wp,
    const float* __restrict__ bp, const float* __restrict__ Wb, const float* __restrict__ bb, int T, int B, int A, float discounting,
    int clip_reward, float clip_rho, float clip_pg, float baseline_cost, float entropy_cost, float* __restrict__ logits,
    float* __restrict__ baseline, float* __restrict__ vs, float* __restrict__ pg, float* __restrict__ dlogits,
    float* __restrict__ dbaseline, __nv_bfloat16* __restrict__ dh, float* __restrict__ losses, float* __restrict__ scratch,
    __nv_bfloat16* __restrict__ dh_lo) {
  extern __shared__ __align__(16) float csm[];
  const int CORE = 513 + A, WS = (CORE + 3) & ~3, N = (T + 1) * B;
  float* s_w = csm;                                   // [A+1][WS]: policy rows, then the baseline row
  float* s_h = s_w + (size_t)(A + 1) * WS;            // [T+1][512]
  float* s_log = s_h + (size_t)(T + 1) * 512;         // [T+1][A]
  float* s_base = s_log + (size_t)(T + 1) * A;        // [T+1]
  float* s_dl = s_base + (T + 1);                     // [T][A+1]: dlogits..., dbaseline
  __shared__ bool is_last;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, b = blockIdx.x;
  // the head weights were final before the step started: loaded before griddepcontrol.wait (overlaps the fc GEMM's tail)
  for (int j = tid; j < CORE; j += COL_THREADS) {       // a thread copies column j of every row: A + 1 independent loads in flight
    float wv[AMAX + 1];
#pragma unroll
    for (int a = 0; a <= AMAX; ++a)
      if (a <= A) wv[a] = a < A ? __ldg(Wp + (size_t)a * CORE + j) : __ldg(Wb + j);
#pragma unroll
    for (int a = 0; a <= AMAX; ++a)
      if (a <= A) s_w[a * WS + j] = wv[a];
  }
  pdl_wait(41);
  pdl_launch();
  __syncthreads();
  // ---- A: frames t = warp, warp + 32, ...; a lane owns features j = 128 i + 4 lane .. +3 (i < 4)
  for (int t = warp; t <= T; t += COL_THREADS / 32) {
    const size_t n = (size_t)t * B + b;
    // operands of the last stage of this frame (lanes 0..A), requested now so their latency hides under the partial sums
    float pre_r = 0.f, pre_bias = 0.f;
    int pre_act = 0;
    if (lane <= A) {
      pre_r = __ldg(reward + n);
      pre_act = ld_action(action + n, A);
      pre_bias = lane < A ? __ldg(bp + lane) : __ldg(bb);
    }
    float4 x[4];
    float dot[AMAX + 1];
#pragma unroll
    for (int a = 0; a <= AMAX; ++a) dot[a] = 0.f;
    {
      float4 part[4][NSPLIT];                  // all 4 * NSPLIT loads in flight together; summed in split order (deterministic)
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int k = 0; k < NSPLIT; ++k)
          part[i][k] = __ldg(reinterpret_cast<const float4*>(hpart + ((size_t)k * N + n) * 512 + 128 * i + 4 * lane));
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int j = 128 * i + 4 * lane;
        float4 v = part[i][0];
#pragma unroll
        for (int k = 1; k < NSPLIT; ++k) { v.x += part[i][k].x; v.y += part[i][k].y; v.z += part[i][k].z; v.w += part[i][k].w; }
        const float4 b4 = __ldg(reinterpret_cast<const float4*>(bfc + j));
        v.x = fmaxf(v.x + b4.x, 0.f); v.y = fmaxf(v.y + b4.y, 0.f); v.z = fmaxf(v.z + b4.z, 0.f); v.w = fmaxf(v.w + b4.w, 0.f);
        *reinterpret_cast<float4*>(h + n * 512 + j) = v;
        *reinterpret_cast<float4*>(s_h + (size_t)t * 512 + j) = v;
        x[i] = v;
      }
    }
#pragma unroll
    for (int a = 0; a <= AMAX; ++a) {
      if (a <= A) {
        float sacc = 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float4 w = *reinterpret_cast<const float4*>(s_w + (size_t)a * WS + 128 * i + 4 * lane);
          sacc += x[i].x * w.x + x[i].y * w.y + x[i].z * w.z + x[i].w * w.w;
        }
        dot[a] = warp_sum(sacc);
      }
    }
    if (lane <= A) {
      const int a = lane;
      const float r = fminf(fmaxf(pre_r, -1.f), 1.f);
      const int act = pre_act;
      float sv = 0.f;
#pragma unroll
      for (int q = 0; q <= AMAX; ++q) if (q == a) sv = dot[q];          // warp_sum left the total in every lane
      sv += s_w[(size_t)a * WS + 512] * r + s_w[(size_t)a * WS + 513 + act] + pre_bias;
      if (a < A) { logits[n * A + a] = sv; s_log[(size_t)t * A + a] = sv; }
      else       { baseline[n] = sv; s_base[t] = sv; }
    }
  }
  __syncthreads();
  // ---- B: V-trace, losses and head gradients of this column (one warp)
  if (warp == 0) {
    float l_pg = 0.f, l_bl = 0.f, l_ent = 0.f;
    tail_column_warp<false>(bl, s_log, (size_t)A, s_base, (size_t)1, action, reward, done, T, B, A, b, lane, discounting, clip_reward,
                            clip_rho, clip_pg, baseline_cost, entropy_cost, vs, pg, dlogits, dbaseline, s_dl, l_pg, l_bl, l_ent);
    l_pg = warp_sum(l_pg); l_bl = warp_sum(l_bl); l_ent = warp_sum(l_ent);
    if (lane == 0) {
      scratch[4 + b * 3 + 0] = l_pg; scratch[4 + b * 3 + 1] = l_bl; scratch[4 + b * 3 + 2] = l_ent;
      is_last = take_ticket(scratch);
    }
  }
  __syncthreads();
  // fixed-order sum of the column partials, as in impala_tail_warp_kernel: through one helper this kernel compiles differently
  if (is_last && warp == 0) {
    __threadfence();
    float s3[3] = {0.f, 0.f, 0.f};
    for (unsigned k = lane; k < gridDim.x; k += 32)
      for (int i = 0; i < 3; ++i) s3[i] += reinterpret_cast<volatile float*>(scratch)[4 + k * 3 + i];
    for (int i = 0; i < 3; ++i) s3[i] = warp_sum(s3[i]);
    if (lane == 0) write_losses(losses, scratch, s3[0], s3[1], s3[2], baseline_cost, entropy_cost);
  }
  // ---- C: dh[n][j] for the T learning frames of the column; thread = (feature j, parity of t)
  {
    const int j = tid & 511;
    float w[AMAX + 1];
#pragma unroll
    for (int a = 0; a <= AMAX; ++a) w[a] = a <= A ? s_w[(size_t)a * WS + j] : 0.f;
    for (int t = tid >> 9; t < T; t += COL_THREADS / 512) {
      const float* d = s_dl + (size_t)t * (A + 1);
      float acc = 0.f;
#pragma unroll
      for (int a = 0; a <= AMAX; ++a) if (a <= A) acc = fmaf(d[a], w[a], acc);
      const float hv = s_h[(size_t)t * 512 + j];
      const float dv = hv > 0.f ? acc : 0.f;
      const __nv_bfloat16 hi = __float2bfloat16_rn(dv);
      dh[((size_t)t * B + b) * 512 + j] = hi;
      if (dh_lo) dh_lo[((size_t)t * B + b) * 512 + j] = __float2bfloat16_rn(dv - __bfloat162float(hi));   // fp32-accurate operand mode
    }
  }
}

static size_t column_smem_bytes(int T, int A) {
  const int CORE = 513 + A, WS = (CORE + 3) & ~3;
  return sizeof(float) * ((size_t)(A + 1) * WS + (size_t)(T + 1) * 512 + (size_t)(T + 1) * A + (T + 1) + (size_t)T * (A + 1));
}
SRL_KSTAMP_SETTER(kstamp_set_vtrace)

bool column_step_supported(int T, int B, int A) {
  return T >= 1 && B >= 1 && B <= 512 && A >= 1 && A <= COL_MAX_A && column_smem_bytes(T, A) <= 200 * 1024;
}
cudaError_t launch_column_step(const TailStep& s, const float* hpart, int nsplit, const float* bfc, float* h, const float* Wp, const float* bp,
                               const float* Wb, const float* bb, float* logits, float* baseline, __nv_bfloat16* dh, __nv_bfloat16* dh_lo,
                               cudaStream_t st) {
  if (!column_step_supported(s.T, s.B, s.A) || nsplit != 4) return cudaErrorInvalidValue;
  static PerDeviceOnce once[2];
  const bool narrow = s.A <= 8;
  const auto kernel = narrow ? column_step_kernel<4, 8> : column_step_kernel<4, 32>;
  const cudaError_t e = ensure_max_dynamic_smem(once[narrow ? 0 : 1], kernel, 200 * 1024);
  if (e != cudaSuccess) return e;
  return launch_chain(kernel, dim3(s.B), dim3(COL_THREADS), column_smem_bytes(s.T, s.A), st, hpart, bfc, h, s.reward, s.action, s.done, s.bl,
                      Wp, bp, Wb, bb, s.T, s.B, s.A, s.discounting, s.clip_reward, s.clip_rho, s.clip_pg, s.baseline_cost, s.entropy_cost, logits,
                      baseline, s.vs, s.pg, s.dlogits, s.dbaseline, dh, s.losses, s.scratch, dh_lo);
}

cudaError_t launch_impala_tail(const TailStep& s, const float* tl, const float* baseline, cudaStream_t st) {
  // latency-bound sizes: one warp per column, shuffle scan over T (block partials: 3*ceil(B/4) <= 1536 floats)
  const bool warp = s.B <= 2048;
  return launch_chain(warp ? impala_tail_warp_kernel : impala_tail_kernel, dim3(warp ? (s.B + 3) / 4 : (s.B + 127) / 128), dim3(128), 0, st,
                      s.bl, tl, baseline, s.action, s.reward, s.done, s.T, s.B, s.A, s.discounting, s.clip_reward, s.clip_rho, s.clip_pg,
                      s.baseline_cost, s.entropy_cost, s.vs, s.pg, s.dlogits, s.dbaseline, s.losses, s.scratch);
}

}  // namespace srl
