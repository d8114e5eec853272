// extern "C" entry points (include/scalerl_b200.h).  Argument checking + the learner context that owns
// the activation workspaces and sequences the kernels of one learner step on the caller's stream.
#include <string.h>
#include <cmath>
#include <new>

#include "../../include/scalerl_b200.h"
#include "errors.h"
#include "kernels.h"

using namespace srl;

extern "C" const char* srl_last_error(void) { return error_message(); }
extern "C" int srl_version(void) { return 100; }

// ------------------------------------------------------------------------------------------------
// stand-alone ops
// ------------------------------------------------------------------------------------------------
extern "C" int srl_vtrace_from_importance_weights(const float* log_rhos, const float* discounts, const float* rewards,
                                                  const float* values, const float* bootstrap_value, int T, int B,
                                                  float clip_rho, float clip_pg, float* vs, float* pg, int variant, void* stream) {
  REQ(T >= 0 && B >= 0, "vtrace: negative shape T=%d B=%d", T, B);
  REQ(!std::isnan(clip_rho) && !std::isnan(clip_pg), "vtrace: a clip threshold is NaN (< 0 means None)");
  if (T == 0 || B == 0) return 0;
  REQ(log_rhos && discounts && rewards && values && bootstrap_value && vs && pg, "vtrace: NULL pointer");
  CU(launch_vtrace_iw(log_rhos, discounts, rewards, values, bootstrap_value, T, B, clip_rho, clip_pg, vs, pg, variant,
                      (cudaStream_t)stream), "vtrace_from_importance_weights");
  return 0;
}

extern "C" int srl_vtrace_from_logits(const float* bl, const float* tl, const int64_t* actions, const float* discounts,
                                      const float* rewards, const float* values, const float* bootstrap_value, int T, int B, int A,
                                      float clip_rho, float clip_pg, float* vs, float* pg, float* log_rhos, float* balp, float* talp,
                                      void* stream) {
  REQ(T >= 0 && B >= 0 && A >= 1, "vtrace_from_logits: bad shape T=%d B=%d A=%d", T, B, A);
  REQ(!std::isnan(clip_rho) && !std::isnan(clip_pg), "vtrace_from_logits: a clip threshold is NaN (< 0 means None)");
  if (T == 0 || B == 0) return 0;
  REQ(bl && tl && actions && discounts && rewards && values && bootstrap_value && vs && pg, "vtrace_from_logits: NULL pointer");
  CU(launch_vtrace_logits(bl, tl, actions, discounts, rewards, values, bootstrap_value, T, B, A, clip_rho, clip_pg, vs, pg, log_rhos,
                          balp, talp, (cudaStream_t)stream), "vtrace_from_logits");
  return 0;
}

// a tail's shape and loss settings from c (fields assigned by name: several neighbours share a type)
static TailStep tail_step(const srl_config_t& c, const float* bl, const int64_t* action, const float* reward, const uint8_t* done, float* vs,
                          float* pg, float* dlogits, float* dbaseline, float* losses, float* scratch) {
  TailStep s;
  s.bl = bl; s.action = action; s.reward = reward; s.done = done; s.T = c.T; s.B = c.B; s.A = c.A;
  s.discounting = c.discounting; s.clip_reward = c.reward_clip_abs_one; s.clip_rho = c.clip_rho_threshold; s.clip_pg = c.clip_pg_rho_threshold;
  s.baseline_cost = c.baseline_cost; s.entropy_cost = c.entropy_cost;
  s.vs = vs; s.pg = pg; s.dlogits = dlogits; s.dbaseline = dbaseline; s.losses = losses; s.scratch = scratch;
  return s;
}

extern "C" int srl_impala_loss_and_head_grads(const float* bl, const float* tl, const float* baseline, const int64_t* action,
                                              const float* reward, const uint8_t* done, int T, int B, int A, float discounting,
                                              int reward_clip_abs_one, float clip_rho, float clip_pg, float baseline_cost,
                                              float entropy_cost, float* vs, float* pg, float* dlogits, float* dbaseline, float* losses,
                                              float* scratch, void* stream) {
  REQ(T >= 1 && B >= 1 && A >= 1, "impala_loss: bad shape T=%d B=%d A=%d", T, B, A);
  REQ(!std::isnan(clip_rho) && !std::isnan(clip_pg), "impala_loss: a clip threshold is NaN (< 0 means None)");
  REQ(bl && tl && baseline && action && reward && done && dlogits && dbaseline && losses && scratch, "impala_loss: NULL pointer");
  srl_config_t c = {};
  c.T = T; c.B = B; c.A = A; c.discounting = discounting; c.reward_clip_abs_one = reward_clip_abs_one;
  c.clip_rho_threshold = clip_rho; c.clip_pg_rho_threshold = clip_pg; c.baseline_cost = baseline_cost; c.entropy_cost = entropy_cost;
  pdl_set_active(true);      // no learner call: SRL_PDL alone decides
  CU(launch_impala_tail(tail_step(c, bl, action, reward, done, vs, pg, dlogits, dbaseline, losses, scratch), tl, baseline, (cudaStream_t)stream),
     "impala_tail");
  return 0;
}

extern "C" int srl_policy_rows_forward(const float* logits, const int64_t* actions, int64_t N, int A, float* logp, float* ent, void* stream) {
  REQ(N >= 0 && A >= 1, "policy_rows_forward: bad shape N=%lld A=%d", (long long)N, A);
  if (N == 0) return 0;
  REQ(logits && (logp || ent) && (!logp || actions), "policy_rows_forward: NULL pointer");
  CU(launch_policy_rows_fwd(logits, actions, N, A, logp, ent, (cudaStream_t)stream), "policy_rows_forward");
  return 0;
}
extern "C" int srl_policy_rows_backward(const float* logits, const int64_t* actions, const float* w_logp, const float* w_ent, int64_t N, int A,
                                        float* dlogits, void* stream) {
  REQ(N >= 0 && A >= 1, "policy_rows_backward: bad shape N=%lld A=%d", (long long)N, A);
  if (N == 0) return 0;
  REQ(logits && dlogits && (!w_logp || actions), "policy_rows_backward: NULL pointer");
  CU(launch_policy_rows_bwd(logits, actions, w_logp, w_ent, N, A, dlogits, (cudaStream_t)stream), "policy_rows_backward");
  return 0;
}
extern "C" int srl_sample_actions(const float* logits, const float* uniforms, int64_t N, int A, int64_t* actions, void* stream) {
  REQ(N >= 0 && A >= 1, "sample_actions: bad shape N=%lld A=%d", (long long)N, A);
  if (N == 0) return 0;
  REQ(logits && actions, "sample_actions: NULL pointer");
  CU(launch_sample_actions(logits, uniforms, N, A, actions, (cudaStream_t)stream), "sample_actions");
  return 0;
}
extern "C" int srl_reduce_sum(const float* x, int64_t n, int square, float scale, float* out, void* stream) {
  REQ(n >= 0 && out && (x || n == 0), "reduce_sum: bad argument");
  CU(launch_reduce_sum(x, n, square, scale, out, (cudaStream_t)stream), "reduce_sum");
  return 0;
}

extern "C" int srl_unpack_slots(const uint8_t* staging, int64_t slot_bytes, const int64_t* offsets6_host, int T, int B, int A, uint8_t* obs,
                                float* reward, uint8_t* done, int64_t* action, float* policy_logits, float* episode_return, void* stream) {
  REQ(staging && offsets6_host && obs && reward && done && action && policy_logits, "unpack_slots: NULL pointer");
  REQ(T >= 1 && B >= 1 && A >= 1 && A <= 32 && slot_bytes > 0, "unpack_slots: bad shape");
  REQ((slot_bytes & 15) == 0 && (offsets6_host[0] & 15) == 0 && !misaligned(staging, 16) && !misaligned(obs, 16),
      "unpack_slots: obs record and buffers must be 16-byte aligned");
  CU(launch_unpack_slots(staging, slot_bytes, offsets6_host, T, B, A, obs, reward, done, action, policy_logits, episode_return,
                         (cudaStream_t)stream), "unpack_slots");
  return 0;
}

extern "C" int srl_grad_norm_clip_coef(const float* grads, int64_t n, float max_norm, float* coef, float* scratch, void* stream) {
  REQ(grads && coef && scratch && n >= 0, "grad_norm: bad argument");
  REQ(!misaligned(grads, 16), "grad_norm: grads must be 16-byte aligned");
  CU(launch_grad_norm(grads, n, max_norm, coef, scratch, (cudaStream_t)stream), "grad_norm");
  return 0;
}
extern "C" int srl_rmsprop_step(float* params, const float* grads, float* square_avg, int64_t n, const float* coef, float lr, float alpha,
                                float eps, void* stream) {
  REQ(params && grads && square_avg && n >= 0, "rmsprop: bad argument");
  REQ(!misaligned(params, 16) && !misaligned(grads, 16) && !misaligned(square_avg, 16), "rmsprop: buffers must be 16-byte aligned");
  CU(launch_rmsprop(params, grads, square_avg, n, coef, lr, alpha, eps, (cudaStream_t)stream), "rmsprop");
  return 0;
}
extern "C" int srl_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n, const float* coef, float lr,
                             float beta1, float beta2, float eps, int step, void* stream) {
  REQ(params && grads && exp_avg && exp_avg_sq && n >= 0 && step >= 1, "adam: bad argument");
  CU(launch_adam(params, grads, exp_avg, exp_avg_sq, n, coef, lr, beta1, beta2, eps, step, (cudaStream_t)stream), "adam");
  return 0;
}

// ------------------------------------------------------------------------------------------------
// parameter layout
// ------------------------------------------------------------------------------------------------
// Flat buffer order: every small tensor first (conv1..3, fc.bias, heads), fc.weight LAST.  The small block is one
// contiguous range (one memset, one late all-reduce); fc.weight (95 % of the bytes) is final early in the backward pass
// and can be all-reduced while the conv layers are still back-propagating.  off/cnt are indexed in state_dict order.
static int64_t layout_ex(int A, int use_lstm, int64_t* off, int64_t* cnt) {
  const int64_t core = 513 + A;
  const int64_t counts[20] = {32 * 256, 32, 64 * 512, 64, 64 * 576, 64, 512 * 3136, 512, A * core, A, core, 1,
                              4 * core * core, 4 * core * core, 4 * core, 4 * core, 4 * core * core, 4 * core * core, 4 * core, 4 * core};
  const int order[20] = {0, 1, 2, 3, 4, 5, 7, 8, 9, 10, 11, 6, 12, 13, 14, 15, 16, 17, 18, 19};
  int64_t o = 0;
  const int n = use_lstm ? 20 : 12;
  for (int k = 0; k < 20; ++k) {
    const int i = order[k];
    if (k >= n) { if (off) off[i] = o; if (cnt) cnt[i] = 0; continue; }
    if (off) off[i] = o;
    if (cnt) cnt[i] = counts[i];
    o += (counts[i] + 3) & ~int64_t(3);
  }
  return o;
}
static int64_t layout(int A, int64_t* off, int64_t* cnt) {
  int64_t o20[20], c20[20];
  const int64_t total = layout_ex(A, 0, o20, c20);
  for (int i = 0; i < 12; ++i) { if (off) off[i] = o20[i]; if (cnt) cnt[i] = c20[i]; }
  return total;
}
extern "C" int64_t srl_param_layout(int A, int64_t* offsets, int64_t* counts) { return layout(A, offsets, counts); }
extern "C" int64_t srl_param_layout_ex(int A, int use_lstm, int64_t* offsets20, int64_t* counts20) { return layout_ex(A, use_lstm, offsets20, counts20); }

static ParamPtrs make_ptrs(float* base, int A) {
  int64_t off[12];
  layout(A, off, nullptr);
  ParamPtrs p;
  p.w1 = base + off[0]; p.b1 = base + off[1]; p.w2 = base + off[2]; p.b2 = base + off[3]; p.w3 = base + off[4]; p.b3 = base + off[5];
  p.wf = base + off[6]; p.bf = base + off[7]; p.wp = base + off[8]; p.bp = base + off[9]; p.wb = base + off[10]; p.bb = base + off[11];
  return p;
}

// ------------------------------------------------------------------------------------------------
// learner context
// ------------------------------------------------------------------------------------------------
struct srl_learner {
  srl_config_t cfg;
  float *params, *grads, *opt0, *opt1;
  int64_t nparams;
  ParamPtrs P, G;
  EncoderBuffers buf;
  float *logits, *baseline;       // [NF][A], [NF]
  float *dlogits, *dbaseline;     // [NB][A], [NB]
  float *scratch;                 // reductions (tail + grad norm)
  float* head_part;               // [HEAD_GROUPS][A+1][514+A] partial head weight gradients
  float *coef;                    // {norm, clip coef, lr of the step}
  char* arena;                    // every workspace tensor (workspace_table)
  int64_t arena_bytes;
  int64_t small_len;              // floats before fc.weight in the flat buffer: the small gradients cleared at the start of a step
  int step;                       // optimizer step count (Adam bias correction)
  bool have_fwd;
  TmaMaps maps;                   // tensor maps of the TMA mainloop
  StepStreams S;                  // the lanes beside the caller's stream, and the per-kernel profiler
  int* dstep;                     // device-side optimizer step count (graph-replay safe Adam bias correction and lr schedule)
  OptExtra ox;                    // lr schedule + RMSprop momentum of the optimizer step (srl_learner_set_lr_schedule / _set_momentum)
  bool report_lr;                 // grad_norm_out receives coef[2] too (after srl_learner_set_lr_schedule)
  srl_lstm_t* lstm;               // use_lstm: the 2-layer LSTM core (csrc/lstm.cu) working on views of params/grads
  float *core, *lstm_out, *dout, *dcore;   // [NF][H], [NF][H], [NB][H], [NB][H]
  int64_t lstm_off0, lstm_len;    // LSTM gradient range inside the flat buffer
  LstmStep* lstm_step;            // use_lstm: the one-row actor step (packed weights + operands; csrc/lstm.cu)
  int lstm_step_ksplit;           // K split of its GEMM (cluster size; srl_learner_set_option "lstm_step_ksplit")
  bool fused_front;               // frame conversion + conv1 + conv2 as one kernel (SRL_FUSED_FWD / srl_learner_set_option "fused_fwd")
  bool column_fusion;             // heads + V-trace/loss + dh in one column kernel (SRL_NO_COLUMN_FUSION / srl_learner_set_option)
};

static const char* kSlotNames[PS_COUNT] = {"obs_s2d", "conv1_fwd", "conv2_fwd", "conv3_fwd", "fc_fwd", "head_fwd", "vtrace_loss_tail",
                                           "zero_grads", "head_bwd", "fc_wgrad", "fc_dgrad", "conv3_wgrad", "conv3_dgrad", "conv2_wgrad",
                                           "conv2_dgrad", "conv1_wgrad", "conv_wgrad_finalize", "grad_norm", "optimizer", "pack_weights", "enc_fused_fwd"};

static int check_cfg(const srl_config_t* c) {
  REQ(c, "config is NULL");
  REQ(c->T >= 1 && c->B >= 1, "config: T=%d B=%d must be >= 1", c->T, c->B);
  REQ(c->A >= 1 && c->A <= 31, "config: A=%d must be in [1,31] (one warp lane per action plus one for the baseline)", c->A);
  REQ((int64_t)(c->T + 1) * c->B <= MAX_FRAMES, "config: (T+1)*B=%lld frames per GPU exceeds %d", (long long)(c->T + 1) * c->B, MAX_FRAMES);
  REQ(c->optimizer == 0 || c->optimizer == 1, "config: optimizer must be 0 (rmsprop) or 1 (adam)");
  REQ(c->use_lstm == 0 || c->use_lstm == 1, "config: use_lstm must be 0 or 1");
  REQ(c->precision == 0 || c->precision == 1, "config: precision must be 0 (bf16 operands) or 1 (fp32-accurate split operands)");
  REQ(!(c->precision == 1 && c->use_lstm), "config: the fp32-accurate operand mode covers the non-LSTM learner only");
  REQ(!std::isnan(c->clip_rho_threshold) && !std::isnan(c->clip_pg_rho_threshold), "config: a clip threshold is NaN (< 0 means None)");
  return 0;
}

// The device workspace of a learner context, one row per tensor in carving order (WsRow, kernels.h).  The arena is zero-filled at
// creation (the zeros of the da*g grids are the padding of the transposed convolutions).  In the fp32-accurate operand mode a row
// with a low twin is followed by the twin, which srl_learner_debug_buffer calls "<name>_lo".  Rows without a name are internal.
constexpr int WS_MAX_ROWS = 32;
// (the encoder's rows: encoder_rows, kernels.h)
static int workspace_table(srl_learner* L, WsRow* t) {
  const srl_config_t& c = L->cfg;
  const int64_t NF = (int64_t)(c.T + 1) * c.B, NB = (int64_t)c.T * c.B, A = c.A, H = 513 + A;
  int n = encoder_rows(L->buf, NF, NB, t);
  t[n++] = ws_row("logits", NF * A, &L->logits);
  t[n++] = ws_row("baseline", NF, &L->baseline);
  t[n++] = ws_row("dlogits", NB * A, &L->dlogits);
  t[n++] = ws_row("dbaseline", NB, &L->dbaseline);
  t[n++] = ws_row(nullptr, 4096, &L->scratch);
  t[n++] = ws_row(nullptr, 4, &L->coef);
  t[n++] = ws_row(nullptr, 4, &L->dstep);
  t[n++] = ws_row(nullptr, HEAD_GROUPS * (A + 1) * (514 + A), &L->head_part);
  if (c.use_lstm) {
    t[n++] = ws_row(nullptr, NF * H, &L->core);
    t[n++] = ws_row(nullptr, NF * H, &L->lstm_out);
    t[n++] = ws_row(nullptr, NB * H, &L->dout);
    t[n++] = ws_row(nullptr, NB * H, &L->dcore);
    t[n++] = ws_row<char>(nullptr, 1024, nullptr);      // 1 KiB of zeros behind dcore
  }
  return n;
}

// the re-pack lane sits one level BELOW the greatest priority (which the learner's capture stream uses for the main chain) and above the wgrad
// lanes (default = least): its short blocks fill the slots the frame conversion leaves free without delaying it
static int pack_priority(int least, int greatest) {
  return greatest + 1 > least ? least : greatest + 1;
}
// the lanes of a context: without them every call runs collapsed on the caller's stream
static void create_lanes(StepStreams& S) {
  int lo = 0, hi = 0;       // (numerically lowest = greatest priority)
  bool ok = cudaDeviceGetStreamPriorityRange(&lo, &hi) == cudaSuccess;
  for (int l = 0; l < LANE_COUNT && ok; ++l)        // the wgrad lanes take the default priority (0, the least)
    ok = cudaStreamCreateWithPriority(&S.side[l], cudaStreamNonBlocking, l == LANE_PACK ? pack_priority(lo, hi) : 0) == cudaSuccess &&
         cudaEventCreateWithFlags(&S.forked[l], cudaEventDisableTiming) == cudaSuccess &&
         cudaEventCreateWithFlags(&S.joined[l], cudaEventDisableTiming) == cudaSuccess;
  S.have_lanes = ok;
  cudaGetLastError();
}
static void destroy_lanes(StepStreams& S) {
  for (int l = 0; l < LANE_COUNT; ++l) {
    if (S.forked[l]) cudaEventDestroy(S.forked[l]);
    if (S.joined[l]) cudaEventDestroy(S.joined[l]);
    if (S.side[l]) cudaStreamDestroy(S.side[l]);
  }
}

extern "C" int srl_learner_create(const srl_config_t* cfg, float* params, float* grads, float* opt0, float* opt1, srl_learner_t** out) {
  int rc = check_cfg(cfg);
  if (rc) return rc;
  REQ(params && grads && opt0 && out, "learner_create: NULL buffer");
  REQ(cfg->optimizer == 0 || opt1, "learner_create: Adam needs opt_state1");
  REQ(!misaligned(params, 16) && !misaligned(grads, 16) && !misaligned(opt0, 16) && !misaligned(opt1, 16),
      "learner_create: flat buffers must be 16-byte aligned");
  srl_learner* L = new (std::nothrow) srl_learner();      // value-initialised: srl_learner_destroy can release any partial context
  REQ(L, "out of host memory");
  auto undo = [L](int code) { srl_learner_destroy(L); return code; };      // the error message is written before the release
  L->cfg = *cfg; L->params = params; L->grads = grads; L->opt0 = opt0; L->opt1 = opt1;
  int64_t off[20];
  L->nparams = layout_ex(cfg->A, cfg->use_lstm, off, nullptr);
  L->small_len = off[6];
  L->lstm_step_ksplit = LSTM_STEP_KSPLIT;
  L->P = make_ptrs(params, cfg->A);
  L->G = make_ptrs(grads, cfg->A);
  { const char* nf = getenv("SRL_NO_COLUMN_FUSION"); L->column_fusion = !(nf && atoi(nf) != 0); }   // read once, at creation
  // opt-in: the fused front has not been measured on H100 against the three kernels it replaces
  { const char* ff = getenv("SRL_FUSED_FWD"); L->fused_front = ff && atoi(ff) != 0; }
  const int64_t NF = (int64_t)(cfg->T + 1) * cfg->B, NB = (int64_t)cfg->T * cfg->B;
  WsRow t[WS_MAX_ROWS];
  const int n = workspace_table(L, t);
  const bool split = cfg->precision == 1;
  const int64_t total = rows_bytes(t, n, split);
  cudaError_t e = cudaMalloc(&L->arena, total);
  if (e != cudaSuccess) return undo(cuda_fail(e, "learner_create: cudaMalloc workspace"));
  e = cudaMemset(L->arena, 0, total);
  if (e != cudaSuccess) return undo(cuda_fail(e, "learner_create: cudaMemset"));
  L->arena_bytes = total;
  carve_rows(t, n, split, L->arena);
  L->buf.NF = (int)NF;
  create_lanes(L->S);
  const char* why = nullptr;
  if (build_tma_maps(L->buf, (int)NF, (int)NB, &L->maps, &why) != cudaSuccess)
    return undo(fail(SRL_ESTATE, "learner_create: building TMA tensor map '%s' failed (driver without cuTensorMapEncodeTiled?)", why ? why : "?"));
  if (cfg->use_lstm) {
    const int H = 513 + cfg->A;
    const float* wp[8]; float* gp[8];
    for (int i = 0; i < 8; ++i) { wp[i] = params + off[12 + i]; gp[i] = grads + off[12 + i]; }
    L->lstm_off0 = off[12]; L->lstm_len = L->nparams - off[12];
    // the callee's message stays in place
    if (srl_lstm_create(cfg->T + 1, cfg->B, H, wp, gp, &L->lstm) != 0 || lstm_step_create(cfg->B, H, wp, &L->lstm_step) != 0) return undo(SRL_ESTATE);
  }
  *out = L;
  return 0;
}

extern "C" int srl_learner_destroy(srl_learner_t* L) {
  if (!L) return 0;
  for (int i = 0; i < 2 * PS_COUNT; ++i) if (L->S.slot_events[i]) cudaEventDestroy(L->S.slot_events[i]);
  destroy_lanes(L->S);
  if (L->lstm) srl_lstm_destroy(L->lstm);
  lstm_step_destroy(L->lstm_step);
  cudaFree(L->arena);
  delete L;
  return 0;
}
extern "C" int srl_debug_kernel_timeline(void* buffer) {
#ifdef SRL_KSTAMP
  kstamp_set_encoder((unsigned long long*)buffer); kstamp_set_vtrace((unsigned long long*)buffer); kstamp_set_heads((unsigned long long*)buffer);
  kstamp_set_optim((unsigned long long*)buffer);
  cudaError_t e = cudaDeviceSynchronize();
  return e == cudaSuccess ? 0 : cuda_fail(e, "debug_kernel_timeline");
#else
  (void)buffer;
  return fail(SRL_ESTATE, "debug_kernel_timeline: this library was not built with SRL_DEFINES=SRL_KSTAMP");
#endif
}

extern "C" int64_t srl_learner_workspace_bytes(const srl_learner_t* L) { return L ? L->arena_bytes : 0; }

// coef[2] = the configured lr.  The plain optimizer kernel (constant lr, no momentum) never writes coef[2]; the others overwrite
// it with the lr of every step they run.
static int publish_lr(srl_learner* L) {
  CU(cudaMemcpy(L->coef + 2, &L->cfg.learning_rate, sizeof(float), cudaMemcpyHostToDevice), "publish lr");
  return 0;
}

extern "C" int srl_learner_set_config(srl_learner_t* L, const srl_config_t* cfg) {
  REQ(L, "learner is NULL");
  int rc = check_cfg(cfg);
  if (rc) return rc;
  REQ(cfg->T == L->cfg.T && cfg->B == L->cfg.B && cfg->A == L->cfg.A && cfg->optimizer == L->cfg.optimizer &&
      cfg->precision == L->cfg.precision && cfg->use_lstm == L->cfg.use_lstm, "set_config: T/B/A/optimizer/precision/use_lstm are fixed at creation");
  L->cfg = *cfg;
  return L->report_lr ? publish_lr(L) : 0;
}

extern "C" int srl_learner_set_lr_schedule(srl_learner_t* L, int kind, float lr_end, double frames_per_step, double total_frames) {
  REQ(L, "set_lr_schedule: learner is NULL");
  REQ(kind == SRL_LR_CONSTANT || kind == SRL_LR_LINEAR, "set_lr_schedule: unknown schedule kind %d (0 = constant, 1 = linear)", kind);
  REQ(lr_end >= 0.f && std::isfinite(lr_end), "set_lr_schedule: lr_end=%g must be finite and >= 0", (double)lr_end);
  if (kind == SRL_LR_LINEAR) {
    REQ(total_frames > 0.0 && std::isfinite(total_frames), "set_lr_schedule: total_frames=%g must be finite and > 0", total_frames);
    REQ(frames_per_step > 0.0 && std::isfinite(frames_per_step), "set_lr_schedule: frames_per_step=%g must be finite and > 0", frames_per_step);
  }
  OptExtra& x = L->ox;
  x.schedule = kind == SRL_LR_LINEAR ? SCHED_LINEAR : SCHED_CONSTANT;
  x.lr_end = lr_end;
  x.frames_per_step = kind == SRL_LR_LINEAR ? frames_per_step : 0.0;
  x.total_frames = kind == SRL_LR_LINEAR ? total_frames : 1.0;
  L->report_lr = true;
  return publish_lr(L);
}

extern "C" int srl_learner_set_momentum(srl_learner_t* L, float momentum, float* momentum_buf) {
  REQ(L, "set_momentum: learner is NULL");
  REQ(momentum >= 0.f && std::isfinite(momentum), "set_momentum: momentum=%g must be finite and >= 0", (double)momentum);
  REQ(momentum == 0.f || L->cfg.optimizer == 0, "set_momentum: momentum is an RMSprop option; this learner runs Adam");
  REQ(momentum == 0.f || momentum_buf, "set_momentum: momentum=%g needs a momentum buffer", (double)momentum);
  REQ(!misaligned(momentum_buf, 16), "set_momentum: the momentum buffer must be 16-byte aligned");
  L->ox.momentum = momentum;
  L->ox.buf = momentum == 0.f ? nullptr : momentum_buf;
  return 0;
}

extern "C" int srl_learner_set_option(srl_learner_t* L, const char* name, int value) {
  REQ(L && name, "set_option: NULL argument");
  if (strcmp(name, "column_fusion") == 0) { L->column_fusion = value != 0; return 0; }
  if (strcmp(name, "fused_fwd") == 0) { L->fused_front = value != 0; return 0; }
  if (strcmp(name, "lstm_step_ksplit") == 0) {
    REQ(lstm_step_ksplit_supported(value), "set_option: lstm_step_ksplit=%d must be 1, 2, 3 or 6", value);
    L->lstm_step_ksplit = value;
    return 0;
  }
  return fail(SRL_EINVAL, "set_option: unknown option '%s'", name);
}

extern "C" int srl_learner_set_step(srl_learner_t* L, int64_t step, void* stream) {
  REQ(L && step >= 0 && step < (int64_t(1) << 31), "set_step: bad argument");
  L->step = (int)step;
  const int v = (int)step;       // the device counter drives Adam's bias correction under graph replay
  CU(cudaMemcpyAsync(L->dstep, &v, sizeof(int), cudaMemcpyHostToDevice, (cudaStream_t)stream), "set_step");
  CU(cudaStreamSynchronize((cudaStream_t)stream), "set_step");      // `v` is a stack variable
  return 0;
}
extern "C" int64_t srl_learner_get_step(srl_learner_t* L, void* stream) {
  if (!L) return -1;
  int v = 0;
  if (cudaMemcpyAsync(&v, L->dstep, sizeof(int), cudaMemcpyDeviceToHost, (cudaStream_t)stream) != cudaSuccess) return -1;
  if (cudaStreamSynchronize((cudaStream_t)stream) != cudaSuccess) return -1;
  return v;
}

extern "C" int srl_learner_pack_weights(srl_learner_t* L, void* stream) {
  REQ(L, "learner is NULL");
  L->S.begin_call((cudaStream_t)stream);
  CU(launch_pack_weights(L->P, L->buf.hi.wpack, L->S.main, L->buf.lo.wpack), "pack_weights");
  // the actor step's [W_ih | W_hh] copy: packed here, once per weight version, and never by the learner's own forward
  if (L->lstm_step) CU(lstm_step_pack(L->lstm_step, L->S.main), "lstm_step_pack");
  return 0;
}

namespace srl {
static thread_local bool g_pdl_on = true;      // per calling thread: two learners driven from two threads do not race on it
bool pdl_active() {
  static const bool env_on = [] { const char* e = getenv("SRL_PDL"); return !e || atoi(e) != 0; }();
  return env_on && g_pdl_on;
}
void pdl_set_active(bool on) { g_pdl_on = on; }
}  // namespace srl

// learner step (bf16 mode, lanes): a3 -> fc.weight column order for the fc wgrad GEMM runs on the fc_wgrad lane right after the fc
// forward, under the column kernel (32 CTAs, the GPU is otherwise idle), not in the crowded backward phase; else encoder_backward runs it
static bool early_a3_transpose(const srl_learner* L) { return !L->S.collapsed && L->cfg.precision == 0; }

// step: the forward of the non-LSTM learner step (clears the small gradients; early a3 transpose)
static int encode_impl(srl_learner* L, const uint8_t* obs, int frames, bool step = false) {
  StepStreams& S = L->S;
  // The bf16 operand copies are re-derived from the fp32 master weights at the START of every forward (not at the end
  // of the optimizer step): the pack kernel runs on the pack lane underneath the frame conversion.
  CU(S.fork(LANE_PACK), "fork pack");
  if (step) {     // the accumulated gradient segments (everything before fc.weight) are cleared under the frame conversion
    S.b(PS_ZERO_GRADS);
    CU(cudaMemsetAsync(L->grads, 0, L->small_len * sizeof(float), S.lane(LANE_PACK)), "zero small grads");
    S.e(PS_ZERO_GRADS);
  }
  S.b(PS_PACK);
  CU(launch_pack_weights(L->P, L->buf.hi.wpack, S.lane(LANE_PACK), L->buf.lo.wpack, true), "pack_weights");
  S.e(PS_PACK);
  CU(encoder_forward(obs, frames, L->P, L->buf, L->maps, L->cfg.precision, S, L->fused_front), "encoder_forward");
  if (step && early_a3_transpose(L)) {
    CU(S.fork(LANE_FC_WGRAD), "fork a3 transpose");
    CU(launch_a3_transpose(L->buf.hi.a3, L->buf.a3t, L->cfg.T * L->cfg.B, S.lane(LANE_FC_WGRAD)), "a3_transpose");
  }
  return 0;
}

static int forward_impl(srl_learner* L, const uint8_t* obs, const float* reward, const int64_t* action, int frames, float* logits,
                        float* baseline, bool step = false) {
  REQ(!L->cfg.use_lstm, "this learner was created with use_lstm=1: call the *_lstm entry points");
  int rc = encode_impl(L, obs, frames, step);
  if (rc) return rc;
  L->S.b(PS_HEAD_FWD);
  CU(launch_head_fwd(L->buf.hpart, FC_SPLITS, L->P.bf, L->buf.h, reward, action, L->P.wp, L->P.bp, L->P.wb, L->P.bb, frames, L->cfg.A,
                     logits, baseline, L->S.main), "head_fwd");
  L->S.e(PS_HEAD_FWD);
  return 0;
}

extern "C" int srl_learner_forward(srl_learner_t* L, const uint8_t* obs, const float* reward, const int64_t* action, int rows,
                                   float* policy_logits, float* baseline, void* stream) {
  REQ(L && obs && reward && action && policy_logits && baseline, "learner_forward: NULL pointer");
  REQ(rows >= 1 && rows <= L->cfg.T + 1, "learner_forward: rows=%d must be in [1, T+1=%d]", rows, L->cfg.T + 1);
  REQ(!misaligned(obs, 4), "learner_forward: obs must be 4-byte aligned");
  L->S.begin_call((cudaStream_t)stream);
  return forward_impl(L, obs, reward, action, rows * L->cfg.B, policy_logits, baseline);
}

static int fb_begin(srl_learner* L, const uint8_t* obs, const float* reward, const uint8_t* done, const int64_t* action,
                    const float* behavior_logits, float* losses, float* vs, float* pg_advantages, BwdParts parts) {
  const srl_config_t& c = L->cfg;
  const StepStreams& S = L->S;
  const int NF = (c.T + 1) * c.B, NB = c.T * c.B;
  // heads + V-trace/losses + dh: one fused column kernel when its shared-memory footprint fits, else three kernels
  const bool fused = L->column_fusion && column_step_supported(c.T, c.B, c.A);
  const TailStep ts = tail_step(c, behavior_logits, action, reward, done, vs, pg_advantages, L->dlogits, L->dbaseline, losses, L->scratch);
  int rc;
  if (fused) {
    REQ(!L->cfg.use_lstm, "this learner was created with use_lstm=1: call the *_lstm entry points");
    rc = encode_impl(L, obs, NF, true);
    if (rc) return rc;
    S.b(PS_TAIL);
    CU(launch_column_step(ts, L->buf.hpart, FC_SPLITS, L->P.bf, L->buf.h, L->P.wp, L->P.bp, L->P.wb, L->P.bb, L->logits, L->baseline,
                          L->buf.hi.dh, L->buf.lo.dh, S.main), "column_step");
    S.e(PS_TAIL);
  } else {
    rc = forward_impl(L, obs, reward, action, NF, L->logits, L->baseline, true);
    if (rc) return rc;
    S.b(PS_TAIL);
    CU(launch_impala_tail(ts, L->logits, L->baseline, S.main), "impala_tail");
    S.e(PS_TAIL);
  }
  S.b(PS_HEAD_BWD);
  CU(S.fork(LANE_FC_WGRAD), "fork head wgrad");      // joined by encoder_backward with the fc wgrad
  CU(launch_head_bwd(L->dlogits, L->dbaseline, L->buf.h, reward, action, L->P.wp, L->P.wb, NB, c.A, L->buf.hi.dh, L->G.wp, L->G.bp, L->G.wb,
                     L->G.bb, L->head_part, S.main, S.lane(LANE_FC_WGRAD), !fused, L->buf.lo.dh), "head_bwd");
  S.e(PS_HEAD_BWD);
  CU(encoder_backward(NB, L->buf, L->G, L->maps, c.precision, S, parts, early_a3_transpose(L)), "encoder_backward");
  L->have_fwd = true;
  return 0;
}

extern "C" int srl_learner_forward_backward(srl_learner_t* L, const uint8_t* obs, const float* reward, const uint8_t* done,
                                            const int64_t* action, const float* behavior_logits, float* losses, float* vs,
                                            float* pg_advantages, void* stream) {
  REQ(L && obs && reward && done && action && behavior_logits && losses, "learner_forward_backward: NULL pointer");
  REQ(!misaligned(obs, 4), "learner_forward_backward: obs must be 4-byte aligned");
  L->S.begin_call((cudaStream_t)stream);
  return fb_begin(L, obs, reward, done, action, behavior_logits, losses, vs, pg_advantages, BWD_BOTH);
}

extern "C" int srl_learner_forward_backward_begin(srl_learner_t* L, const uint8_t* obs, const float* reward, const uint8_t* done,
                                                  const int64_t* action, const float* behavior_logits, float* losses, float* vs,
                                                  float* pg_advantages, void* stream) {
  REQ(L && obs && reward && done && action && behavior_logits && losses, "learner_forward_backward_begin: NULL pointer");
  REQ(!misaligned(obs, 4), "learner_forward_backward_begin: obs must be 4-byte aligned");
  L->S.begin_call((cudaStream_t)stream);
  return fb_begin(L, obs, reward, done, action, behavior_logits, losses, vs, pg_advantages, BWD_FC);
}

extern "C" int srl_learner_backward_finish(srl_learner_t* L, const uint8_t* obs, void* stream) {
  REQ(L && obs, "learner_backward_finish: NULL pointer");
  REQ(L->have_fwd, "learner_backward_finish: call srl_learner_forward_backward_begin first");
  const srl_config_t& c = L->cfg;
  L->S.begin_call((cudaStream_t)stream);
  CU(encoder_backward(c.T * c.B, L->buf, L->G, L->maps, c.precision, L->S, BWD_CONV, false), "encoder_backward");
  return 0;
}

static int forward_lstm_impl(srl_learner* L, const uint8_t* obs, const float* reward, const uint8_t* done, const int64_t* action,
                             const float* h0, const float* c0, float* logits, float* baseline, float* hT, float* cT) {
  REQ(L->cfg.use_lstm && L->lstm, "this learner was created with use_lstm=0");
  const srl_config_t& c = L->cfg;
  const cudaStream_t st = L->S.main;
  const int NF = (c.T + 1) * c.B;
  int rc = encode_impl(L, obs, NF);
  if (rc) return rc;
  CU(launch_core_build(L->buf.hpart, FC_SPLITS, L->P.bf, reward, action, NF, c.A, L->buf.h, L->core, st), "core_build");
  rc = srl_lstm_forward(L->lstm, L->core, done, h0, c0, L->lstm_out, hT, cT, st);
  if (rc) return rc;
  CU(launch_head_dense_fwd(L->lstm_out, L->P.wp, L->P.bp, L->P.wb, L->P.bb, NF, c.A, logits, baseline, st), "head_dense_fwd");
  return 0;
}

extern "C" int srl_learner_forward_lstm(srl_learner_t* L, const uint8_t* obs, const float* reward, const uint8_t* done, const int64_t* action,
                                        const float* h0, const float* c0, float* policy_logits, float* baseline, float* hT, float* cT,
                                        void* stream) {
  REQ(L && obs && reward && done && action && h0 && c0 && policy_logits && baseline, "learner_forward_lstm: NULL pointer");
  L->S.begin_call((cudaStream_t)stream);
  return forward_lstm_impl(L, obs, reward, done, action, h0, c0, policy_logits, baseline, hT, cT);
}

extern "C" int srl_learner_forward_lstm_step(srl_learner_t* L, const uint8_t* obs, const float* reward, const uint8_t* done,
                                             const int64_t* action, const float* h_in, const float* c_in, float* policy_logits,
                                             float* baseline, float* h_out, float* c_out, void* stream) {
  // the pointer checks come before any use of the context
  REQ(obs && reward && done && action && h_in && c_in && policy_logits && baseline && h_out && c_out, "learner_forward_lstm_step: NULL pointer");
  REQ(h_out != h_in && h_out != c_in && c_out != h_in && c_out != c_in && h_out != c_out,
      "learner_forward_lstm_step: h_out / c_out must not alias h_in, c_in or each other");
  REQ(L, "learner_forward_lstm_step: learner is NULL");
  REQ(L->cfg.use_lstm && L->lstm_step, "learner_forward_lstm_step: this learner was created with use_lstm=0");
  REQ(L->cfg.precision == 0, "learner_forward_lstm_step: the step runs bf16 operands only (precision = 0)");
  const srl_config_t& c = L->cfg;
  const int B = c.B, H = 513 + c.A;
  const int64_t sb = (int64_t)2 * B * H * 4;
  const Span s[4] = {{h_in, sb, false, "h_in"}, {c_in, sb, false, "c_in"}, {h_out, sb, true, "h_out"}, {c_out, sb, true, "c_out"}};
  int rc = check_spans(s, 4, "learner_forward_lstm_step");
  if (rc) return rc;
  REQ(!misaligned(obs, 4), "learner_forward_lstm_step: obs must be 4-byte aligned");
  const cudaStream_t st = L->S.begin_call((cudaStream_t)stream);
  rc = encode_impl(L, obs, B);
  if (rc) return rc;
  CU(launch_core_build(L->buf.hpart, FC_SPLITS, L->P.bf, reward, action, B, c.A, L->buf.h, L->core, st), "core_build");
  CU(lstm_step_forward(L->lstm_step, L->core, done, h_in, c_in, h_out, c_out, L->lstm_step_ksplit, st), "lstm_step");
  CU(launch_head_dense_fwd(h_out + (size_t)B * H, L->P.wp, L->P.bp, L->P.wb, L->P.bb, B, c.A, policy_logits, baseline, st), "head_dense_fwd");
  return 0;
}

extern "C" int srl_learner_forward_backward_lstm(srl_learner_t* L, const uint8_t* obs, const float* reward, const uint8_t* done,
                                                 const int64_t* action, const float* behavior_logits, const float* h0, const float* c0,
                                                 float* losses, float* vs, float* pg_advantages, void* stream) {
  REQ(L && obs && reward && done && action && behavior_logits && h0 && c0 && losses, "learner_forward_backward_lstm: NULL pointer");
  const cudaStream_t st = L->S.begin_call((cudaStream_t)stream);
  const srl_config_t& c = L->cfg;
  const int NB = c.T * c.B;
  int rc = forward_lstm_impl(L, obs, reward, done, action, h0, c0, L->logits, L->baseline, nullptr, nullptr);
  if (rc) return rc;
  CU(launch_impala_tail(tail_step(c, behavior_logits, action, reward, done, vs, pg_advantages, L->dlogits, L->dbaseline, losses, L->scratch),
                        L->logits, L->baseline, st), "impala_tail");
  CU(cudaMemsetAsync(L->grads, 0, L->small_len * sizeof(float), st), "zero small grads");
  CU(cudaMemsetAsync(L->grads + L->lstm_off0, 0, L->lstm_len * sizeof(float), st), "zero lstm grads");
  CU(launch_head_dense_bwd(L->lstm_out, L->dlogits, L->dbaseline, L->P.wp, L->P.wb, NB, c.A, L->dout, L->G.wp, L->G.bp, L->G.wb, L->G.bb, st),
     "head_dense_bwd");
  rc = srl_lstm_backward(L->lstm, L->dout, done, L->dcore, st);
  if (rc) return rc;
  CU(launch_dcore_to_dh(L->dcore, L->buf.h, NB, c.A, L->buf.hi.dh, st), "dcore_to_dh");
  CU(encoder_backward(NB, L->buf, L->G, L->maps, c.precision, L->S, BWD_BOTH, false), "encoder_backward");
  L->have_fwd = true;
  return 0;
}

// clip_grad_norm_ + optimizer in one cooperative kernel (profile slot: optimizer); P: the data-parallel step over these peers
static int apply_impl(srl_learner_t* L, const DpPeers* P, float* grad_norm_out) {
  const srl_config_t& c = L->cfg;
  const bool adam = c.optimizer != 0;
  const cudaStream_t st = L->S.main;
  L->step += 1;
  const OptStep o = {adam ? 1 : 0, L->params, L->grads, L->opt0, adam ? L->opt1 : nullptr, L->nparams, c.max_grad_norm, L->coef,
                     L->scratch + 2048, c.learning_rate, adam ? c.adam_beta1 : c.alpha, adam ? c.adam_beta2 : 0.f,
                     adam ? c.adam_eps : c.epsilon, L->step, L->dstep, L->ox};
  L->S.b(PS_OPTIMIZER);
  CU(P ? launch_dp_clip_optim(o, *P, st) : launch_clip_optim(o, st), P ? (adam ? "dp clip+adam" : "dp clip+rmsprop") : (adam ? "clip+adam" : "clip+rmsprop"));
  L->S.e(PS_OPTIMIZER);
  if (grad_norm_out) CU(cudaMemcpyAsync(grad_norm_out, L->coef, (L->report_lr ? 3 : 2) * sizeof(float), cudaMemcpyDeviceToDevice, st), "copy coef");
  return 0;
}

extern "C" int srl_learner_apply_gradients(srl_learner_t* L, float* grad_norm_out, void* stream) {
  REQ(L, "learner is NULL");
  L->S.begin_call((cudaStream_t)stream);
  return apply_impl(L, nullptr, grad_norm_out);
}

extern "C" int srl_learner_apply_gradients_dp(srl_learner_t* L, const srl_dp_peers_t* peers, float* grad_norm_out, void* stream) {
  REQ(L && peers, "apply_gradients_dp: NULL argument");
  REQ(peers->world >= 2 && peers->world <= 8 && peers->rank >= 0 && peers->rank < peers->world, "apply_gradients_dp: world=%d rank=%d",
      peers->world, peers->rank);
  REQ(peers->grads[peers->rank] == (void*)L->grads, "apply_gradients_dp: grads[rank] must be the learner's gradient buffer");
  DpPeers P;
  for (int i = 0; i < 8; ++i) {
    P.g[i] = i < peers->world ? (float*)peers->grads[i] : nullptr;
    P.ctl[i] = i < peers->world ? (unsigned*)peers->ctl[i] : nullptr;
    P.rs[i] = i < peers->world ? (float*)peers->exchange[i] : nullptr;
    REQ(i >= peers->world || (P.g[i] && P.ctl[i] && P.rs[i]), "apply_gradients_dp: NULL peer pointer %d", i);
  }
  P.rank = peers->rank; P.world = peers->world; P.mc_g = (float*)peers->grads_multicast;
  L->S.begin_call((cudaStream_t)stream);
  return apply_impl(L, &P, grad_norm_out);
}

extern "C" int srl_learner_set_profiling(srl_learner_t* L, int enable) {
  REQ(L, "learner is NULL");
  if (enable && !L->S.slot_events[0])
    for (int i = 0; i < 2 * PS_COUNT; ++i) CU(cudaEventCreate(&L->S.slot_events[i]), "cudaEventCreate");
  L->S.profiling = enable != 0;
  return 0;
}
extern "C" int srl_profile_slot_count(void) { return PS_COUNT; }
extern "C" const char* srl_profile_slot_name(int slot) { return (slot >= 0 && slot < PS_COUNT) ? kSlotNames[slot] : ""; }
extern "C" int srl_learner_profile_collect(srl_learner_t* L, float* ms_out_host) {
  REQ(L && ms_out_host, "profile_collect: NULL argument");
  REQ(L->S.profiling, "profile_collect: profiling is off");
  for (int i = 0; i < PS_COUNT; ++i) {
    float ms = 0.f;
    cudaError_t e = cudaEventSynchronize(L->S.slot_events[2 * i + 1]);
    if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, L->S.slot_events[2 * i], L->S.slot_events[2 * i + 1]);
    if (e != cudaSuccess) { cudaGetLastError(); ms = -1.f; }   // slot not recorded in the last step
    ms_out_host[i] = ms;
  }
  return 0;
}

extern "C" int srl_learner_snapshot_params(srl_learner_t* L, float* dst, const float* losses, void* stream) {
  REQ(L && dst, "snapshot_params: NULL argument");
  REQ(!misaligned(dst, 16), "snapshot_params: dst must be 16-byte aligned");
  CU(launch_snapshot_if_finite(dst, L->params, L->nparams, losses, (cudaStream_t)stream), "snapshot_params");
  return 0;
}

// Pinning of caller-owned HOST memory (the shared-memory trajectory ring, the actors' shared parameter tensors) so that the
// copy engine reads / writes it directly.  A stale registration left by a freed mapping at the same address (or a second tensor
// on an already pinned page) is replaced instead of failing, and no sticky error is left behind for the next CUDA call.
extern "C" int srl_host_register(void* ptr_host, int64_t bytes) {
  REQ(ptr_host && bytes > 0, "host_register: bad argument");
  cudaError_t e = cudaHostRegister(ptr_host, (size_t)bytes, cudaHostRegisterDefault);
  if (e == cudaErrorHostMemoryAlreadyRegistered) {
    cudaGetLastError();
    cudaHostUnregister(ptr_host);
    cudaGetLastError();
    e = cudaHostRegister(ptr_host, (size_t)bytes, cudaHostRegisterDefault);
    if (e == cudaErrorHostMemoryAlreadyRegistered) { cudaGetLastError(); return 0; }     // part of a larger live registration: fine
  }
  if (e != cudaSuccess) { cudaGetLastError(); return cuda_fail(e, "cudaHostRegister"); }
  return 0;
}
extern "C" int srl_host_unregister(void* ptr_host) {
  REQ(ptr_host, "host_unregister: NULL");
  cudaError_t e = cudaHostUnregister(ptr_host);
  cudaGetLastError();
  return (e == cudaSuccess || e == cudaErrorHostMemoryNotRegistered) ? 0 : cuda_fail(e, "cudaHostUnregister");
}

extern "C" int srl_memcpy_d2d(void* dst, const void* src, int64_t bytes, void* stream) {
  REQ(dst && src && bytes >= 0, "memcpy_d2d: bad argument");
  CU(cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream), "memcpy_d2d");
  return 0;
}

extern "C" int srl_learner_debug_buffer(srl_learner_t* L, const char* name, void** ptr, int64_t* count) {
  REQ(L && name && ptr && count, "debug_buffer: NULL argument");
  if (strncmp(name, "lstm_step_", 10) == 0) {     // the actor step's bf16 operands: xh [2][B][2Hp] = [x | m.h], w [2][4Hp][2Hp]
    REQ(L->lstm_step, "debug_buffer: '%s' exists only with use_lstm = 1", name);
    void *xh, *w;
    int64_t nxh, nw;
    lstm_step_buffers(L->lstm_step, &xh, &nxh, &w, &nw);
    if (strcmp(name, "lstm_step_xh") == 0) { *ptr = xh; *count = nxh; return 0; }
    if (strcmp(name, "lstm_step_w") == 0) { *ptr = w; *count = nw; return 0; }
  }
  WsRow t[WS_MAX_ROWS];
  const int n = workspace_table(L, t);
  const size_t len = strlen(name);
  const bool twin = len > 3 && strcmp(name + len - 3, "_lo") == 0;
  for (int i = 0; i < n; ++i) {
    const WsRow& r = t[i];
    if (!r.name) continue;
    if (strcmp(r.name, name) == 0) { *ptr = *r.hi; *count = r.count; return 0; }
    if (twin && r.lo && strlen(r.name) == len - 3 && strncmp(r.name, name, len - 3) == 0) {
      if (!*r.lo) return fail(SRL_ESTATE, "debug_buffer: '%s' exists only in the fp32-accurate operand mode (precision = 1)", name);
      *ptr = *r.lo; *count = r.count; return 0;
    }
  }
  return fail(SRL_EINVAL, "debug_buffer: unknown buffer '%s'", name);
}

// ------------------------------------------------------------------------------------------------
// stand-alone encoder: the learner's encoder kernels on caller-owned blocks, one forward and its backward per autograd call
// ------------------------------------------------------------------------------------------------
struct srl_encoder {
  int precision;
  StepStreams S;                  // the lanes beside the caller's stream (no per-kernel profiling)
};

static int check_precision(int precision, const char* what) {
  REQ(precision == 0 || precision == 1, "%s: precision=%d must be 0 (bf16 operands) or 1 (fp32-accurate split operands)", what, precision);
  return 0;
}

extern "C" int srl_encoder_create(int precision, srl_encoder_t** out) {
  REQ(out, "encoder_create: NULL argument");
  int rc = check_precision(precision, "encoder_create");
  if (rc) return rc;
  srl_encoder* E = new (std::nothrow) srl_encoder();
  REQ(E, "out of host memory");
  E->precision = precision;
  create_lanes(E->S);
  *out = E;
  return 0;
}

extern "C" int srl_encoder_destroy(srl_encoder_t* E) {
  if (!E) return 0;
  destroy_lanes(E->S);
  delete E;
  return 0;
}

extern "C" int srl_encoder_sizes(int frames, int precision, int64_t* saved_bytes, int64_t* scratch_bytes) {
  REQ(saved_bytes && scratch_bytes, "encoder_sizes: NULL argument");
  REQ(frames >= 1 && frames <= MAX_FRAMES, "encoder_sizes: frames=%d must be in [1, %d]", frames, MAX_FRAMES);
  int rc = check_precision(precision, "encoder_sizes");
  if (rc) return rc;
  EncoderBuffers b = {};
  WsRow t[ENC_ROWS];
  encoder_rows(b, frames, frames, t);
  block_bytes(t, ENC_ROWS, ENC_SAVED_ROWS, precision == 1, saved_bytes, scratch_bytes);
  return 0;
}

// the argument checks both calls share: shape, the two blocks' alignment and sizes
static int check_encoder_call(const srl_encoder* E, int frames, int A, const void* saved, const void* scratch, int64_t* sb, int64_t* kb,
                              const char* what) {
  REQ(frames >= 1 && frames <= MAX_FRAMES, "%s: frames=%d must be in [1, %d]", what, frames, MAX_FRAMES);
  REQ(A >= 1 && A <= 31, "%s: A=%d must be in [1,31]", what, A);
  REQ(!misaligned(saved, 256) && !misaligned(scratch, 256), "%s: saved and scratch must be 256-byte aligned", what);
  return srl_encoder_sizes(frames, E->precision, sb, kb);
}

// the blocks of one call -> the encoder buffers and their tensor maps, encoded on the host for this call (legal under stream capture)
static int encoder_call_setup(const srl_encoder* E, int frames, void* saved, void* scratch, EncoderBuffers* b, TmaMaps* maps,
                              const char* what) {
  WsRow t[ENC_ROWS];
  *b = EncoderBuffers{};
  encoder_rows(*b, frames, frames, t);
  b->NF = frames;
  CU(carve_blocks(t, ENC_ROWS, ENC_SAVED_ROWS, E->precision == 1, saved, scratch), "cudaSetDevice");
  const char* why = nullptr;
  if (build_tma_maps(*b, frames, frames, maps, &why) != cudaSuccess)
    return fail(SRL_ESTATE, "%s: building TMA tensor map '%s' failed (driver without cuTensorMapEncodeTiled?)", what, why ? why : "?");
  return 0;
}

extern "C" int srl_encoder_forward(srl_encoder_t* E, const uint8_t* obs, const float* reward, const int64_t* action, int frames, int A,
                                   const float* const* weights8, void* saved, void* scratch, float* core_out, void* stream) {
  REQ(E && obs && reward && action && weights8 && saved && scratch && core_out, "encoder_forward: NULL pointer");
  for (int i = 0; i < 8; ++i) REQ(weights8[i], "encoder_forward: weights8[%d] is NULL", i);
  int64_t sb = 0, kb = 0;
  int rc = check_encoder_call(E, frames, A, saved, scratch, &sb, &kb, "encoder_forward");
  if (rc) return rc;
  REQ(!misaligned(obs, 4), "encoder_forward: obs must be 4-byte aligned");
  for (int i = 0; i < 8; ++i) REQ(!misaligned(weights8[i], 16), "encoder_forward: weights8[%d] must be 16-byte aligned", i);
  int64_t cnt[12];
  layout(A, nullptr, cnt);
  Span s[14] = {{obs, (int64_t)frames * 28224, false, "obs"}, {reward, (int64_t)frames * 4, false, "reward"},
                {action, (int64_t)frames * 8, false, "action"}};
  int n = 3;
  for (int i = 0; i < 8; ++i) s[n++] = {weights8[i], cnt[i] * 4, false, kW8[i]};
  s[n++] = {saved, sb, true, "saved"}; s[n++] = {scratch, kb, true, "scratch"}; s[n++] = {core_out, (int64_t)frames * (513 + A) * 4, true, "core_out"};
  rc = check_spans(s, n, "encoder_forward");
  if (rc) return rc;
  ParamPtrs P = {};
  P.w1 = const_cast<float*>(weights8[0]); P.b1 = const_cast<float*>(weights8[1]); P.w2 = const_cast<float*>(weights8[2]);
  P.b2 = const_cast<float*>(weights8[3]); P.w3 = const_cast<float*>(weights8[4]); P.b3 = const_cast<float*>(weights8[5]);
  P.wf = const_cast<float*>(weights8[6]); P.bf = const_cast<float*>(weights8[7]);
  EncoderBuffers b;
  TmaMaps maps;
  rc = encoder_call_setup(E, frames, saved, scratch, &b, &maps, "encoder_forward");
  if (rc) return rc;
  StepStreams& S = E->S;
  const cudaStream_t st = S.begin_call((cudaStream_t)stream);
  // as the learner's forward: the weights are packed into `saved` on the pack lane under the frame conversion (which writes conv1's copy)
  CU(S.fork(LANE_PACK), "fork pack");
  CU(launch_pack_weights(P, b.hi.wpack, S.lane(LANE_PACK), b.lo.wpack, true), "pack_weights");
  CU(encoder_forward(obs, frames, P, b, maps, E->precision, S, false), "encoder_forward");
  CU(launch_core_build(b.hpart, FC_SPLITS, P.bf, reward, action, frames, A, b.h, core_out, st), "core_build");
  return 0;
}

extern "C" int srl_encoder_backward(srl_encoder_t* E, const float* dcore, int frames, int A, void* saved, void* scratch, float* const* grads8,
                                    void* stream) {
  REQ(E && dcore && saved && scratch && grads8, "encoder_backward: NULL pointer");
  for (int i = 0; i < 8; ++i) REQ(grads8[i], "encoder_backward: grads8[%d] is NULL", i);
  int64_t sb = 0, kb = 0;
  int rc = check_encoder_call(E, frames, A, saved, scratch, &sb, &kb, "encoder_backward");
  if (rc) return rc;
  for (int i = 0; i < 8; ++i) REQ(!misaligned(grads8[i], 16), "encoder_backward: grads8[%d] must be 16-byte aligned", i);
  int64_t cnt[12];
  layout(A, nullptr, cnt);
  Span s[11] = {{dcore, (int64_t)frames * (513 + A) * 4, false, "dcore"}, {saved, sb, false, "saved"}, {scratch, kb, true, "scratch"}};
  int n = 3;
  for (int i = 0; i < 8; ++i) s[n++] = {grads8[i], cnt[i] * 4, true, kG8[i]};
  rc = check_spans(s, n, "encoder_backward");
  if (rc) return rc;
  ParamPtrs G = {};
  G.w1 = grads8[0]; G.b1 = grads8[1]; G.w2 = grads8[2]; G.b2 = grads8[3]; G.w3 = grads8[4]; G.b3 = grads8[5]; G.wf = grads8[6]; G.bf = grads8[7];
  EncoderBuffers b;
  TmaMaps maps;
  rc = encoder_call_setup(E, frames, saved, scratch, &b, &maps, "encoder_backward");
  if (rc) return rc;
  StepStreams& S = E->S;
  const cudaStream_t st = S.begin_call((cudaStream_t)stream);
  // the zeros of the gradient grids are the padding of the transposed convolutions: da3 .. da1, low twins included, lie between
  // hi.da3 and wgrad_part (encoder_rows)
  CU(cudaMemsetAsync(b.hi.da3, 0, reinterpret_cast<char*>(b.wgrad_part) - reinterpret_cast<char*>(b.hi.da3), st), "clear gradient grids");
  // the conv bias sums are added into their gradients; every other gradient is stored
  CU(cudaMemsetAsync(G.b1, 0, cnt[1] * 4, st), "zero conv1 bias grad");
  CU(cudaMemsetAsync(G.b2, 0, cnt[3] * 4, st), "zero conv2 bias grad");
  CU(cudaMemsetAsync(G.b3, 0, cnt[5] * 4, st), "zero conv3 bias grad");
  CU(launch_dcore_to_dh(dcore, b.h, frames, A, b.hi.dh, st, b.lo.dh), "dcore_to_dh");
  CU(encoder_backward(frames, b, G, maps, E->precision, S, BWD_BOTH, false), "encoder_backward");
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Ape-X learner step: three encoder forwards on the context's blocks, the Q-learning tail (dqn.cu), the encoder backward over s,
// clip + Adam, and the priorities into the sampler's trees
// ------------------------------------------------------------------------------------------------
// The Q network's tensors in state_dict order: conv1..3 {weight, bias}, then fc and the head layers (q, or value [1, 512] and
// advantage [A, 512]) as {weight, bias}, or noisy as {weight_mu, weight_sigma, bias_mu, bias_sigma}.  In memory (each segment padded
// to 4 floats) they come in groups, each group by (mu / sigma, layer, weight / bias): the conv tensors; fc's biases; the head weights
// and the head biases (plain: the weights first; noisy: the biases first); fc's weights.  So the dueling head's weight rows are one
// [(A + 1)][512] block for the kernels (noisy: the mu rows one, the sigma rows another), the value row first.  The categorical head
// (K atoms) is q with A K rows (row a K + k: atom k of action a), the quantile head (N quantiles) q with A N rows (row a N + i:
// quantile i of action a).  The distributional dueling head (W = K or N rows per action) has value [W, 512] and advantage [A W, 512]
// in the dueling head's places: one [(W + A W)][512] weight block, the value rows first.
namespace srl {
int64_t apex_layout(const ApexNetDesc& d, int64_t* off, int64_t* cnt) {
  const int64_t V = d.vrows, R = adv_rows(d);
  const int64_t layers[6][2] = {{32, 256}, {64, 512}, {64, 576}, {512, 3136}, {V ? V : R, 512}, {R, 512}};  // [out, in]
  const int nl = V ? 6 : 5, S = d.noisy ? 2 : 1;
  // the memory group of [conv, fc, head][weight, bias], without and with noise
  static const int group[2][3][2] = {{{0, 0}, {4, 1}, {2, 3}}, {{0, 0}, {4, 1}, {3, 2}}};
  int64_t o = 0;
  for (int g = 0; g < 5; ++g)
    for (int s = 0; s < S; ++s)
      for (int l = 0, i = 0; l < nl; ++l) {
        const int kind = l < 3 ? 0 : l == 3 ? 1 : 2, ns = kind ? S : 1;       // i: the layer's first tensor, ns: its mu / sigma
        for (int p = 0; p < 2; ++p) {
          if (group[d.noisy][kind][p] != g || s >= ns) continue;
          const int t = i + p * ns + s;
          const int64_t c = p ? layers[l][0] : layers[l][0] * layers[l][1];
          if (off) off[t] = o;
          if (cnt) cnt[t] = c;
          o += (c + 3) & ~int64_t(3);
        }
        i += 2 * ns;
      }
  return o;
}

int make_apex_desc(const char* who, int A, int dueling, int num_atoms, float v_min, float v_max, int num_quantiles, float kappa,
                   int dist_dueling, int noisy, ApexNetDesc* d) {
  REQ(A >= 1 && A <= 31, "%s: A=%d must be in [1,31]", who, A);
  REQ(dueling == 0 || dueling == 1, "%s: dueling=%d must be 0 (q = Linear(512, A)) or 1 (dueling head)", who, dueling);
  REQ(noisy == 0 || noisy == 1, "%s: noisy=%d must be 0 (plain layers) or 1 (noisy fc and head layers)", who, noisy);
  REQ(dist_dueling == 0 || dist_dueling == 1, "%s: dist_dueling=%d must be 0 or 1 (the distributional dueling head)", who, dist_dueling);
  if (dist_dueling) {
    REQ(dueling == 0, "%s: dist_dueling=1 with dueling=1 is not supported (dueling is the scalar dueling head)", who);
    REQ(num_atoms > 0 || num_quantiles > 0, "%s: dist_dueling=1 needs the categorical head (num_atoms > 0) or the quantile head "
        "(num_quantiles > 0)", who);
  }
  REQ(num_atoms == 0 || (num_atoms >= 2 && num_atoms <= CAT_MAX_ATOMS), "%s: num_atoms=%d must be 0 (a scalar Q head) or in [2, %d]", who,
      num_atoms, CAT_MAX_ATOMS);
  REQ(num_quantiles == 0 || (num_quantiles >= 2 && num_quantiles <= QR_MAX_QUANTILES),
      "%s: num_quantiles=%d must be 0 (no quantile head) or in [2, %d]", who, num_quantiles, QR_MAX_QUANTILES);
  *d = ApexNetDesc{QHead{dueling ? Q_DUELING : Q_PLAIN, A, A + dueling}, noisy, dueling};
  if (num_quantiles) {
    REQ(std::isfinite(kappa) && kappa > 0.f, "%s: kappa=%g must be finite and > 0 (the quantile Huber threshold)", who, (double)kappa);
    REQ(dueling == 0, "%s: the quantile head (num_quantiles=%d) with dueling=1 is not supported", who, num_quantiles);
    REQ(num_atoms == 0, "%s: the quantile head (num_quantiles=%d) with the categorical head (num_atoms=%d) is not supported", who,
        num_quantiles, num_atoms);
    d->head.kind = Q_QUANTILE;
    d->head.R = A * num_quantiles;
    d->head.qr = QrSetting{num_quantiles, kappa};
    d->vrows = dist_dueling ? num_quantiles : 0;
    return 0;
  }
  if (num_atoms == 0) return 0;
  REQ(std::isfinite(v_min) && std::isfinite(v_max) && v_min < v_max, "%s: v_min=%g, v_max=%g must be finite with v_min < v_max", who,
      (double)v_min, (double)v_max);
  const CatSupport c = cat_support(num_atoms, v_min, v_max);
  REQ(std::isfinite(c.dz) && c.dz > 0.f, "%s: the atom spacing (v_max - v_min) / (num_atoms - 1) = %g is not a positive finite float", who,
      (double)c.dz);
  REQ(dueling == 0, "%s: the categorical head (num_atoms=%d) with dueling=1 is not supported", who, num_atoms);
  d->head.kind = Q_CATEGORICAL;
  d->head.R = A * num_atoms;
  d->head.c = c;
  d->vrows = dist_dueling ? num_atoms : 0;
  return 0;
}

ApexNet bind_apex(const ApexNetDesc& d, float* base) {
  int64_t off[18];
  apex_layout(d, off, nullptr);
  auto at = [&](int t) { return base + off[t]; };
  const bool dueling = d.vrows > 0;         // a value layer before the advantage layer
  const int S = d.noisy ? 2 : 1, F = 6, H = F + 2 * S, V = H + 2 * S;     // the first tensor of fc, the head, the advantage layer
  ApexNet n = {};
  for (int i = 0; i < 6; ++i) n.w8[i] = at(i);
  n.w8[6] = at(F);
  n.w8[7] = at(F + S);
  n.q = d.head;
  n.q.W = at(H); n.q.b = at(H + S); n.q.ba = dueling ? at(V + S) : nullptr;
  n.g = {at(H), at(H + S), dueling ? at(V + S) : nullptr};
  for (int s = 0; d.noisy && s < 2; ++s) {
    n.nz.fc_w[s] = at(F + s);
    n.nz.fc_b[s] = at(F + S + s);
    n.nz.h_w[s] = at(H + s);
    n.nz.h_b[s] = at(H + S + s);
    n.nz.h_ba[s] = dueling ? at(V + S + s) : nullptr;
  }
  return n;
}

ApexNet apex_forward_net(const ApexNetDesc& d, const ApexNet& net, const NoisyWeights& w) {
  if (!d.noisy) return net;
  ApexNet r = net;
  r.w8[6] = w.fc_w;
  r.w8[7] = w.fc_b;
  r.q.W = w.h_w; r.q.b = w.h_b; r.q.ba = d.vrows ? w.h_ba : nullptr;
  return r;
}

int noise_rows(const ApexNetDesc& d, int which, float** normals, float** noise, NoisyWeights* w, WsRow* t) {
  static const char* const names[3][7] = {
      {"normals", "noise", "fc_weight", "fc_bias", "head_weight", "head_bias", "head_adv_bias"},
      {"normals_online", "noise_online", "fc_weight_online", "fc_bias_online", "head_weight_online", "head_bias_online", "head_adv_bias_online"},
      {"normals_target", "noise_target", "fc_weight_target", "fc_bias_target", "head_weight_target", "head_bias_target", "head_adv_bias_target"}};
  const char* const* nm = names[which];
  const int64_t on = d.noisy, V = d.vrows, R = adv_rows(d);
  t[0] = ws_row(nm[0], noise_count(d), normals);
  t[1] = ws_row(nm[1], noise_count(d), noise);
  t[2] = ws_row(nm[2], on * NOISE_FC_OUT * NOISE_FC_IN, &w->fc_w);
  t[3] = ws_row(nm[3], on * NOISE_FC_OUT, &w->fc_b);
  t[4] = ws_row(nm[4], on * (V + R) * NOISE_HEAD_IN, &w->h_w);
  t[5] = ws_row(nm[5], on * (V ? V : R), &w->h_b);
  t[6] = ws_row(nm[6], on * (V ? R : 0), &w->h_ba);
  return 7;
}
}  // namespace srl

extern "C" int64_t srl_apex_param_layout(int A, int64_t* offsets10, int64_t* counts10) {
  return apex_layout(ApexNetDesc{QHead{Q_PLAIN, A, A}, 0, 0}, offsets10, counts10);
}
extern "C" int64_t srl_apex_param_layout_ex(int A, int dueling, int64_t* offsets12, int64_t* counts12) {
  REQ(A >= 1 && A <= 31, "apex_param_layout: A=%d must be in [1,31]", A);
  REQ(dueling == 0 || dueling == 1, "apex_param_layout: dueling=%d must be 0 or 1", dueling);
  return apex_layout(ApexNetDesc{QHead{dueling ? Q_DUELING : Q_PLAIN, A, A + dueling}, 0, dueling}, offsets12, counts12);
}
extern "C" int64_t srl_apex_param_layout_cat(int A, int num_atoms, int64_t* offsets10, int64_t* counts10) {
  REQ(A >= 1 && A <= 31, "apex_param_layout: A=%d must be in [1,31]", A);
  REQ(num_atoms == 0 || (num_atoms >= 2 && num_atoms <= CAT_MAX_ATOMS), "apex_param_layout: num_atoms=%d must be 0 (a scalar Q head) or in [2, %d]",
      num_atoms, CAT_MAX_ATOMS);
  return apex_layout(ApexNetDesc{QHead{num_atoms ? Q_CATEGORICAL : Q_PLAIN, A, A * (num_atoms ? num_atoms : 1)}, 0, 0}, offsets10, counts10);
}
extern "C" int64_t srl_apex_param_layout_noisy(int A, int dueling, int num_atoms, int noisy, int64_t* offsets18, int64_t* counts18) {
  return srl_apex_param_layout_quantile(A, dueling, num_atoms, 0, noisy, offsets18, counts18);
}
extern "C" int64_t srl_apex_param_layout_quantile(int A, int dueling, int num_atoms, int num_quantiles, int noisy, int64_t* offsets18,
                                                  int64_t* counts18) {
  return srl_apex_param_layout_dist_dueling(A, dueling, num_atoms, num_quantiles, 0, noisy, offsets18, counts18);
}
extern "C" int64_t srl_apex_param_layout_dist_dueling(int A, int dueling, int num_atoms, int num_quantiles, int dist_dueling, int noisy,
                                                      int64_t* offsets18, int64_t* counts18) {
  ApexNetDesc d;      // the support and kappa do not shape the layout
  if (make_apex_desc("apex_param_layout", A, dueling, num_atoms, 0.f, 1.f, num_quantiles, 1.f, dist_dueling, noisy, &d)) return -1;
  return apex_layout(d, offsets18, counts18);
}

struct srl_apex_learner {
  srl_apex_config_t cfg;
  float *params, *grads, *m, *v, *target;
  int64_t nparams;
  ApexNetDesc desc;
  ApexNet net[3];                 // the online and target parameters and the gradients (noisy: the mu tensors)
  ApexNet run[2];                 // what the step's online and target forwards run on (apex_forward_net)
  srl_encoder_t *E, *Eq;          // the step's encoder context, and the q-value forwards' own (lanes, events)
  char *saved_s, *saved_n, *enc_scratch;   // encoder blocks: the forward over s (read by the backward), the forwards over s'
  char *saved_q, *scratch_q;      // the q-value forwards' blocks: they may run on another stream than the step
  float *core_s, *core_n, *core_nt, *dcore, *core_q;
  float *q, *y, *dq, *loss, *tail_scratch, *head_part, *coef, *opt_scratch, *zero_reward;
  double* prio;
  int64_t* zero_action;
  int* dstep;
  // the categorical head (cfg.num_atoms = K > 0): logits [B][A K] over s, s' (online, double DQN only) and s' (target), their
  // gradient, the projected targets m [B][K], the cross-entropies [B] and the q-value chunk's logits.  The quantile head
  // (cfg.num_quantiles = N > 0) keeps its quantiles [B][A N], dtheta, the target quantiles [B][N] and the losses [B] in the same rows.
  float *logits_s, *logits_n, *logits_nt, *dlogits, *mproj, *ce, *logits_q;
  // noisy networks: the step's normals and noise and the composed weights ([0] online, [1] target)
  float *normals[2], *noise[2];
  NoisyWeights cw[2];
  uint2 noise_key;
  // the distributional dueling head: the rows the kernels read, composed for the step's online and target forwards ([0], [1]), their
  // gradients ([2]) and the q-value forwards' own
  HeadRows rows[3], rows_q;
  char* arena;
};

// frames per q-value forward: srl_apex_learner_q_values runs n frames in chunks of at most this many
constexpr int APEX_Q_CHUNK = 256;
static int q_chunk(const srl_apex_config_t& c) { return c.B < APEX_Q_CHUNK ? c.B : APEX_Q_CHUNK; }
// the encoder blocks' bytes for the step's B frames and for one q-value chunk: {saved, scratch, saved_q, scratch_q}
static int apex_block_bytes(const srl_apex_config_t& c, int64_t* b4) {
  int rc = srl_encoder_sizes(c.B, c.precision, &b4[0], &b4[1]);
  return rc ? rc : srl_encoder_sizes(q_chunk(c), c.precision, &b4[2], &b4[3]);
}
// the context's device buffers in carving order; rows with a name are what srl_apex_learner_debug_buffer lends
static int apex_rows(srl_apex_learner* L, const int64_t* b4, WsRow* t) {
  const int64_t B = L->cfg.B, A = L->cfg.A, QC = q_chunk(L->cfg);
  int n = 0;
  t[n++] = ws_row<char>(nullptr, b4[0], &L->saved_s);
  t[n++] = ws_row<char>(nullptr, b4[0], &L->saved_n);
  t[n++] = ws_row<char>(nullptr, b4[1], &L->enc_scratch);
  t[n++] = ws_row<char>(nullptr, b4[2], &L->saved_q);
  t[n++] = ws_row<char>(nullptr, b4[3], &L->scratch_q);
  t[n++] = ws_row(nullptr, QC * ENC_CORE, &L->core_q);
  t[n++] = ws_row("core", B * ENC_CORE, &L->core_s);
  t[n++] = ws_row("core_next", L->cfg.double_dqn ? B * ENC_CORE : 0, &L->core_n);
  t[n++] = ws_row("core_next_target", B * ENC_CORE, &L->core_nt);
  t[n++] = ws_row("dcore", B * ENC_CORE, &L->dcore);
  t[n++] = ws_row("q", B, &L->q);
  t[n++] = ws_row("y", B, &L->y);
  t[n++] = ws_row("priorities", B, &L->prio);
  t[n++] = ws_row("loss", 4, &L->loss);
  t[n++] = ws_row("step", 4, &L->dstep);
  t[n++] = ws_row(nullptr, B, &L->dq);
  t[n++] = ws_row(nullptr, 4 + dqn_tail_blocks((int)B), &L->tail_scratch);
  // K: the atoms or quantiles per action (0: the scalar heads, whose rows below are empty); the quantile head's rows have names of their own
  const QHead& h = L->desc.head;
  const bool qr = h.kind == Q_QUANTILE;
  const int64_t K = h.kind == Q_CATEGORICAL ? h.c.K : qr ? h.qr.N : 0, R = A * K;
  t[n++] = ws_row(nullptr, K ? 0 : HEAD_GROUPS * (A + L->cfg.dueling) * 513, &L->head_part);
  t[n++] = ws_row(nullptr, 4, &L->coef);
  t[n++] = ws_row(nullptr, 2048, &L->opt_scratch);
  t[n++] = ws_row(nullptr, QC, &L->zero_reward);     // the reward / action columns of the q-value forwards (the Q head reads h only)
  t[n++] = ws_row(nullptr, QC, &L->zero_action);
  t[n++] = ws_row(qr ? "theta" : "logits", B * R, &L->logits_s);
  t[n++] = ws_row(qr ? "theta_next" : "logits_next", L->cfg.double_dqn ? B * R : 0, &L->logits_n);
  t[n++] = ws_row(qr ? "theta_next_target" : "logits_next_target", B * R, &L->logits_nt);
  t[n++] = ws_row(qr ? "dtheta" : "dlogits", B * R, &L->dlogits);
  t[n++] = ws_row(qr ? "target_quantiles" : "m", B * K, &L->mproj);
  t[n++] = ws_row(qr ? "qr_loss" : "ce", B * (K ? 1 : 0), &L->ce);
  t[n++] = ws_row(nullptr, QC * R, &L->logits_q);
  for (int i = 0; i < 2; ++i) n += noise_rows(L->desc, 1 + i, &L->normals[i], &L->noise[i], &L->cw[i], t + n);
  const int64_t DR = dist_dueling(L->desc) ? R : 0;
  static const char* const rows_names[3][2] = {{"rows_weight_online", "rows_bias_online"}, {"rows_weight_target", "rows_bias_target"},
                                               {"rows_weight_grad", "rows_bias_grad"}};
  for (int i = 0; i < 3; ++i) {
    t[n++] = ws_row(rows_names[i][0], DR * 512, &L->rows[i].W);
    t[n++] = ws_row(rows_names[i][1], DR, &L->rows[i].b);
  }
  t[n++] = ws_row(nullptr, DR * 512, &L->rows_q.W);
  t[n++] = ws_row(nullptr, DR, &L->rows_q.b);
  return n;
}
constexpr int APEX_ROWS = 51;

// -> the network of a valid config
static int check_apex_cfg(const srl_apex_config_t* c, ApexNetDesc* d) {
  REQ(c, "apex_learner: config is NULL");
  REQ(c->B >= 1 && c->B <= MAX_FRAMES, "apex_learner: B=%d must be in [1, %d]", c->B, MAX_FRAMES);
  REQ(c->precision == 0 || c->precision == 1, "apex_learner: precision must be 0 (bf16 operands) or 1 (fp32-accurate split operands)");
  REQ(c->double_dqn == 0 || c->double_dqn == 1, "apex_learner: double_dqn must be 0 or 1");
  REQ(std::isfinite(c->gamma) && c->gamma >= 0.f, "apex_learner: gamma=%g must be finite and >= 0", (double)c->gamma);
  REQ(c->max_grad_norm > 0.f, "apex_learner: max_grad_norm=%g must be > 0 (+inf: no clipping)", (double)c->max_grad_norm);
  REQ(std::isfinite(c->learning_rate) && c->learning_rate > 0.f, "apex_learner: learning_rate=%g must be finite and > 0", (double)c->learning_rate);
  REQ(c->adam_beta1 >= 0.f && c->adam_beta1 < 1.f && c->adam_beta2 >= 0.f && c->adam_beta2 < 1.f, "apex_learner: Adam betas must be in [0, 1)");
  REQ(std::isfinite(c->adam_eps) && c->adam_eps >= 0.f, "apex_learner: adam_eps=%g must be finite and >= 0", (double)c->adam_eps);
  REQ(std::isfinite(c->priority_eps) && c->priority_eps >= 0.f, "apex_learner: priority_eps=%g must be finite and >= 0", (double)c->priority_eps);
  return make_apex_desc("apex_learner", c->A, c->dueling, c->num_atoms, c->v_min, c->v_max, c->num_quantiles, c->kappa, c->dist_dueling,
                        c->noisy, d);
}

extern "C" int srl_apex_learner_create(const srl_apex_config_t* cfg, float* params, float* grads, float* exp_avg, float* exp_avg_sq,
                                       float* target_params, srl_apex_learner_t** out) {
  ApexNetDesc d;
  int rc = check_apex_cfg(cfg, &d);
  if (rc) return rc;
  REQ(params && grads && exp_avg && exp_avg_sq && target_params && out, "apex_learner_create: NULL argument");
  REQ(!misaligned(params, 16) && !misaligned(grads, 16) && !misaligned(exp_avg, 16) && !misaligned(exp_avg_sq, 16) &&
      !misaligned(target_params, 16), "apex_learner_create: flat buffers must be 16-byte aligned");
  const int64_t np = apex_layout(d, nullptr, nullptr);
  const Span s[5] = {{params, np * 4, true, "params"}, {grads, np * 4, true, "grads"}, {exp_avg, np * 4, true, "exp_avg"},
                     {exp_avg_sq, np * 4, true, "exp_avg_sq"}, {target_params, np * 4, true, "target_params"}};
  rc = check_spans(s, 5, "apex_learner_create");
  if (rc) return rc;
  srl_apex_learner* L = new (std::nothrow) srl_apex_learner();
  REQ(L, "out of host memory");
  auto undo = [L](int code) { srl_apex_learner_destroy(L); return code; };
  L->cfg = *cfg; L->params = params; L->grads = grads; L->m = exp_avg; L->v = exp_avg_sq; L->target = target_params; L->nparams = np;
  L->desc = d;
  L->net[0] = bind_apex(d, params); L->net[1] = bind_apex(d, target_params); L->net[2] = bind_apex(d, grads);
  L->noise_key = make_uint2((uint32_t)cfg->noise_seed, (uint32_t)(cfg->noise_seed >> 32));
  rc = srl_encoder_create(cfg->precision, &L->E);
  if (!rc) rc = srl_encoder_create(cfg->precision, &L->Eq);
  if (rc) return undo(rc);
  int64_t b4[4];
  rc = apex_block_bytes(*cfg, b4);
  if (rc) return undo(rc);
  WsRow t[APEX_ROWS];
  const int n = apex_rows(L, b4, t);
  const int64_t total = rows_bytes(t, n, false);
  cudaError_t e = cudaMalloc(&L->arena, total);
  if (e != cudaSuccess) return undo(cuda_fail(e, "apex_learner_create: cudaMalloc workspace"));
  e = cudaMemset(L->arena, 0, total);        // the tail's ticket, the step count and the zero reward / action columns
  if (e == cudaSuccess) e = cudaMemset(grads, 0, np * 4);      // the padding between the segments enters the gradient norm
  if (e != cudaSuccess) return undo(cuda_fail(e, "apex_learner_create: cudaMemset"));
  carve_rows(t, n, false, L->arena);
  for (int i = 0; i < 2; ++i) L->run[i] = apex_forward_net(d, L->net[i], L->cw[i]);
  *out = L;
  return 0;
}

extern "C" int srl_apex_learner_destroy(srl_apex_learner_t* L) {
  if (!L) return 0;
  srl_encoder_destroy(L->E);
  srl_encoder_destroy(L->Eq);
  cudaFree(L->arena);
  delete L;
  return 0;
}

extern "C" int srl_apex_learner_step(srl_apex_learner_t* L, const uint8_t* obs, const int64_t* action, const float* reward, const uint8_t* next_obs,
                                     const uint8_t* done, const float* weights, const int64_t* idxs, srl_per_t* per, float* stats_out, void* stream) {
  REQ(L && obs && action && reward && next_obs && done, "apex_learner_step: NULL pointer");
  REQ(!idxs == !per, "apex_learner_step: idxs and per go together (both NULL or both set)");
  const srl_apex_config_t& c = L->cfg;
  const int B = c.B;
  const cudaStream_t st = (cudaStream_t)stream;
  if (L->desc.noisy) {      // update k's noise (k = the device step count) for both networks, and their composed weights
    CU(launch_noisy_draw(L->noise_key, L->dstep, nullptr, 2, noise_count(L->desc), L->normals, L->noise, st), "noisy_draw");
    const float* noise[2] = {L->noise[0], L->noise[1]};
    const NoisyTensors nz[2] = {L->net[0].nz, L->net[1].nz};
    CU(launch_noisy_compose(nz, L->cw, noise, 2, L->desc, st), "noisy_compose");
  }
  // the heads the tail reads and the gradients q_wgrad writes: the distributional dueling head's composed rows (the target's from
  // target_params as they are now, so an update of them between replays is seen) and their gradients
  QHead head_on = L->run[0].q, head_tg = L->run[1].q;
  QHeadGrad head_g = L->net[2].g;
  const bool dd = dist_dueling(L->desc);
  if (dd) {
    const QHead p[2] = {head_on, head_tg};
    CU(launch_dist_dueling_compose(p, L->rows, 2, L->desc.vrows, st), "dist_dueling_compose");
    head_on = on_rows(head_on, L->rows[0]);
    head_tg = on_rows(head_tg, L->rows[1]);
    head_g = QHeadGrad{L->rows[2].W, L->rows[2].b, nullptr};
  }
  // the three forwards (the encoder checks obs / next_obs and the blocks); the target forward runs last so that its rows are the
  // ones left in saved_n
  const ApexNet &on = L->run[0], &tg = L->run[1];
  int rc = srl_encoder_forward(L->E, obs, reward, action, B, 1, on.w8, L->saved_s, L->enc_scratch, L->core_s, stream);
  if (!rc && c.double_dqn) rc = srl_encoder_forward(L->E, next_obs, reward, action, B, 1, on.w8, L->saved_n, L->enc_scratch, L->core_n, stream);
  if (!rc) rc = srl_encoder_forward(L->E, next_obs, reward, action, B, 1, tg.w8, L->saved_n, L->enc_scratch, L->core_nt, stream);
  if (rc) return rc;
  const QTail t = {L->core_s, c.double_dqn ? L->core_n : nullptr, L->core_nt, action, reward, done, weights, B, c.gamma, c.priority_eps,
                   L->q, L->y, L->dcore, L->loss, L->tail_scratch, L->prio, L->dq, L->head_part, L->logits_s, L->logits_n, L->logits_nt,
                   L->mproj, L->ce, L->dlogits};
  CU(launch_q_tail(head_on, head_tg, t, st), "q_tail");
  CU(launch_q_wgrad(head_on, head_g, t, st), "q_wgrad");
  if (dd) CU(launch_dist_dueling_grad(L->rows[2], L->net[2].g, c.A, L->desc.vrows, st), "dist_dueling_grad");
  // the gradients of the composed weights land in the mu segments
  rc = srl_encoder_backward(L->E, L->dcore, B, 1, L->saved_s, L->enc_scratch, L->net[2].w8, stream);
  if (rc) return rc;
  if (L->desc.noisy) CU(launch_noisy_sigma_grad(L->net[2].nz, L->noise[0], L->desc, st), "noisy_sigma_grad");
  const OptStep o = {1, L->params, L->grads, L->m, L->v, L->nparams, c.max_grad_norm, L->coef, L->opt_scratch, c.learning_rate,
                     c.adam_beta1, c.adam_beta2, c.adam_eps, 0, L->dstep, OptExtra{}};
  CU(launch_clip_optim(o, st), "clip+adam");
  if (per) {
    rc = srl_per_update_priorities(per, idxs, L->prio, B, stream);       // <= 1024 pairs per launch, in order: the last idx wins
    if (rc) return rc;
  }
  if (stats_out) {
    CU(cudaMemcpyAsync(stats_out, L->loss, sizeof(float), cudaMemcpyDeviceToDevice, st), "copy loss");
    CU(cudaMemcpyAsync(stats_out + 1, L->coef, 2 * sizeof(float), cudaMemcpyDeviceToDevice, st), "copy coef");
  }
  return 0;
}

extern "C" int srl_apex_learner_update_target(srl_apex_learner_t* L, float tau, void* stream) {
  REQ(L, "apex_learner_update_target: learner is NULL");
  REQ(tau >= 0.f && tau <= 1.f, "apex_learner_update_target: tau=%g must be in [0, 1]", (double)tau);
  // torch evaluates (1.0 - tau) in double and rounds it once to the tensor's float
  CU(launch_apex_soft_update(L->params, L->target, L->nparams, tau, (float)(1.0 - (double)tau), (cudaStream_t)stream), "apex_soft_update");
  return 0;
}

extern "C" int srl_apex_learner_set_step(srl_apex_learner_t* L, int64_t step, void* stream) {
  REQ(L && step >= 0 && step < (int64_t(1) << 31), "apex_learner_set_step: bad argument");
  const int v = (int)step;
  CU(cudaMemcpyAsync(L->dstep, &v, sizeof(int), cudaMemcpyHostToDevice, (cudaStream_t)stream), "apex_learner_set_step");
  CU(cudaStreamSynchronize((cudaStream_t)stream), "apex_learner_set_step");      // `v` is a stack variable
  return 0;
}

extern "C" int srl_apex_learner_q_values(srl_apex_learner_t* L, const uint8_t* obs, int n, float* q_out, void* stream) {
  REQ(L && obs && q_out, "apex_learner_q_values: NULL pointer");
  REQ(n >= 1, "apex_learner_q_values: n=%d must be >= 1", n);
  const int QC = q_chunk(L->cfg), A = L->cfg.A;
  const Span s[2] = {{obs, (int64_t)n * 28224, false, "obs"}, {q_out, (int64_t)n * A * 4, true, "q_out"}};
  int rc = check_spans(s, 2, "apex_learner_q_values");
  if (rc) return rc;
  QHead head = L->net[0].q;
  if (dist_dueling(L->desc)) {                // composed into the q-value forwards' own rows: the step's may be in use on another stream
    CU(launch_dist_dueling_compose(&head, &L->rows_q, 1, L->desc.vrows, (cudaStream_t)stream), "dist_dueling_compose");
    head = on_rows(head, L->rows_q);
  }
  for (int f0 = 0; f0 < n; f0 += QC) {       // chunks through the q-value forwards' own context and blocks
    const int f = n - f0 < QC ? n - f0 : QC;
    rc = srl_encoder_forward(L->Eq, obs + (size_t)f0 * 28224, L->zero_reward, L->zero_action, f, 1, L->net[0].w8, L->saved_q, L->scratch_q,
                             L->core_q, stream);
    if (rc) return rc;
    CU(launch_q_values(head, L->core_q, f, L->logits_q, q_out + (size_t)f0 * A, (cudaStream_t)stream), "q_values");
  }
  return 0;
}

extern "C" int srl_apex_learner_debug_buffer(srl_apex_learner_t* L, const char* name, void** ptr, int64_t* count) {
  REQ(L && name && ptr && count, "apex_learner_debug_buffer: NULL argument");
  {   // the activations the forward over s saved for its backward (bf16; the high parts in the fp32-accurate mode)
    EncoderBuffers b = {};
    WsRow e[ENC_ROWS];
    encoder_rows(b, L->cfg.B, L->cfg.B, e);
    carve_rows(e, ENC_SAVED_ROWS, L->cfg.precision == 1, L->saved_s);
    for (int i = 0; i < ENC_SAVED_ROWS; ++i)
      if (strcmp(name, "a1") == 0 || strcmp(name, "a2") == 0 || strcmp(name, "a3") == 0)
        if (strcmp(e[i].name, name) == 0) { *ptr = *e[i].hi; *count = e[i].count; return 0; }
  }
  int64_t b4[4];
  int rc = apex_block_bytes(L->cfg, b4);
  if (rc) return rc;
  srl_apex_learner shadow = *L;        // the table's rows re-derived on a copy: the same sizes give the same addresses
  WsRow t[APEX_ROWS];
  const int n = apex_rows(&shadow, b4, t);
  carve_rows(t, n, false, L->arena);
  for (int i = 0; i < n; ++i)
    if (t[i].name && strcmp(t[i].name, name) == 0 && t[i].count > 0) { *ptr = *t[i].hi; *count = t[i].count; return 0; }
  return fail(SRL_EINVAL, "apex_learner_debug_buffer: unknown buffer '%s'", name);
}
