// extern "C" entry points (include/scalerl_b200.h).  Argument checking + the learner context that owns
// the activation workspaces and sequences the kernels of one learner step on the caller's stream.
#include <stdio.h>
#include <string.h>
#include <stdarg.h>
#include <cmath>
#include <new>

#include "../../include/scalerl_b200.h"
#include "kernels.h"

using namespace srl;

static thread_local char g_err[512] = "";

static int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
static int cuda_fail(cudaError_t e, const char* what) {
  snprintf(g_err, sizeof(g_err), "%s: %s (%s)", what, cudaGetErrorName(e), cudaGetErrorString(e));
  return (int)e;
}
#define CU(x, what) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return cuda_fail(e_, what); } while (0)
#define REQ(c, ...) do { if (!(c)) return fail(SRL_EINVAL, __VA_ARGS__); } while (0)

extern "C" const char* srl_last_error(void) { return g_err; }
extern "C" int srl_version(void) { return 100; }

// ------------------------------------------------------------------------------------------------
// stand-alone ops
// ------------------------------------------------------------------------------------------------
extern "C" int srl_vtrace_from_importance_weights(const float* log_rhos, const float* discounts, const float* rewards,
                                                  const float* values, const float* bootstrap_value, int T, int B,
                                                  float clip_rho, float clip_pg, float* vs, float* pg, int variant, void* stream) {
  REQ(T >= 0 && B >= 0, "vtrace: negative shape T=%d B=%d", T, B);
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
  if (T == 0 || B == 0) return 0;
  REQ(bl && tl && actions && discounts && rewards && values && bootstrap_value && vs && pg, "vtrace_from_logits: NULL pointer");
  CU(launch_vtrace_logits(bl, tl, actions, discounts, rewards, values, bootstrap_value, T, B, A, clip_rho, clip_pg, vs, pg, log_rhos,
                          balp, talp, (cudaStream_t)stream), "vtrace_from_logits");
  return 0;
}

extern "C" int srl_impala_loss_and_head_grads(const float* bl, const float* tl, const float* baseline, const int64_t* action,
                                              const float* reward, const uint8_t* done, int T, int B, int A, float discounting,
                                              int reward_clip_abs_one, float clip_rho, float clip_pg, float baseline_cost,
                                              float entropy_cost, float* vs, float* pg, float* dlogits, float* dbaseline, float* losses,
                                              float* scratch, void* stream) {
  REQ(T >= 1 && B >= 1 && A >= 1, "impala_loss: bad shape T=%d B=%d A=%d", T, B, A);
  REQ(bl && tl && baseline && action && reward && done && dlogits && dbaseline && losses && scratch, "impala_loss: NULL pointer");
  CU(launch_impala_tail(bl, tl, baseline, action, reward, done, T, B, A, discounting, reward_clip_abs_one, clip_rho, clip_pg,
                        baseline_cost, entropy_cost, vs, pg, dlogits, dbaseline, losses, scratch, (cudaStream_t)stream), "impala_tail");
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
  REQ((slot_bytes & 15) == 0 && (offsets6_host[0] & 15) == 0 && (reinterpret_cast<uintptr_t>(staging) & 15) == 0 &&
      (reinterpret_cast<uintptr_t>(obs) & 15) == 0, "unpack_slots: obs record and buffers must be 16-byte aligned");
  CU(launch_unpack_slots(staging, slot_bytes, offsets6_host, T, B, A, obs, reward, done, action, policy_logits, episode_return,
                         (cudaStream_t)stream), "unpack_slots");
  return 0;
}

extern "C" int srl_grad_norm_clip_coef(const float* grads, int64_t n, float max_norm, float* coef, float* scratch, void* stream) {
  REQ(grads && coef && scratch && n >= 0, "grad_norm: bad argument");
  REQ((reinterpret_cast<uintptr_t>(grads) & 15) == 0, "grad_norm: grads must be 16-byte aligned");
  CU(launch_grad_norm(grads, n, max_norm, coef, scratch, (cudaStream_t)stream), "grad_norm");
  return 0;
}
extern "C" int srl_rmsprop_step(float* params, const float* grads, float* square_avg, int64_t n, const float* coef, float lr, float alpha,
                                float eps, void* stream) {
  REQ(params && grads && square_avg && n >= 0, "rmsprop: bad argument");
  REQ(((reinterpret_cast<uintptr_t>(params) | reinterpret_cast<uintptr_t>(grads) | reinterpret_cast<uintptr_t>(square_avg)) & 15) == 0,
      "rmsprop: buffers must be 16-byte aligned");
  CU(launch_rmsprop(params, grads, square_avg, n, coef, lr, alpha, eps, (cudaStream_t)stream), "rmsprop");
  return 0;
}
extern "C" int srl_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n, const float* coef, float lr,
                             float beta1, float beta2, float eps, int step, void* stream) {
  REQ(params && grads && exp_avg && exp_avg_sq && n >= 0 && step >= 1, "adam: bad argument");
  CU(launch_adam(params, grads, exp_avg, exp_avg_sq, n, coef, lr, beta1, beta2, eps, step, nullptr, (cudaStream_t)stream), "adam");
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
  SideStream ss;                  // wgrad side stream + fork/join events
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
  Profiler pf;                    // per-kernel event bracketing (off by default)
  cudaEvent_t events[2 * PS_COUNT];
};

static const char* kSlotNames[PS_COUNT] = {"obs_s2d", "conv1_fwd", "conv2_fwd", "conv3_fwd", "fc_fwd", "head_fwd", "vtrace_loss_tail",
                                           "zero_grads", "head_bwd", "fc_wgrad", "fc_dgrad", "conv3_wgrad", "conv3_dgrad", "conv2_wgrad",
                                           "conv2_dgrad", "conv1_wgrad", "conv_wgrad_finalize", "grad_norm", "optimizer", "pack_weights", "enc_fused_fwd"};

static int check_cfg(const srl_config_t* c) {
  REQ(c, "config is NULL");
  REQ(c->T >= 1 && c->B >= 1, "config: T=%d B=%d must be >= 1", c->T, c->B);
  REQ(c->A >= 1 && c->A <= 31, "config: A=%d must be in [1,31] (one warp lane per action plus one for the baseline)", c->A);
  REQ((int64_t)(c->T + 1) * c->B <= 65536, "config: (T+1)*B=%lld frames per GPU exceeds 65536", (long long)(c->T + 1) * c->B);
  REQ(c->optimizer == 0 || c->optimizer == 1, "config: optimizer must be 0 (rmsprop) or 1 (adam)");
  REQ(c->use_lstm == 0 || c->use_lstm == 1, "config: use_lstm must be 0 or 1");
  REQ(c->precision == 0 || c->precision == 1, "config: precision must be 0 (bf16 operands) or 1 (fp32-accurate split operands)");
  REQ(!(c->precision == 1 && c->use_lstm), "config: the fp32-accurate operand mode covers the non-LSTM learner only");
  return 0;
}

// The device workspace of a learner context, one row per tensor in carving order.  Every tensor is 256-byte aligned and zero-filled
// at creation (the zeros of the da*g grids are the padding of the transposed convolutions).  In the fp32-accurate operand mode a row
// with a low twin is followed by the twin, which srl_learner_debug_buffer calls "<name>_lo".  Rows without a name are internal.
struct WsRow {
  const char* name;
  int elem;                       // bytes per element
  int64_t count;                  // elements
  void** hi;                      // receives the tensor's address (null: zeros only)
  void** lo;                      // receives the low twin's address (null: no twin)
};
template <class T>
static WsRow ws_row(const char* name, int64_t count, T** hi, T** lo = nullptr) {
  return {name, (int)sizeof(T), count, reinterpret_cast<void**>(hi), reinterpret_cast<void**>(lo)};
}
constexpr int WS_MAX_ROWS = 32;
static int workspace_table(srl_learner* L, WsRow* t) {
  const srl_config_t& c = L->cfg;
  const int64_t NF = (int64_t)(c.T + 1) * c.B, NB = (int64_t)c.T * c.B, A = c.A, H = 513 + A;
  EncoderBuffers& b = L->buf;
  OperandTensors &hi = b.hi, &lo = b.lo;
  int n = 0;
  t[n++] = ws_row("xs", NF * 441 * 64, &b.xs);
  t[n++] = ws_row(nullptr, FC_SPLITS * NF * 512, &b.hpart);
  t[n++] = ws_row("a1", NF * 400 * 32, &hi.a1, &lo.a1);
  t[n++] = ws_row("a2", NF * 81 * 64, &hi.a2, &lo.a2);
  t[n++] = ws_row("a3", NF * 49 * 64, &hi.a3, &lo.a3);
  t[n++] = ws_row("h", NF * 512, &b.h);
  t[n++] = ws_row("dh", NB * 512, &hi.dh, &lo.dh);
  t[n++] = ws_row("da3", NB * 81 * 64, &hi.da3, &lo.da3);      // da3g (9x9 grid)
  t[n++] = ws_row("da2", NB * 100 * 64, &hi.da2, &lo.da2);     // da2g (10x10 grid)
  t[n++] = ws_row("da1", NB * 441 * 32, &hi.da1, &lo.da1);     // da1g (21x21 grid, 32 channels)
  t[n++] = ws_row("wpack", WPack::TOTAL, &hi.wpack, &lo.wpack);
  t[n++] = ws_row("logits", NF * A, &L->logits);
  t[n++] = ws_row("baseline", NF, &L->baseline);
  t[n++] = ws_row("dlogits", NB * A, &L->dlogits);
  t[n++] = ws_row("dbaseline", NB, &L->dbaseline);
  t[n++] = ws_row(nullptr, 4096, &L->scratch);
  t[n++] = ws_row(nullptr, 4, &L->coef);
  t[n++] = ws_row(nullptr, 4, &L->dstep);
  t[n++] = ws_row(nullptr, WS_TOTAL, &b.wgrad_ws);
  t[n++] = ws_row(nullptr, WSP_TOTAL, &b.wgrad_part);
  t[n++] = ws_row(nullptr, HEAD_GROUPS * (A + 1) * (514 + A), &L->head_part);
  t[n++] = ws_row("a3t", NF * 49 * 64, &b.a3t);
  if (c.use_lstm) {
    t[n++] = ws_row(nullptr, NF * H, &L->core);
    t[n++] = ws_row(nullptr, NF * H, &L->lstm_out);
    t[n++] = ws_row(nullptr, NB * H, &L->dout);
    t[n++] = ws_row(nullptr, NB * H, &L->dcore);
    t[n++] = ws_row<char>(nullptr, 1024, nullptr);      // 1 KiB of zeros behind dcore
  }
  return n;
}
static int64_t ws_bytes(const WsRow& r) { return ((int64_t)r.elem * r.count + 255) & ~int64_t(255); }

static int pack_priority(int least, int greatest);
extern "C" int srl_learner_create(const srl_config_t* cfg, float* params, float* grads, float* opt0, float* opt1, srl_learner_t** out) {
  int rc = check_cfg(cfg);
  if (rc) return rc;
  REQ(params && grads && opt0 && out, "learner_create: NULL buffer");
  REQ(cfg->optimizer == 0 || opt1, "learner_create: Adam needs opt_state1");
  REQ(((reinterpret_cast<uintptr_t>(params) | reinterpret_cast<uintptr_t>(grads) | reinterpret_cast<uintptr_t>(opt0) |
        reinterpret_cast<uintptr_t>(opt1)) & 15) == 0, "learner_create: flat buffers must be 16-byte aligned");
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
  int64_t total = 0;
  for (int i = 0; i < n; ++i) total += ws_bytes(t[i]) * (split && t[i].lo ? 2 : 1);
  cudaError_t e = cudaMalloc(&L->arena, total);
  if (e != cudaSuccess) return undo(cuda_fail(e, "learner_create: cudaMalloc workspace"));
  e = cudaMemset(L->arena, 0, total);
  if (e != cudaSuccess) return undo(cuda_fail(e, "learner_create: cudaMemset"));
  L->arena_bytes = total;
  char* q = L->arena;
  for (int i = 0; i < n; ++i) {
    if (t[i].hi) *t[i].hi = q;
    q += ws_bytes(t[i]);
    if (split && t[i].lo) { *t[i].lo = q; q += ws_bytes(t[i]); }
  }
  L->buf.NF = (int)NF;
  if (cudaStreamCreateWithFlags(&L->ss.side, cudaStreamNonBlocking) != cudaSuccess ||
      cudaStreamCreateWithFlags(&L->ss.side2, cudaStreamNonBlocking) != cudaSuccess ||
      cudaStreamCreateWithFlags(&L->ss.side3, cudaStreamNonBlocking) != cudaSuccess) L->ss.side = nullptr;
  {
    int lo = 0, hi = 0;       // (numerically lowest = greatest priority)
    if (L->ss.side && (cudaDeviceGetStreamPriorityRange(&lo, &hi) != cudaSuccess ||
                       cudaStreamCreateWithPriority(&L->ss.pack, cudaStreamNonBlocking, pack_priority(lo, hi)) != cudaSuccess)) L->ss.side = nullptr;
  }
  for (int e2 = 0; e2 < 12 && L->ss.side; ++e2)
    if (cudaEventCreateWithFlags(&L->ss.ev[e2], cudaEventDisableTiming) != cudaSuccess) { L->ss.side = nullptr; }
  cudaGetLastError();
  const char* why = nullptr;
  if (build_tma_maps(L->buf, (int)NF, (int)NB, &L->maps, &why) != cudaSuccess)
    return undo(fail(SRL_ESTATE, "learner_create: building TMA tensor map '%s' failed (driver without cuTensorMapEncodeTiled?)", why ? why : "?"));
  if (cfg->use_lstm) {
    const int H = 513 + cfg->A;
    const float* wp[8]; float* gp[8];
    for (int i = 0; i < 8; ++i) { wp[i] = params + off[12 + i]; gp[i] = grads + off[12 + i]; }
    L->lstm_off0 = off[12]; L->lstm_len = L->nparams - off[12];
    why = srl_lstm_last_error();
    if (srl_lstm_create(cfg->T + 1, cfg->B, H, wp, gp, &L->lstm) != 0 || lstm_step_create(cfg->B, H, wp, &L->lstm_step, &why) != cudaSuccess)
      return undo(fail(SRL_ESTATE, "learner_create: LSTM core allocation failed: %s", why));
  }
  *out = L;
  return 0;
}

extern "C" int srl_learner_destroy(srl_learner_t* L) {
  if (!L) return 0;
  for (int i = 0; i < 2 * PS_COUNT; ++i) if (L->events[i]) cudaEventDestroy(L->events[i]);
  for (int i = 0; i < 12; ++i) if (L->ss.ev[i]) cudaEventDestroy(L->ss.ev[i]);
  if (L->ss.side) cudaStreamDestroy(L->ss.side);
  if (L->ss.side2) cudaStreamDestroy(L->ss.side2);
  if (L->ss.side3) cudaStreamDestroy(L->ss.side3);
  if (L->ss.pack) cudaStreamDestroy(L->ss.pack);
  if (L->lstm) srl_lstm_destroy(L->lstm);
  lstm_step_destroy(L->lstm_step);
  cudaFree(L->arena);
  delete L;
  return 0;
}
extern "C" int srl_debug_kernel_timeline(void* buffer) {
#ifdef SRL_KSTAMP
  kstamp_set_encoder((unsigned long long*)buffer); kstamp_set_vtrace((unsigned long long*)buffer); kstamp_set_heads((unsigned long long*)buffer);
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
  REQ((reinterpret_cast<uintptr_t>(momentum_buf) & 15) == 0, "set_momentum: the momentum buffer must be 16-byte aligned");
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
  CU(launch_pack_weights(L->P, L->buf.hi.wpack, (cudaStream_t)stream, L->buf.lo.wpack), "pack_weights");
  // the actor step's [W_ih | W_hh] copy: packed here, once per weight version, and never by the learner's own forward
  if (L->lstm_step) CU(lstm_step_pack(L->lstm_step, (cudaStream_t)stream), "lstm_step_pack");
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

// the re-pack stream sits one level BELOW the greatest priority (which the learner's capture stream uses for the main chain) and above the wgrad
// streams (default = least): its short blocks fill the slots the frame conversion leaves free without delaying it
static int pack_priority(int least, int greatest) {
  return greatest + 1 > least ? least : greatest + 1;
}

static int encode_impl(srl_learner* L, const uint8_t* obs, int frames, cudaStream_t st, bool zero_small_grads = false) {
  L->pf.st = st;
  pdl_set_active(!L->pf.on);
  // The bf16 operand copies are re-derived from the fp32 master weights at the START of every forward (not at the end
  // of the optimizer step): the pack kernel runs on the side stream underneath the frame conversion.
  // Without side streams, or with per-kernel profiling on, both run on `st` (the profiler brackets are no-ops otherwise).
  const bool fork = L->ss.side && !L->pf.on;
  cudaStream_t pack_st = fork ? L->ss.pack : st;
  if (fork) {
    CU(cudaEventRecord(L->ss.ev[5], st), "fork pack");
    CU(cudaStreamWaitEvent(pack_st, L->ss.ev[5], 0), "fork pack");
  }
  if (zero_small_grads) {     // the accumulated gradient segments (everything before fc.weight) are cleared under the frame conversion
    L->pf.b(PS_ZERO_GRADS);
    CU(cudaMemsetAsync(L->grads, 0, L->small_len * sizeof(float), pack_st), "zero small grads");
    L->pf.e(PS_ZERO_GRADS);
  }
  L->pf.b(PS_PACK);
  CU(launch_pack_weights(L->P, L->buf.hi.wpack, pack_st, L->buf.lo.wpack, true), "pack_weights");
  L->pf.e(PS_PACK);
  cudaEvent_t packed = nullptr;
  if (fork) {
    CU(cudaEventRecord(L->ss.ev[6], pack_st), "join pack");
    packed = L->ss.ev[6];
  }
  CU(encoder_forward(obs, frames, L->P, L->buf, L->maps, L->cfg.precision, st, L->pf, packed, L->fused_front), "encoder_forward");
  // learner step (bf16 mode): a3 -> fc.weight column order for the fc weight-gradient GEMM, on the wgrad side stream right after the fc forward,
  // i.e. under the column kernel (32 CTAs, the GPU is otherwise idle) instead of in the crowded backward phase
  L->buf.a3t_ready = false;
  if (zero_small_grads && fork && L->cfg.precision == 0 && L->buf.a3t && !L->cfg.use_lstm) {
    CU(cudaEventRecord(L->ss.ev[10], st), "fork a3 transpose");
    CU(cudaStreamWaitEvent(L->ss.side, L->ss.ev[10], 0), "fork a3 transpose");
    CU(launch_a3_transpose(L->buf.hi.a3, L->buf.a3t, L->cfg.T * L->cfg.B, L->ss.side), "a3_transpose");
    L->buf.a3t_ready = true;
  }
  return 0;
}

static int forward_impl(srl_learner* L, const uint8_t* obs, const float* reward, const int64_t* action, int frames, float* logits,
                        float* baseline, cudaStream_t st, bool zero_small_grads = false) {
  REQ(!L->cfg.use_lstm, "this learner was created with use_lstm=1: call the *_lstm entry points");
  int rc = encode_impl(L, obs, frames, st, zero_small_grads);
  if (rc) return rc;
  L->pf.b(PS_HEAD_FWD);
  CU(launch_head_fwd(L->buf.hpart, FC_SPLITS, L->P.bf, L->buf.h, reward, action, L->P.wp, L->P.bp, L->P.wb, L->P.bb, frames, L->cfg.A,
                     logits, baseline, st), "head_fwd");
  L->pf.e(PS_HEAD_FWD);
  return 0;
}

extern "C" int srl_learner_forward(srl_learner_t* L, const uint8_t* obs, const float* reward, const int64_t* action, int rows,
                                   float* policy_logits, float* baseline, void* stream) {
  REQ(L && obs && reward && action && policy_logits && baseline, "learner_forward: NULL pointer");
  REQ(rows >= 1 && rows <= L->cfg.T + 1, "learner_forward: rows=%d must be in [1, T+1=%d]", rows, L->cfg.T + 1);
  REQ((reinterpret_cast<uintptr_t>(obs) & 3) == 0, "learner_forward: obs must be 4-byte aligned");
  return forward_impl(L, obs, reward, action, rows * L->cfg.B, policy_logits, baseline, (cudaStream_t)stream);
}

static int fb_begin(srl_learner* L, const uint8_t* obs, const float* reward, const uint8_t* done, const int64_t* action,
                    const float* behavior_logits, float* losses, float* vs, float* pg_advantages, cudaStream_t st, int phase) {
  const srl_config_t& c = L->cfg;
  const int NF = (c.T + 1) * c.B, NB = c.T * c.B;
  // heads + V-trace/losses + dh: one fused column kernel when its shared-memory footprint fits, else three kernels
  const bool fused = L->column_fusion && column_step_supported(c.T, c.B, c.A);
  int rc;
  if (fused) {
    REQ(!L->cfg.use_lstm, "this learner was created with use_lstm=1: call the *_lstm entry points");
    rc = encode_impl(L, obs, NF, st, true);
    if (rc) return rc;
    L->pf.b(PS_TAIL);
    CU(launch_column_step(L->buf.hpart, FC_SPLITS, L->P.bf, L->buf.h, reward, action, done, behavior_logits, L->P.wp, L->P.bp, L->P.wb,
                          L->P.bb, c.T, c.B, c.A, c.discounting, c.reward_clip_abs_one, c.clip_rho_threshold, c.clip_pg_rho_threshold,
                          c.baseline_cost, c.entropy_cost, L->logits, L->baseline, vs, pg_advantages, L->dlogits, L->dbaseline, L->buf.hi.dh,
                          losses, L->scratch, st, L->buf.lo.dh), "column_step");
    L->pf.e(PS_TAIL);
  } else {
    rc = forward_impl(L, obs, reward, action, NF, L->logits, L->baseline, st, true);
    if (rc) return rc;
    L->pf.b(PS_TAIL);
    CU(launch_impala_tail(behavior_logits, L->logits, L->baseline, action, reward, done, c.T, c.B, c.A, c.discounting,
                          c.reward_clip_abs_one, c.clip_rho_threshold, c.clip_pg_rho_threshold, c.baseline_cost, c.entropy_cost, vs,
                          pg_advantages, L->dlogits, L->dbaseline, losses, L->scratch, st), "impala_tail");
    L->pf.e(PS_TAIL);
  }
  L->pf.b(PS_HEAD_BWD);
  {
    const bool fork = L->ss.side != nullptr && !L->pf.on;
    cudaStream_t sw = fork ? L->ss.side : st;
    if (fork) { CU(cudaEventRecord(L->ss.ev[8], st), "fork head wgrad"); CU(cudaStreamWaitEvent(sw, L->ss.ev[8], 0), "fork head wgrad"); }
    CU(launch_head_bwd(L->dlogits, L->dbaseline, L->buf.h, reward, action, L->P.wp, L->P.wb, NB, c.A, L->buf.hi.dh, L->G.wp, L->G.bp, L->G.wb,
                       L->G.bb, L->head_part, st, sw, !fused, L->buf.lo.dh), "head_bwd");      // side stream `side` is joined by encoder_backward (after the fc wgrad)
  }
  L->pf.e(PS_HEAD_BWD);
  CU(encoder_backward(NB, L->buf, L->G, L->maps, c.precision, st, L->pf, L->ss, phase), "encoder_backward");
  L->have_fwd = true;
  return 0;
}

extern "C" int srl_learner_forward_backward(srl_learner_t* L, const uint8_t* obs, const float* reward, const uint8_t* done,
                                            const int64_t* action, const float* behavior_logits, float* losses, float* vs,
                                            float* pg_advantages, void* stream) {
  REQ(L && obs && reward && done && action && behavior_logits && losses, "learner_forward_backward: NULL pointer");
  REQ((reinterpret_cast<uintptr_t>(obs) & 3) == 0, "learner_forward_backward: obs must be 4-byte aligned");
  return fb_begin(L, obs, reward, done, action, behavior_logits, losses, vs, pg_advantages, (cudaStream_t)stream, 2);
}

extern "C" int srl_learner_forward_backward_begin(srl_learner_t* L, const uint8_t* obs, const float* reward, const uint8_t* done,
                                                  const int64_t* action, const float* behavior_logits, float* losses, float* vs,
                                                  float* pg_advantages, void* stream) {
  REQ(L && obs && reward && done && action && behavior_logits && losses, "learner_forward_backward_begin: NULL pointer");
  REQ((reinterpret_cast<uintptr_t>(obs) & 3) == 0, "learner_forward_backward_begin: obs must be 4-byte aligned");
  return fb_begin(L, obs, reward, done, action, behavior_logits, losses, vs, pg_advantages, (cudaStream_t)stream, 0);
}

extern "C" int srl_learner_backward_finish(srl_learner_t* L, const uint8_t* obs, void* stream) {
  REQ(L && obs, "learner_backward_finish: NULL pointer");
  REQ(L->have_fwd, "learner_backward_finish: call srl_learner_forward_backward_begin first");
  const srl_config_t& c = L->cfg;
  L->pf.st = (cudaStream_t)stream;
  pdl_set_active(!L->pf.on);
  CU(encoder_backward(c.T * c.B, L->buf, L->G, L->maps, c.precision, (cudaStream_t)stream, L->pf, L->ss, 1), "encoder_backward");
  return 0;
}

static int forward_lstm_impl(srl_learner* L, const uint8_t* obs, const float* reward, const uint8_t* done, const int64_t* action,
                             const float* h0, const float* c0, float* logits, float* baseline, float* hT, float* cT, cudaStream_t st) {
  REQ(L->cfg.use_lstm && L->lstm, "this learner was created with use_lstm=0");
  const srl_config_t& c = L->cfg;
  const int NF = (c.T + 1) * c.B;
  int rc = encode_impl(L, obs, NF, st);
  if (rc) return rc;
  CU(launch_core_build(L->buf.hpart, FC_SPLITS, L->P.bf, reward, action, NF, c.A, L->buf.h, L->core, st), "core_build");
  rc = srl_lstm_forward(L->lstm, L->core, done, h0, c0, L->lstm_out, hT, cT, st);
  if (rc) return fail(rc, "lstm_forward: %s", srl_lstm_last_error());
  CU(launch_head_dense_fwd(L->lstm_out, L->P.wp, L->P.bp, L->P.wb, L->P.bb, NF, c.A, logits, baseline, st), "head_dense_fwd");
  return 0;
}

extern "C" int srl_learner_forward_lstm(srl_learner_t* L, const uint8_t* obs, const float* reward, const uint8_t* done, const int64_t* action,
                                        const float* h0, const float* c0, float* policy_logits, float* baseline, float* hT, float* cT,
                                        void* stream) {
  REQ(L && obs && reward && done && action && h0 && c0 && policy_logits && baseline, "learner_forward_lstm: NULL pointer");
  return forward_lstm_impl(L, obs, reward, done, action, h0, c0, policy_logits, baseline, hT, cT, (cudaStream_t)stream);
}

static bool overlaps(const void* a, const void* b, int64_t bytes) {
  const uintptr_t x = reinterpret_cast<uintptr_t>(a), y = reinterpret_cast<uintptr_t>(b);
  return x < y + (uintptr_t)bytes && y < x + (uintptr_t)bytes;
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
  REQ(!overlaps(h_out, h_in, sb) && !overlaps(h_out, c_in, sb) && !overlaps(c_out, h_in, sb) && !overlaps(c_out, c_in, sb) &&
      !overlaps(h_out, c_out, sb), "learner_forward_lstm_step: h_out / c_out must not alias h_in, c_in or each other");
  REQ((reinterpret_cast<uintptr_t>(obs) & 3) == 0, "learner_forward_lstm_step: obs must be 4-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  int rc = encode_impl(L, obs, B, st);
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
  cudaStream_t st = (cudaStream_t)stream;
  const srl_config_t& c = L->cfg;
  const int NB = c.T * c.B;
  int rc = forward_lstm_impl(L, obs, reward, done, action, h0, c0, L->logits, L->baseline, nullptr, nullptr, st);
  if (rc) return rc;
  CU(launch_impala_tail(behavior_logits, L->logits, L->baseline, action, reward, done, c.T, c.B, c.A, c.discounting, c.reward_clip_abs_one,
                        c.clip_rho_threshold, c.clip_pg_rho_threshold, c.baseline_cost, c.entropy_cost, vs, pg_advantages, L->dlogits,
                        L->dbaseline, losses, L->scratch, st), "impala_tail");
  CU(cudaMemsetAsync(L->grads, 0, L->small_len * sizeof(float), st), "zero small grads");
  CU(cudaMemsetAsync(L->grads + L->lstm_off0, 0, L->lstm_len * sizeof(float), st), "zero lstm grads");
  CU(launch_head_dense_bwd(L->lstm_out, L->dlogits, L->dbaseline, L->P.wp, L->P.wb, NB, c.A, L->dout, L->G.wp, L->G.bp, L->G.wb, L->G.bb, st),
     "head_dense_bwd");
  rc = srl_lstm_backward(L->lstm, L->dout, done, L->dcore, st);
  if (rc) return fail(rc, "lstm_backward: %s", srl_lstm_last_error());
  CU(launch_dcore_to_dh(L->dcore, L->buf.h, NB, c.A, L->buf.hi.dh, st), "dcore_to_dh");
  CU(encoder_backward(NB, L->buf, L->G, L->maps, c.precision, st, L->pf, L->ss, 2), "encoder_backward");
  L->have_fwd = true;
  return 0;
}

extern "C" int srl_learner_apply_gradients(srl_learner_t* L, float* grad_norm_out, void* stream) {
  REQ(L, "learner is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  const srl_config_t& c = L->cfg;
  L->pf.st = st;
  L->step += 1;
  // clip_grad_norm_ + optimizer in one cooperative kernel (profile slot: optimizer)
  L->pf.b(PS_OPTIMIZER);
  if (c.optimizer == 0) {
    CU(launch_clip_optim(0, L->params, L->grads, L->opt0, nullptr, L->nparams, c.max_grad_norm, L->coef, L->scratch + 2048, c.learning_rate,
                         c.alpha, 0.f, c.epsilon, L->step, L->dstep, L->ox, st), "clip+rmsprop");
  } else {
    CU(launch_clip_optim(1, L->params, L->grads, L->opt0, L->opt1, L->nparams, c.max_grad_norm, L->coef, L->scratch + 2048, c.learning_rate,
                         c.adam_beta1, c.adam_beta2, c.adam_eps, L->step, L->dstep, L->ox, st), "clip+adam");
  }
  L->pf.e(PS_OPTIMIZER);
  if (grad_norm_out) CU(cudaMemcpyAsync(grad_norm_out, L->coef, (L->report_lr ? 3 : 2) * sizeof(float), cudaMemcpyDeviceToDevice, st), "copy coef");
  return 0;
}

extern "C" int srl_learner_apply_gradients_dp(srl_learner_t* L, const srl_dp_peers_t* peers, float* grad_norm_out, void* stream) {
  REQ(L && peers, "apply_gradients_dp: NULL argument");
  REQ(peers->world >= 2 && peers->world <= 8 && peers->rank >= 0 && peers->rank < peers->world, "apply_gradients_dp: world=%d rank=%d",
      peers->world, peers->rank);
  REQ(peers->grads[peers->rank] == (void*)L->grads, "apply_gradients_dp: grads[rank] must be the learner's gradient buffer");
  cudaStream_t st = (cudaStream_t)stream;
  const srl_config_t& c = L->cfg;
  DpPeers P;
  for (int i = 0; i < 8; ++i) {
    P.g[i] = i < peers->world ? (float*)peers->grads[i] : nullptr;
    P.ctl[i] = i < peers->world ? (unsigned*)peers->ctl[i] : nullptr;
    P.rs[i] = i < peers->world ? (float*)peers->exchange[i] : nullptr;
    REQ(i >= peers->world || (P.g[i] && P.ctl[i] && P.rs[i]), "apply_gradients_dp: NULL peer pointer %d", i);
  }
  P.rank = peers->rank; P.world = peers->world; P.mc_g = (float*)peers->grads_multicast;
  L->pf.st = st;
  L->step += 1;
  L->pf.b(PS_OPTIMIZER);
  if (c.optimizer == 0) {
    CU(launch_dp_clip_optim(0, L->params, L->grads, L->opt0, nullptr, L->nparams, c.max_grad_norm, L->coef, L->scratch + 2048,
                            c.learning_rate, c.alpha, 0.f, c.epsilon, L->step, L->dstep, P, L->ox, st), "dp clip+rmsprop");
  } else {
    CU(launch_dp_clip_optim(1, L->params, L->grads, L->opt0, L->opt1, L->nparams, c.max_grad_norm, L->coef, L->scratch + 2048,
                            c.learning_rate, c.adam_beta1, c.adam_beta2, c.adam_eps, L->step, L->dstep, P, L->ox, st), "dp clip+adam");
  }
  L->pf.e(PS_OPTIMIZER);
  if (grad_norm_out) CU(cudaMemcpyAsync(grad_norm_out, L->coef, (L->report_lr ? 3 : 2) * sizeof(float), cudaMemcpyDeviceToDevice, st), "copy coef");
  return 0;
}

extern "C" int srl_learner_set_profiling(srl_learner_t* L, int enable) {
  REQ(L, "learner is NULL");
  if (enable && !L->events[0])
    for (int i = 0; i < 2 * PS_COUNT; ++i) CU(cudaEventCreate(&L->events[i]), "cudaEventCreate");
  L->pf.on = enable != 0;
  L->pf.ev = L->events;
  return 0;
}
extern "C" int srl_profile_slot_count(void) { return PS_COUNT; }
extern "C" const char* srl_profile_slot_name(int slot) { return (slot >= 0 && slot < PS_COUNT) ? kSlotNames[slot] : ""; }
extern "C" int srl_learner_profile_collect(srl_learner_t* L, float* ms_out_host) {
  REQ(L && ms_out_host, "profile_collect: NULL argument");
  REQ(L->pf.on, "profile_collect: profiling is off");
  for (int i = 0; i < PS_COUNT; ++i) {
    float ms = 0.f;
    cudaError_t e = cudaEventSynchronize(L->events[2 * i + 1]);
    if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, L->events[2 * i], L->events[2 * i + 1]);
    if (e != cudaSuccess) { cudaGetLastError(); ms = -1.f; }   // slot not recorded in the last step
    ms_out_host[i] = ms;
  }
  return 0;
}

extern "C" int srl_learner_snapshot_params(srl_learner_t* L, float* dst, const float* losses, void* stream) {
  REQ(L && dst, "snapshot_params: NULL argument");
  REQ((reinterpret_cast<uintptr_t>(dst) & 15) == 0, "snapshot_params: dst must be 16-byte aligned");
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
