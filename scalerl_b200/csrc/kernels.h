// Internal launch prototypes shared by the .cu translation units (not part of the C ABI).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

namespace srl {

// per-kernel CUDA-event bracketing (bench.py's roofline numbers): slots of one learner step
enum ProfSlot { PS_S2D = 0, PS_CONV1_FWD, PS_CONV2_FWD, PS_CONV3_FWD, PS_FC_FWD, PS_HEAD_FWD, PS_TAIL, PS_ZERO_GRADS, PS_HEAD_BWD,
                PS_FC_WGRAD, PS_FC_DGRAD, PS_CONV3_WGRAD, PS_CONV3_DGRAD, PS_CONV2_WGRAD, PS_CONV2_DGRAD, PS_CONV1_WGRAD,
                PS_WGRAD_FINALIZE, PS_GRAD_NORM, PS_OPTIMIZER, PS_PACK, PS_ENC_FUSED, PS_COUNT };
// ---- programmatic dependent launch (see common.cuh) ----------------------------------------------------------
// pdl_active(): SRL_PDL != 0 (default on) and not switched off by the caller (per-kernel profiling records events between
// the kernels, which would serialise them anyway).
bool pdl_active();
void pdl_set_active(bool on);      // per calling thread: every C-ABI entry point that reaches launch_chain sets it first
template <class... KA, class... A>
inline cudaError_t launch_chain(void (*kernel)(KA...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = pdl_active() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, args...);
}

// Per-DEVICE once flags (a process may drive several GPUs: function attributes and occupancy are per device).
struct PerDeviceOnce {
  bool done[64] = {};
  // returns the current device ordinal, or -1 on error; *first = true when this device has not been marked yet
  int device(bool* first) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) { *first = true; return -1; }
    *first = !done[dev];
    return dev;
  }
  void mark(int dev) { if (dev >= 0 && dev < 64) done[dev] = true; }
};
template <class K>
inline cudaError_t ensure_max_dynamic_smem(PerDeviceOnce& once, K kernel, int bytes) {
  bool first;
  const int dev = once.device(&first);
  if (!first) return cudaSuccess;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess) once.mark(dev);
  return e;
}

void kstamp_set_encoder(unsigned long long*); void kstamp_set_vtrace(unsigned long long*); void kstamp_set_heads(unsigned long long*);   // diagnostics build (common.cuh)
void kstamp_set_optim(unsigned long long*);

// The stream schedule of one learner call: `main` is the caller's stream, each lane a stream of the learner context that runs work
// beside it (also under capture): pack (weight re-pack + gradient memset; priority: api.cu pack_priority), fc_wgrad (a3 transpose,
// head wgrad, fc wgrad), conv3_wgrad and conv2_wgrad (each with its reduce).  fork(l): the lane waits for all work on main so far;
// join(l): main waits for all work on the lane so far.  cudaStreamWaitEvent binds to the event's latest record (eagerly and under
// capture), so one fork and one join event per lane serve every edge.  Collapsed (per-kernel profiling on, or the lanes could not be
// created): every lane is main and fork / join do nothing.
enum Lane { LANE_PACK, LANE_FC_WGRAD, LANE_CONV3_WGRAD, LANE_CONV2_WGRAD, LANE_COUNT };
struct StepStreams {
  cudaStream_t main = nullptr;
  cudaStream_t side[LANE_COUNT] = {};
  cudaEvent_t forked[LANE_COUNT] = {}, joined[LANE_COUNT] = {};
  bool have_lanes = false;          // every lane stream and event was created (srl_learner_create)
  bool collapsed = true;
  bool profiling = false;           // per-kernel event bracketing on main (srl_learner_set_profiling): slots of one learner step
  cudaEvent_t slot_events[2 * PS_COUNT] = {};
  // the start of every learner call that launches work: main, the collapse state and the PDL mode; returns main
  cudaStream_t begin_call(cudaStream_t st) { main = st; collapsed = !have_lanes || profiling; pdl_set_active(!profiling); return st; }
  cudaStream_t lane(Lane l) const { return collapsed ? main : side[l]; }
  cudaError_t fork(Lane l) const { return collapsed ? cudaSuccess : edge(forked[l], main, side[l]); }
  cudaError_t join(Lane l) const { return collapsed ? cudaSuccess : edge(joined[l], side[l], main); }
  void b(int slot) const { if (profiling) cudaEventRecord(slot_events[2 * slot], main); }
  void e(int slot) const { if (profiling) cudaEventRecord(slot_events[2 * slot + 1], main); }
  static cudaError_t edge(cudaEvent_t ev, cudaStream_t from, cudaStream_t to) {
    const cudaError_t e = cudaEventRecord(ev, from);
    return e != cudaSuccess ? e : cudaStreamWaitEvent(to, ev, 0);
  }
};

// A device buffer table: one row per tensor in carving order, every tensor 256-byte aligned.  The learner's workspace (api.cu), the
// stand-alone encoder's blocks (api.cu encoder_rows) and the LSTM core's (lstm.cu lstm_rows) are carved from such tables.
struct WsRow {
  const char* name;
  int elem;                       // bytes per element
  int64_t count;                  // elements
  void** hi;                      // receives the tensor's address (null: zeros only)
  void** lo;                      // receives the low twin's address (null: no twin)
};
template <class T>
inline WsRow ws_row(const char* name, int64_t count, T** hi, T** lo = nullptr) {
  return {name, (int)sizeof(T), count, reinterpret_cast<void**>(hi), reinterpret_cast<void**>(lo)};
}
inline int64_t ws_bytes(const WsRow& r) { return ((int64_t)r.elem * r.count + 255) & ~int64_t(255); }
// bytes of rows [0, n), a low twin after each row that has one in the fp32-accurate mode (split)
inline int64_t rows_bytes(const WsRow* t, int n, bool split) {
  int64_t total = 0;
  for (int i = 0; i < n; ++i) total += ws_bytes(t[i]) * (split && t[i].lo ? 2 : 1);
  return total;
}
// gives rows [0, n) consecutive addresses from q (each row padded to 256 bytes), in table order
inline void carve_rows(const WsRow* t, int n, bool split, char* q) {
  for (int i = 0; i < n; ++i) {
    if (t[i].hi) *t[i].hi = q;
    q += ws_bytes(t[i]);
    if (split && t[i].lo) { *t[i].lo = q; q += ws_bytes(t[i]); }
  }
}
// The two caller-owned blocks of the stand-alone encoder and LSTM core calls: rows [0, n_saved) of a table form the saved block (what
// a backward reads of its forward), rows [n_saved, n) the scratch block (one call's temporaries).
inline void block_bytes(const WsRow* t, int n, int n_saved, bool split, int64_t* saved, int64_t* scratch) {
  *saved = rows_bytes(t, n_saved, split);
  *scratch = rows_bytes(t + n_saved, n - n_saved, split);
}
// carves both blocks, then makes the device's primary context current on this thread: encoding the call's tensor maps needs it, and
// this may be the thread's first CUDA call (torch runs a backward on an autograd thread of its own)
inline cudaError_t carve_blocks(const WsRow* t, int n, int n_saved, bool split, void* saved, void* scratch) {
  carve_rows(t, n_saved, split, static_cast<char*>(saved));
  carve_rows(t + n_saved, n - n_saved, split, static_cast<char*>(scratch));
  int dev = 0;
  const cudaError_t e = cudaGetDevice(&dev);
  return e != cudaSuccess ? e : cudaSetDevice(dev);
}
// most frames of one call: (T+1)*B of a learner context, the stand-alone encoder's frames, the stand-alone LSTM core's T1*B rows
constexpr int MAX_FRAMES = 65536;

// per-CTA partials of the wgrad kernels (each CTA stores its accumulators, in the kernel's native [tap-block][row][co] order, and its
// bias sums; conv_wgrad_reduce_kernel<layer> adds the CTAs in a fixed order into the PyTorch-layout gradient, so the gradients are the
// same bits on every run).  Floats per CTA: accumulators, then bias.
constexpr int WG_PART_CTAS = 160;              // most CTAs a wgrad launch may use
constexpr int WSP_W3 = 5 * 128 * 64 + 64, WSP_W2 = 4 * 128 * 64 + 64, WSP_W1 = 2 * 128 * 32 + 32;
constexpr int64_t WSP_TOTAL = (int64_t)WG_PART_CTAS * (WSP_W3 + WSP_W2 + WSP_W1);
constexpr int HEAD_GROUPS = 32;                // slab groups (partial sums) of the head weight gradients (heads.cu)

// ---- vtrace.cu
cudaError_t launch_vtrace_iw(const float* log_rhos, const float* discounts, const float* rewards, const float* values,
                             const float* bootstrap, int T, int B, float clip_rho, float clip_pg, float* vs, float* pg, int variant,
                             cudaStream_t st);
cudaError_t launch_vtrace_logits(const float* bl, const float* tl, const int64_t* actions, const float* discounts, const float* rewards,
                                 const float* values, const float* bootstrap, int T, int B, int A, float clip_rho, float clip_pg,
                                 float* vs, float* pg, float* lr, float* balp, float* talp, cudaStream_t st);
cudaError_t launch_policy_rows_fwd(const float* logits, const int64_t* actions, int64_t N, int A, float* logp, float* ent, cudaStream_t st);
cudaError_t launch_policy_rows_bwd(const float* logits, const int64_t* actions, const float* w_logp, const float* w_ent, int64_t N, int A,
                                   float* dlogits, cudaStream_t st);
cudaError_t launch_sample_actions(const float* logits, const float* u, int64_t N, int A, int64_t* actions, cudaStream_t st);
cudaError_t launch_reduce_sum(const float* x, int64_t n, int square, float scale, float* out, cudaStream_t st);
// one learner tail over [T+1, B] batch rows (V-trace, losses, head gradients): trajectory (rows 1..T used), shape, srl_config_t's loss
// settings (clip < 0: none), outputs as srl_impala_loss_and_head_grads (vs, pg may be null; scratch zero before the first launch)
struct TailStep {
  const float* bl; const int64_t* action; const float* reward; const uint8_t* done;
  int T, B, A;
  float discounting; int clip_reward; float clip_rho, clip_pg, baseline_cost, entropy_cost;
  float *vs, *pg, *dlogits, *dbaseline, *losses, *scratch;
};
// the tail from target logits tl [T+1][B][A] and baseline [T+1][B] in global memory
cudaError_t launch_impala_tail(const TailStep& s, const float* tl, const float* baseline, cudaStream_t st);
// the heads from the fc layer's split-K partials, then the tail, then dh (and dh_lo when not null), one block per column
bool column_step_supported(int T, int B, int A);
cudaError_t launch_column_step(const TailStep& s, const float* hpart, int nsplit, const float* bfc, float* h, const float* Wp, const float* bp,
                               const float* Wb, const float* bb, float* logits, float* baseline, __nv_bfloat16* dh, __nv_bfloat16* dh_lo,
                               cudaStream_t st);

// ---- heads.cu
// hpart: FC_SPLITS split-K partials [s][N][512] of the fc layer; writes h = relu(sum_s hpart + bfc) and the head outputs
cudaError_t launch_head_fwd(const float* hpart, int nsplit, const float* bfc, float* h, const float* reward, const int64_t* action,
                            const float* Wp, const float* bp, const float* Wb, const float* bb, int N, int A, float* logits,
                            float* baseline, cudaStream_t st);
cudaError_t launch_head_bwd(const float* dlogits, const float* dbaseline, const float* h, const float* reward, const int64_t* action,
                            const float* Wp, const float* Wb, int N, int A, __nv_bfloat16* dh, float* gWp, float* gbp, float* gWb,
                            float* gbb, float* part, cudaStream_t st, cudaStream_t st_wgrad, bool do_dh = true, __nv_bfloat16* dh_lo = nullptr);
cudaError_t launch_core_build(const float* hpart, int nsplit, const float* bfc, const float* reward, const int64_t* action, int N, int A, float* h,
                              float* core, cudaStream_t st);
cudaError_t launch_head_dense_fwd(const float* X, const float* Wp, const float* bp, const float* Wb, const float* bb, int N, int A, float* logits,
                                  float* baseline, cudaStream_t st);
cudaError_t launch_head_dense_bwd(const float* X, const float* dlogits, const float* dbaseline, const float* Wp, const float* Wb, int N, int A,
                                  float* dX, float* gWp, float* gbp, float* gWb, float* gbb, cudaStream_t st);
// dh_lo != nullptr: also the low twin bf16(v - bf16(v)) of the fp32-accurate operand mode
cudaError_t launch_dcore_to_dh(const float* dcore, const float* h, int N, int A, __nv_bfloat16* dh, cudaStream_t st, __nv_bfloat16* dh_lo = nullptr);
cudaError_t launch_unpack_slots(const uint8_t* staging, int64_t slot_bytes, const int64_t* off6, int T, int B, int A, uint8_t* obs, float* reward,
                                uint8_t* done, int64_t* action, float* logits, float* episode_return, cudaStream_t st);

// ---- optim.cu
// learning-rate schedule and RMSprop momentum of the fused clip + optimizer step (srl_learner_set_lr_schedule / _set_momentum).
// The default value is the plain step: constant lr, no momentum.
enum { SCHED_CONSTANT = 0, SCHED_LINEAR = 1 };
struct OptExtra {
  int schedule = SCHED_CONSTANT;
  float lr_end = 0.f;                               // SCHED_LINEAR: floor of the decayed lr
  double frames_per_step = 0.0, total_frames = 1.0; // SCHED_LINEAR: F (frames of one optimizer step, all ranks) and Ftot
  float* buf = nullptr;                             // momentum buffer, parameter layout (null: no momentum)
  float momentum = 0.f;
};
// one fused clip + optimizer step.  optimizer 0 = RMSprop: s0 = square_avg, a = alpha; 1 = Adam: s0, s1 = exp_avg, exp_avg_sq,
// a, b = beta1, beta2.  coef receives the norm, the clip coefficient and (but for the constant-lr, no-momentum step) the lr;
// scratch holds the block partials.  The step count is *dstep + 1 (step when dstep is null); the kernel stores it back to *dstep.
struct OptStep {
  int optimizer;
  float *p, *g, *s0, *s1;
  int64_t n;
  float max_norm;
  float *coef, *scratch;
  float lr, a, b, eps;
  int step;
  int* dstep;
  OptExtra x;
};
// blocks (may be null) receives the grid size launched, variant (may be null) the template's parameters 4 OPT + 2 SCHED + MOM
cudaError_t launch_clip_optim(const OptStep& o, cudaStream_t st, int* blocks = nullptr, int* variant = nullptr);
struct DpPeers { float* g[8]; float* rs[8]; unsigned* ctl[8]; int rank, world; float* mc_g; };      // peer-mapped gradient buffers / control blocks; mc_g: NVLS multicast address of the gradient buffers (or null)
cudaError_t launch_dp_clip_optim(const OptStep& o, const DpPeers& P, cudaStream_t st);
cudaError_t launch_snapshot_if_finite(float* dst, const float* src, int64_t n, const float* losses, cudaStream_t st);
cudaError_t launch_grad_norm(const float* g, int64_t n, float max_norm, float* coef, float* scratch, cudaStream_t st);
cudaError_t launch_rmsprop(float* p, const float* g, float* v, int64_t n, const float* coef, float lr, float alpha, float eps,
                           cudaStream_t st);
cudaError_t launch_adam(float* p, const float* g, float* m, float* v, int64_t n, const float* coef, float lr, float b1, float b2, float eps,
                        int step, cudaStream_t st);

// ---- dqn.cu, dqn_cat.cu, dqn_qr.cu: the Q head of the Ape-X learner step and actors (srl_apex_*)
// The encoder runs with a one-hot width of 1 for the Q network: its core rows are [h (512), clamp(reward), 1], ENC_CORE floats.
constexpr int ENC_CORE = 514;
constexpr int CAT_MAX_ATOMS = 64;
constexpr int QR_MAX_QUANTILES = 256;
// the categorical head's support z_k = v_min + k dz (dqn_cat.cuh)
struct CatSupport {
  float v_min, v_max, dz;
  int K;
};
// dz = (v_max - v_min) / (K - 1) in double, rounded once to fp32
inline CatSupport cat_support(int K, float v_min, float v_max) {
  return {v_min, v_max, (float)(((double)v_max - (double)v_min) / (double)(K - 1)), K};
}
// the quantile head's N quantiles per action and its Huber threshold kappa > 0 (dqn_qr.cuh)
struct QrSetting {
  int N;
  float kappa;
};
enum QKind { Q_PLAIN, Q_DUELING, Q_CATEGORICAL, Q_QUANTILE };
// One Q head on the 512 h columns of the core rows, bound onto a flat parameter buffer (apex_layout order):
//   Q_PLAIN        q = Linear(512, A): W = q.weight [A][512], b = q.bias [A]
//   Q_DUELING      V + Adv - mean(Adv) (dqn_head.cuh's dueling_q): W = [value.weight; advantage.weight] [(A + 1)][512] (the value row
//                  first), b = value.bias [1], ba = advantage.bias [A]
//   Q_CATEGORICAL  C51, q = Linear(512, A K) (dqn_cat.cuh): W = q.weight [A K][512], b = q.bias [A K] (row a K + k: atom k of action
//                  a) on the support c
//   Q_QUANTILE     QR-DQN, q = Linear(512, A N) (dqn_qr.cuh): W = q.weight [A N][512], b = q.bias [A N] (row a N + i: quantile i of
//                  action a), with the setting qr
// R = W's rows: A, A + 1, A K or A N.  The distributional dueling head (ApexNetDesc.vrows) is a Q_CATEGORICAL or Q_QUANTILE head on
// the composed rows of its value and advantage layers (dueling_rows.cu).
struct QHead {
  QKind kind;
  int A, R;
  const float *W, *b, *ba;
  CatSupport c;
  QrSetting qr;
};
// the categorical and quantile heads run a GEMM to their rows [N][R] (logits, quantiles) before anything else of theirs
inline bool head_has_logits(const QHead& h) { return h.kind == Q_CATEGORICAL || h.kind == Q_QUANTILE; }
// the same tensors of a gradient buffer
struct QHeadGrad {
  float *gW, *gb, *gba;
};

// One batch of B transitions: the core rows of the online forward over s, of the online forward over s' (NULL: no double DQN) and of
// the target forward over s'; the batch columns; outputs q (Q(s, a); categorical: sum z p at the taken action), y (the target;
// categorical: sum z m; quantile: the mean of the target quantiles), priorities f64 [B], dcore [B][ENC_CORE] and loss [1] (mean(w
// (q - y)^2); categorical: mean(w ce); quantile: mean(w loss)).
// scratch: 4 + dqn_tail_blocks(B) floats, zero before the first launch (re-armed by the kernel).  The scalar heads write dq [B] and
// reduce the head gradients through head_part (HEAD_GROUPS * R * 513 floats); the categorical head writes the logits [B][A K] of the
// three forwards (logits_n: double DQN only), the projected targets m [B][K], ce [B] and dlogits [B][A K] (zero outside the taken
// action's K rows).  The quantile head writes the same slots: its quantiles theta [B][A N] in the logits, the target quantiles
// [B][N] in m, the per-transition loss [B] in ce and dtheta [B][A N] in dlogits.
struct QTail {
  const float *core_s, *core_n, *core_nt;
  const int64_t* action; const float* reward; const uint8_t* done; const float* weight;
  int B;
  float gamma, priority_eps;
  float *q, *y, *dcore, *loss, *scratch;
  double* prio;
  float *dq, *head_part;
  float *logits_s, *logits_n, *logits_nt, *m, *ce, *dlogits;
};
inline int dqn_tail_blocks(int B) { return (B + 3) / 4; }
// the tail of `on` (the online head) and `tg` (the target head); the categorical and quantile heads run their logits GEMMs first
cudaError_t launch_q_tail(const QHead& on, const QHead& tg, const QTail& t, cudaStream_t st);
// the head gradients (stored) of the tail t has run
cudaError_t launch_q_wgrad(const QHead& h, const QHeadGrad& g, const QTail& t, cudaStream_t st);
// q_out [N][A] = Q(h) over N core rows; the categorical and quantile heads go through logits [N][R]
cudaError_t launch_q_values(const QHead& h, const float* core, int N, float* logits, float* q_out, cudaStream_t st);
cudaError_t launch_apex_soft_update(const float* p, float* pt, int64_t n, float tau, float one_minus_tau, cudaStream_t st);
// ---- noisy.cu: noisy networks (Fortunato et al. 2018, factorised Gaussian noise) on the fc layer and the Q head
// One network's noise vector f(x) = sgn(x) sqrt|x| of standard normals x, nn = noise_count floats:
//   [fc in 3136 | fc out 512 | head in 512 (value and advantage layers: the value layer's, then the advantage layer's) | head out
//   (the head's parameter rows: the value rows, then the advantage rows)]; every segment but the last starts on a multiple of 4 floats.
constexpr int NOISE_FC_IN = 3136, NOISE_FC_OUT = 512, NOISE_HEAD_IN = 512, NOISE_HEAD_IN_OFF = NOISE_FC_IN + NOISE_FC_OUT;
// the noisy layers' tensors on one flat buffer, [0] mu and [1] sigma (of the parameters, or of their gradients): the fc weight
// [512][3136] and bias [512]; the head's parameter rows: W [rows][512], b and (value and advantage layers) ba
struct NoisyTensors {
  float *fc_w[2], *fc_b[2];
  float *h_w[2], *h_b[2], *h_ba[2];
};
// the composed (effective) weights of one network in the same layouts
struct NoisyWeights {
  float *fc_w, *fc_b, *h_w, *h_b, *h_ba;
};
// the normals and noise of `nets` (1 or 2) networks; network i's go to normals[i] / noise[i] (nn floats each).  Philox4x32-10 under
// `key`, counter (g, 'nois', c, c >> 32 | i << 31) for the normals 4g .. 4g + 3 (Box-Muller).  c = *step (the learner's Adam step
// count, read only), or *draws (the actor's noise counter: nets = 1, advanced by one when the draw ends)
cudaError_t launch_noisy_draw(uint2 key, const int* step, unsigned long long* draws, int nets, int nn, float* const* normals,
                              float* const* noise, cudaStream_t st);
struct ApexNetDesc;
// w[i] = p[i]'s mu + sigma (.) (f(eps_out) f(eps_in)^T) and mu_b + sigma_b (.) f(eps_out) under noise[i], for the `nets` networks of d
cudaError_t launch_noisy_compose(const NoisyTensors* p, const NoisyWeights* w, const float* const* noise, int nets, const ApexNetDesc& d,
                                 cudaStream_t st);
// the sigma gradients g.x[1] = g.x[0] (.) eps of the online network's noise (the mu gradients are those of the composed weights)
cudaError_t launch_noisy_sigma_grad(const NoisyTensors& g, const float* noise, const ApexNetDesc& d, cudaStream_t st);

// The Ape-X Q network a setting describes: its head as the kernels read it, unbound, whether fc and the head layers are noisy (0 or 1),
// and the head's value rows, the one place that decides the head's parameter rows: 0 (one layer, q), 1 (the scalar dueling head,
// whose kernels read value and advantage themselves) or W = K or N (the distributional dueling head: value [W][512] and advantage
// [A W][512], composed into the A W rows the head's kernels read)
struct ApexNetDesc {
  QHead head;
  int noisy;
  int vrows;
};
// the rows of the advantage layer (of q without a value layer)
inline int adv_rows(const ApexNetDesc& d) { return d.head.kind == Q_DUELING ? d.head.A : d.head.R; }
// the head's parameter rows: the value rows, then the advantage rows
inline int param_rows(const ApexNetDesc& d) { return d.vrows + adv_rows(d); }
// the distributional dueling head: the kernels read composed rows, not the parameters
inline bool dist_dueling(const ApexNetDesc& d) { return d.vrows > 0 && d.head.kind != Q_DUELING; }
// api.cu: the network of a setting (num_atoms 0: no categorical head, whose support is not read; num_quantiles 0: no quantile
// head, whose kappa is not read; dist_dueling 1: that head as value and advantage layers).  0, or SRL_EINVAL with "<who>: ..." as the
// message
int make_apex_desc(const char* who, int A, int dueling, int num_atoms, float v_min, float v_max, int num_quantiles, float kappa,
                   int dist_dueling, int noisy, ApexNetDesc* d);
// the floats of one network's noise vector (0 without noise)
inline int noise_count(const ApexNetDesc& d) {
  return d.noisy ? NOISE_HEAD_IN_OFF + NOISE_HEAD_IN * (d.vrows ? 2 : 1) + param_rows(d) : 0;
}
// api.cu: the flat parameter layout of network d (srl_apex_param_layout*'s): the offsets and counts (NULL: not wanted) of its
// tensors in state_dict order (10, 12 dueling; noisy: 14, 18 dueling) -> the buffer's floats
int64_t apex_layout(const ApexNetDesc& d, int64_t* off, int64_t* cnt);
// One network of d on a flat buffer of its layout: the encoder's 8 tensors and the Q head (noisy: fc's and the head's mu tensors),
// the head as a gradient binding, and (noisy) the noisy layers' mu / sigma pairs
struct ApexNet {
  float* w8[8];
  QHead q;
  QHeadGrad g;
  NoisyTensors nz;
};
// api.cu
ApexNet bind_apex(const ApexNetDesc& d, float* base);
// the network a forward of `net` runs on: noisy, net's conv tensors with fc and the head from the composed weights w; else net
ApexNet apex_forward_net(const ApexNetDesc& d, const ApexNet& net, const NoisyWeights& w);
// ---- dueling_rows.cu: the distributional dueling head's rows W_eff [R][512], b_eff [R] (R = A W), or their gradients
struct HeadRows {
  float *W, *b;
};
// the head h reads on rows r
inline QHead on_rows(QHead h, const HeadRows& r) { h.W = r.W; h.b = r.b; h.ba = nullptr; return h; }
// rows[i] = (v + adv) - mean_a adv of p[i] (bound as the scalar dueling head: W = [value.weight; advantage.weight], b = value.bias,
// ba = advantage.bias) for the `nets` networks, V = W rows per action
cudaError_t launch_dist_dueling_compose(const QHead* p, const HeadRows* rows, int nets, int V, cudaStream_t st);
// the value and advantage gradients (out: the parameter-side binding, stored) of the rows' gradients g
cudaError_t launch_dist_dueling_grad(const HeadRows& g, const QHeadGrad& out, int A, int V, cudaStream_t st);
// the rows of one network's normals, noise and composed weights (empty without noise), named with the suffix `which` (0: none,
// 1: _online, 2: _target) -> the rows written
int noise_rows(const ApexNetDesc& d, int which, float** normals, float** noise, NoisyWeights* w, WsRow* t);

// dqn_cat.cu: the categorical halves of the launchers above
// logits [N][R] = h W^T + b over N core rows (stride ENC_CORE), W [R][512]: one fmaf chain per logit over j = 0 .. 511 from 0, then
// + b rounded once, whatever the tiling
cudaError_t launch_cat_logits(const float* core, const float* W, const float* b, int N, int R, float* logits, cudaStream_t st);
cudaError_t launch_cat_tail(const QHead& on, const QHead& tg, const QTail& t, cudaStream_t st);
// gW [R][512] = dlogits^T h, gb [R] = dlogits^T 1 over the N core rows (stored), each a fmaf chain over n = 0 .. N-1 in order
cudaError_t launch_cat_wgrad(const float* dlogits, const float* core, int N, int R, float* gW, float* gb, cudaStream_t st);
// dqn_qr.cu: the quantile head's tail (its quantiles, head gradients and q values run dqn_cat.cu's GEMMs)
cudaError_t launch_qr_tail(const QHead& on, const QHead& tg, const QTail& t, cudaStream_t st);

}  // namespace srl
struct srl_per;
struct srl_apex_actor;
namespace srl {
// ---- per.cu: what the replay memory (replay.cu) shares with its sampler, whose leaf i is the memory's ring slot i
int64_t per_tree_ptr(const srl_per* P);          // the leaf the next add writes
// n new leaves at tree_ptr.. = priorities[i]^alpha (f64 [n], device), max_priority updated, the count advanced as by srl_per_add; a
// non-finite priority is stored as max_priority^alpha and counted by srl_per_invalid_updates.  0, or an error code with the message set
int per_add_prioritized(srl_per* P, const double* priorities, int64_t n, cudaStream_t st);
// the per-leaf retired mask (u8 [memory_size] on the device, zeroed, owned by the caller; frame_replay.cu).  With it, srl_per_update_priorities
// skips retired leaves without counting them, every add makes the leaves it writes live again, and the sample's descent skips subtrees
// of sum 0.  Without it (a NULL mask, the default) every kernel computes what it computed before retirement existed.
void per_attach_retired(srl_per* P, uint8_t* retired);
// leaves[0 .. *n_dev) (device count, read when the kernel runs) retire: sum 0, min +inf, marked in the mask.  Needs the mask attached.
int per_retire(srl_per* P, const int64_t* leaves, const unsigned long long* n_dev, cudaStream_t st);
// ---- apex_actor.cu: what the prioritized add (replay.cu) uses of an Ape-X actor
int apex_actor_num_envs(const srl_apex_actor* X);
// the actor's initial priorities of E transitions that sit in ring slots (ptr + e) mod M: s = state rows, s' = next_state rows (u8
// [E,4,84,84] each), action / reward / done read from the ring's slots.  p = |Q(s)[a] - (R + gamma_n (1 - d) max_a Q(s'))| + eps with
// the learner tail's arithmetic (dqn_head.cuh) -> *prio, the actor's f64 [E] device buffer.  0, or an error code with the message set
int apex_actor_priorities(srl_apex_actor* X, const uint8_t* s, const uint8_t* s_next, const int64_t* action, const float* reward,
                          const uint8_t* done, int64_t ptr, int64_t M, float gamma_n, float eps, const double** prio, cudaStream_t st);
// srl_per_sample with an optional device beta (beta_dev, read when the kernel runs; NULL: `beta`)
int per_sample(srl_per* P, const double* uniforms, int batch, double beta, const double* beta_dev, int64_t* idxs, double* weights64,
               float* weights32, cudaStream_t st);

// ---- encoder.cu
// packed bf16 operand copies of the conv/fc weights (element offsets into one buffer)
struct WPack {
  static constexpr int64_t W1K = 0;                       // [32][256]            k = (kh2,kw2,c,dy,dx), kh=4kh2+dy, kw=4kw2+dx
  static constexpr int64_t W2K = W1K + 32 * 256;          // [64][512]            k = (kh,kw,c)
  static constexpr int64_t W3K = W2K + 64 * 512;          // [64][576]            k = (kh,kw,c)
  static constexpr int64_t WFK = W3K + 64 * 576;          // [512][3136]          k = (hw,c)
  static constexpr int64_t WFD = WFK + 512 * 3136;        // [3136][512]          row = (hw,c), k = j
  static constexpr int64_t W3D = WFD + 3136 * 512;        // [64 c][576]          k = (kh,kw,co)
  static constexpr int64_t W2D = W3D + 64 * 576;          // [4 cls][32 c][256]   k = (kh',kw',co)
  static constexpr int64_t TOTAL = W2D + 4 * 32 * 256;
};
// pointers to the fp32 master tensors inside the flat parameter (or gradient) buffer
struct ParamPtrs {
  float *w1, *b1, *w2, *b2, *w3, *b3, *wf, *bf, *wp, *bp, *wb, *bb;
};
constexpr int FC_SPLITS = 4;
// The bf16 operand tensors of the GEMMs.  The fp32-accurate operand mode (srl_config_t.precision = 1) holds a second set, the "low"
// twins bf16(v - bf16(v)) in the same layouts.  xs has none: u8 frames are exact in bf16.
struct OperandTensors {
  __nv_bfloat16 *a1, *a2, *a3;          // a1 [2 planes][NF*100][64], a2 [NF*81][64], a3 [NF*49][64]
  __nv_bfloat16 *dh, *da3, *da2, *da1;  // dh [NB][512]; da3g [NB*81][64], da2g [NB*100][64], da1g [NB*441][32] (grid layouts, zero-padded)
  __nv_bfloat16* wpack;
};
struct EncoderBuffers {   // row layouts: see res_problems.cuh
  __nv_bfloat16* xs;                    // space-to-depth bf16 copy of the u8 frames [NF*441][64], 64 = (c,dy,dx)
  OperandTensors hi, lo = {};           // lo: all null in the bf16 mode
  __nv_bfloat16* a3t = nullptr;         // [NF][64*49]: a3 of the learning frames in fc.weight's own column order (c,h,w) -- fc wgrad's B operand (bf16 mode)
  float* hpart;                         // [FC_SPLITS][NF][512] split-K partials of the fc layer
  float* h;                             // [NF][512] fc output (post-ReLU), fp32
  float* wgrad_part;                    // per-CTA partials of the conv wgrad kernels (WSP_TOTAL floats)
  int NF;                               // frames the forward buffers were sized for (plane stride of a1)
};
// The encoder's rows, for NF forward and NB backward frames.  The first ENC_SAVED_ROWS are what a backward reads of its forward: the
// activations and the packed weights the forward ran with.  The rest live for one call: the fc layer's split-K partials (forward),
// the gradient operands and the wgrad partials (backward).  da3, da2 and da1 are adjacent, low twins included: one memset clears them.
// The learner's workspace (api.cu), the stand-alone encoder's two blocks (api.cu) and the test hook that names a row of those blocks
// (testhooks.cu) all carve this one table.
constexpr int ENC_SAVED_ROWS = 6, ENC_ROWS = 13;
inline int encoder_rows(EncoderBuffers& b, int64_t NF, int64_t NB, WsRow* t) {
  OperandTensors &hi = b.hi, &lo = b.lo;
  int n = 0;
  t[n++] = ws_row("xs", NF * 441 * 64, &b.xs);
  t[n++] = ws_row("a1", NF * 400 * 32, &hi.a1, &lo.a1);
  t[n++] = ws_row("a2", NF * 81 * 64, &hi.a2, &lo.a2);
  t[n++] = ws_row("a3", NF * 49 * 64, &hi.a3, &lo.a3);
  t[n++] = ws_row("h", NF * 512, &b.h);
  t[n++] = ws_row("wpack", WPack::TOTAL, &hi.wpack, &lo.wpack);
  t[n++] = ws_row(nullptr, FC_SPLITS * NF * 512, &b.hpart);
  t[n++] = ws_row("dh", NB * 512, &hi.dh, &lo.dh);
  t[n++] = ws_row("da3", NB * 81 * 64, &hi.da3, &lo.da3);      // da3g (9x9 grid)
  t[n++] = ws_row("da2", NB * 100 * 64, &hi.da2, &lo.da2);     // da2g (10x10 grid)
  t[n++] = ws_row("da1", NB * 441 * 32, &hi.da1, &lo.da1);     // da1g (21x21 grid, 32 channels)
  t[n++] = ws_row("wgrad_part", WSP_TOTAL, &b.wgrad_part);
  t[n++] = ws_row("a3t", NF * 49 * 64, &b.a3t);
  return n;
}
// tensor maps of the TMA kernels (built once per learner context: every operand buffer is fixed).
// Activations are [rows][64] bf16; "w" = window box (128 + max tap shift rows), "b" = 128-row box.
struct OperandMaps {      // the maps over one OperandTensors set
  alignas(64) CUtensorMap a1p0_w, a1p1_w, a2_w, da3g_w, da3g_b, da2g_w, da2g_b, da1g_b;      // conv layers (res_problems.cuh)
  alignas(64) CUtensorMap a3m128, a3m64, dhm128, dhm64;                                      // fc layer (tma_problems.cuh)
  alignas(64) CUtensorMap w1k, w2k, w3k, wfk, wfd, w3d, w2d;
};
struct TmaMaps {
  alignas(64) CUtensorMap xs_w;
  alignas(64) CUtensorMap a3tm64;       // a3 in fc.weight's native column order (c,h,w): fc wgrad's B operand
  OperandMaps hi, lo = {};              // lo: built only in the fp32-accurate mode
  bool valid = false;
};
// bf16 tensor map, dims innermost-first, strides in ELEMENTS for dims 1..rank-1, SWIZZLE_128B, zero OOB fill (encoder.cu)
bool make_map(CUtensorMap* m, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_elems, const uint32_t* box, bool swizzle64 = false);
// the maps of buf.hi, and of buf.lo when it is allocated.  Returns cudaSuccess or an error; `why` gets the name of the map that failed
cudaError_t build_tma_maps(const EncoderBuffers& buf, int NF, int NB, TmaMaps* maps, const char** why);
// wpack_lo != nullptr: also the low copies bf16(w - bf16(w)) in the same layouts
cudaError_t launch_a3_transpose(const __nv_bfloat16* a3, __nv_bfloat16* a3t, int frames, cudaStream_t st);
cudaError_t launch_pack_weights(const ParamPtrs& p, __nv_bfloat16* wpack, cudaStream_t st, __nv_bfloat16* wpack_lo = nullptr, bool skip_w1k = false);
// on S.main; joins the pack lane (the weight re-pack forked by the caller) before the first reader of the re-packed weights.
// mode: 0 = bf16 operands, 1 = fp32-accurate split operands (buf.lo and maps.lo must be built)
// fused_front: frame conversion + conv1 + conv2 in one kernel (enc_fused.cuh; bf16 mode)
cudaError_t encoder_forward(const uint8_t* obs, int frames, const ParamPtrs& p, const EncoderBuffers& buf, const TmaMaps& maps, int mode,
                            const StepStreams& S, bool fused_front);
// backward for the first `frames` frames given buf.hi.dh; accumulates into the (pre-zeroed) gradient tensors in `g`.  BWD_FC: the fc
// layer only (fc.weight / fc.bias gradients complete and joined to main on return: 95 % of the gradient bytes, ready for an early
// all-reduce); BWD_CONV: the conv layers only.  a3t_done: the caller already launched a3 -> buf.a3t on the fc_wgrad lane (bf16 mode)
enum BwdParts { BWD_FC = 1, BWD_CONV = 2, BWD_BOTH = BWD_FC | BWD_CONV };
cudaError_t encoder_backward(int frames, const EncoderBuffers& buf, const ParamPtrs& g, const TmaMaps& maps, int mode,
                             const StepStreams& S, BwdParts parts, bool a3t_done);
// ---- lstm.cu: the actor step of the 2-layer LSTM core (one row of B environments, no BPTT)
struct LstmStep;
// weights8: the 8 nn.LSTM tensors of the flat parameter buffer (srl_lstm_create order); H = 513 + A.  0, or an error code with the
// message set (errors.h)
int lstm_step_create(int B, int H, const float* const* weights8, LstmStep** out);
void lstm_step_destroy(LstmStep* S);
cudaError_t lstm_step_pack(LstmStep* S, cudaStream_t st);           // packed [W_ih | W_hh] bf16 copy of both layers from the fp32 parameters
bool lstm_step_ksplit_supported(int ks);                            // K split (cluster size) of the step GEMM: 1, 2, 3 or 6
constexpr int LSTM_STEP_KSPLIT = 3;                                 // default split (DESIGN.md §4: measured per N on H100)
// core f32 [B][H], done u8 [B], h_in/c_in f32 [2][B][H] -> h_out/c_out f32 [2][B][H]; uses the weights of the last lstm_step_pack
cudaError_t lstm_step_forward(LstmStep* S, const float* core, const uint8_t* done, const float* h_in, const float* c_in, float* h_out,
                              float* c_out, int ksplit, cudaStream_t st);
void lstm_step_buffers(const LstmStep* S, void** xh, int64_t* nxh, void** w, int64_t* nw);   // debug views of the bf16 operands
cudaError_t test_shift(const void* A, const void* B, float* D, int shift, int mn_major, int bo_mode, cudaStream_t st);
cudaError_t test_poison_smem(cudaStream_t st);
cudaError_t test_pdl(int* flag, int* out, int nblk, unsigned delay_ns, cudaStream_t st);

}  // namespace srl
