/* scalerl_b200 -- C ABI of the H100-native (sm_90a) IMPALA learner hot path.
 *
 * The reference (jianzhnie/ScaleRL) is 100 % Python and has no FFI; the interface these entry points
 * replace is the Python one of scalerl/algorithms/impala (file:line given per function).  A host
 * binds them with ctypes (see INTEGRATION.md and scalerl_b200/_lib.py).  Plain pointers and sizes
 * only -- no torch types.  Every pointer is a DEVICE pointer unless the name ends in `_host`.
 * `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).  Return value: 0 on
 * success, otherwise a cudaError_t (>0) or a negative SRL_E* argument error; srl_last_error()
 * returns the message of the calling thread's last failed call, whichever entry point it was.  Nothing here synchronises the stream.
 */
#ifndef SCALERL_B200_H_
#define SCALERL_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SRL_EINVAL (-1)   /* bad argument (shape / alignment / NULL) */
#define SRL_ESTATE (-2)   /* call order violated */

const char* srl_last_error(void);
int srl_version(void);

/* ---- V-trace -------------------------------------------------------------------------------------------
 * replaces vtrace.from_importance_weights (scalerl/algorithms/impala/vtrace.py:78-172).
 * log_rhos, discounts, rewards, values: f32 [T,B] row-major; bootstrap_value f32 [B]; outputs f32 [T,B].
 * clip thresholds < 0 mean None (no clipping), as the Python API's clip_*=None; a NaN threshold is refused (SRL_EINVAL).
 * variant: 0 = column-sequential (float4 over B when B%4==0), 1 = warp-shuffle affine scan over T. */
int srl_vtrace_from_importance_weights(const float* log_rhos, const float* discounts, const float* rewards,
                                       const float* values, const float* bootstrap_value, int T, int B,
                                       float clip_rho_threshold, float clip_pg_rho_threshold,
                                       float* vs, float* pg_advantages, int variant, void* stream);

/* replaces vtrace.from_logits (vtrace.py:43-75): logits f32 [T,B,A], actions i64 [T,B].
 * Outputs (any may be NULL except vs/pg): vs, pg_advantages, log_rhos, behavior_alp, target_alp, all f32 [T,B]. */
int srl_vtrace_from_logits(const float* behavior_policy_logits, const float* target_policy_logits,
                           const int64_t* actions, const float* discounts, const float* rewards,
                           const float* values, const float* bootstrap_value, int T, int B, int A,
                           float clip_rho_threshold, float clip_pg_rho_threshold,
                           float* vs, float* pg_advantages, float* log_rhos, float* behavior_action_log_probs,
                           float* target_action_log_probs, void* stream);

/* ---- fused learner tail: learn() pre-processing + V-trace + the three losses + head gradients ----------
 * replaces impala_atari.py:293-330 + loss_fn.py:5-23 + the autograd step from total_loss to
 * (policy_logits, baseline).  Inputs are the [T+1,B] batch rows as they lie in the trajectory batch
 * (impala_atari.py:122-151): the kernel applies the [1:] / [:-1] shifts itself.
 *   behavior_logits f32 [T+1,B,A] (batch['policy_logits']), target_logits f32 [T+1,B,A] and baseline f32 [T+1,B]
 *   (learner outputs), action i64 [T+1,B], reward f32 [T+1,B], done u8/bool [T+1,B].
 * Outputs: vs, pg_advantages f32 [T,B]; dlogits f32 [T,B,A]; dbaseline f32 [T,B];
 *   losses f32 [4] = {pg_loss, baseline_loss (x baseline_cost), entropy_loss (x entropy_cost), total}.
 * scratch: zero-initialised f32 [3*ceil(B/4)+4] workspace (block partials + ticket; re-armed by the kernel). */
int srl_impala_loss_and_head_grads(const float* behavior_logits, const float* target_logits, const float* baseline,
                                   const int64_t* action, const float* reward, const uint8_t* done,
                                   int T, int B, int A, float discounting, int reward_clip_abs_one,
                                   float clip_rho_threshold, float clip_pg_rho_threshold,
                                   float baseline_cost, float entropy_cost,
                                   float* vs, float* pg_advantages, float* dlogits, float* dbaseline,
                                   float* losses, float* scratch, void* stream);

/* ---- row-wise policy ops: the pieces of loss_fn.py / vtrace.action_log_probs as stand-alone, differentiable operators ------
 * (used by the autograd drop-ins scalerl_b200/algorithms/impala/{loss_fn,vtrace}.py; the learner step itself uses the fused tail)
 * forward : logp[n] = log_softmax(logits[n])[actions[n]] (vtrace.py:31-40; loss_fn.py:16-23), ent[n] = sum_a p log p (loss_fn.py:9-13);
 *           logits f32 [N,A], actions i64 [N]; either output may be NULL (actions may be NULL when logp is).
 * backward: dlogits[n][a] = w_logp[n] * (1{a == actions[n]} - p[a]) + w_ent[n] * p[a] * (log p[a] - ent[n]) -- the gradient of
 *           sum_n w_logp[n] logp[n] + w_ent[n] ent[n]; a NULL weight array means zeros.
 * srl_reduce_sum: out[0] = scale * sum x[i] (square = 0) or scale * sum x[i]^2 (square = 1), fixed summation order
 *           (loss_fn.py:5-6 compute_baseline_loss = 0.5 * sum(adv^2)). */
int srl_policy_rows_forward(const float* logits, const int64_t* actions, int64_t N, int A, float* logp, float* ent, void* stream);
int srl_policy_rows_backward(const float* logits, const int64_t* actions, const float* w_logp, const float* w_ent, int64_t N, int A,
                             float* dlogits, void* stream);
int srl_reduce_sum(const float* x, int64_t n, int square, float scale, float* out, void* stream);
/* actions[n] ~ softmax(logits[n]) through the inverse CDF of uniforms[n] in [0,1) (torch.multinomial of AtariNet.forward in training
 * mode, atari_model.py:130-132); uniforms == NULL: argmax (evaluation mode, :133-134).  logits f32 [N,A], actions i64 [N]. */
int srl_sample_actions(const float* logits, const float* uniforms, int64_t N, int A, int64_t* actions, void* stream);

/* ---- learner context: encoder fwd/bwd on wgmma + heads + optimizer ------------------------------------
 * replaces AtariNet.forward (scalerl/algorithms/utils/atari_model.py:77-143, use_lstm=False) and
 * ImpalaTrainer.learn (impala_atari.py:270-349) for one GPU's shard of the batch.                         */
typedef struct srl_learner srl_learner_t;

typedef struct srl_config {
  int32_t T;                 /* rollout_length                                   */
  int32_t B;                 /* batch columns processed by THIS GPU              */
  int32_t A;                 /* num_actions (<= 31)                              */
  int32_t optimizer;         /* 0 = RMSprop (reference, impala_atari.py:99-105), 1 = Adam */
  int32_t reward_clip_abs_one;
  int32_t precision;         /* encoder operand precision: 0 = bf16 (default, the measured configuration); 1 = fp32-accurate:
                              * every bf16 operand tensor gets a low twin bf16(v - bf16(v)) and each tensor-core product runs as
                              * hi*hi + hi*lo + lo*hi into the fp32 accumulator (16 significant operand bits, tighter than
                              * kind::tf32's 11) -- the whole-step parity mode SURVEY.md §7.9 asks for; ~3x the MMAs */
  float discounting, baseline_cost, entropy_cost;
  float clip_rho_threshold, clip_pg_rho_threshold;   /* < 0: None; NaN: refused */
  float max_grad_norm;       /* clip_grad_norm_ threshold (rl_args.py:108)       */
  float learning_rate, alpha, epsilon;               /* RMSprop (rl_args.py:112-117) */
  float adam_beta1, adam_beta2, adam_eps;
  int32_t use_lstm;          /* 1: AtariNet(use_lstm=True): 2-layer LSTM core between the encoder and the heads (config 5) */
} srl_config_t;

/* Number of fp32 elements of the flat parameter buffer for A actions, and the element offset / count of
 * each of the 12 AtariNet tensors in state_dict order (conv1.weight, conv1.bias, ..., baseline.bias),
 * PyTorch layouts.  Segments are padded to multiples of 4 floats. offsets/counts: int64[12], indexed in state_dict order;
 * in memory the small tensors come first and fc.weight last (offsets[6] is the largest), so [0, offsets[6]) is the
 * "small" gradient block and [offsets[6], total) is fc.weight. */
int64_t srl_param_layout(int A, int64_t* offsets, int64_t* counts);

/* Same with the 8 LSTM tensors (nn.LSTM state_dict order: weight_ih_l0, weight_hh_l0, bias_ih_l0, bias_hh_l0, *_l1) appended
 * after fc.weight when use_lstm != 0: offsets/counts are int64[20] (entries 12..19 = LSTM; unused when use_lstm == 0). */
int64_t srl_param_layout_ex(int A, int use_lstm, int64_t* offsets20, int64_t* counts20);

/* params / grads / opt_state0 / opt_state1: flat f32 device buffers of srl_param_layout() (srl_param_layout_ex() with use_lstm) elements, owned
 * by the caller (so torch can expose state_dict views and NCCL can all-reduce `grads` in place).
 * opt_state1 is only used by Adam (may be NULL for RMSprop). */
int srl_learner_create(const srl_config_t* cfg, float* params, float* grads, float* opt_state0, float* opt_state1,
                       srl_learner_t** out);
int srl_learner_destroy(srl_learner_t* L);
/* Diagnostics builds only (SRL_DEFINES=SRL_KSTAMP; tests/diag/diag_timeline.py): `buffer` = 1 + 3*2000 uint64 of device memory, zeroed by the
 * caller; every kernel then appends {kernel id, %globaltimer at entry, %globaltimer when its stream predecessor had completed} (word 0 = count).
 * NULL switches the stamps off.  The product build returns SRL_ESTATE. */
int srl_debug_kernel_timeline(void* buffer);
/* bytes of device workspace held by the context */
int64_t srl_learner_workspace_bytes(const srl_learner_t* L);
/* update a hyper-parameter that does not change buffer sizes (lr, costs, clip...) */
int srl_learner_set_config(srl_learner_t* L, const srl_config_t* cfg);

/* Learning-rate schedule of the optimizer step.  The lr of the 1-based optimizer step t (the device step count, so a replayed
 * CUDA graph follows the schedule and a restored step count resumes it):
 *   SRL_LR_CONSTANT: cfg.learning_rate (the default; frames_per_step and total_frames are not read)
 *   SRL_LR_LINEAR  : max(lr * (1 - min((t-1) * frames_per_step, total_frames) / total_frames), lr_end), evaluated in double and
 *                    rounded once to float.  lr_end = 0 is torchbeast's LambdaLR(1 - min(epoch*T*B, total)/total) stepped after each
 *                    optimizer step; lr_end > 0 is the floor of ScaleRL's LinearDecayScheduler (scalerl/utils/lr_scheduler.py:50-88).
 * frames_per_step: frames of one optimizer step over all ranks (T * B * world); total_frames: the frame budget of the run.
 * SRL_EINVAL: unknown kind, lr_end < 0, or (linear) frames_per_step <= 0 / total_frames <= 0.
 * After this call srl_learner_apply_gradients[_dp] write THREE floats to grad_norm_out: {norm, clip coefficient, lr of the step}.
 * Synchronous (writes the configured lr into the context's coefficient block).  The call affects launches issued after it: a
 * CUDA graph captured before it keeps the schedule it was captured with. */
#define SRL_LR_CONSTANT 0
#define SRL_LR_LINEAR 1
int srl_learner_set_lr_schedule(srl_learner_t* L, int kind, float lr_end, double frames_per_step, double total_frames);
/* RMSprop momentum (torch.optim.RMSprop(momentum=..., centered=False); reference impala_atari.py:99-105, rl_args.py:116):
 * v = alpha v + (1 - alpha) g^2;  buf = momentum buf + g / (sqrt(v) + eps);  p -= lr buf  (g: the clipped gradient).
 * momentum_buf: caller-owned flat f32 device buffer of the parameter layout (torch's 'momentum_buffer'), 16-byte aligned; zero it
 * before the first step.  momentum = 0 (buffer NULL or ignored) turns momentum off.  SRL_EINVAL: momentum < 0, momentum > 0
 * without a buffer or with Adam, a misaligned buffer.  Affects launches issued after the call; graphs captured before keep the
 * old setting. */
int srl_learner_set_momentum(srl_learner_t* L, float momentum, float* momentum_buf);

/* run-time switches of one learner context: "column_fusion" (default 1; 0 = three kernels head_fwd / impala_tail / head_bwd
 * instead of the fused column kernel -- the environment variable SRL_NO_COLUMN_FUSION is read once, at creation);
 * "fused_fwd" (default 0, SRL_FUSED_FWD=1): u8 frame conversion + conv1 + conv2 as ONE persistent kernel (bf16 mode) instead of three;
 * "lstm_step_ksplit" (1, 2, 3 or 6; default 3): thread-block cluster size over which srl_learner_forward_lstm_step splits K. */
int srl_learner_set_option(srl_learner_t* L, const char* name, int value);

/* optimizer step count (Adam's bias-correction t; torch.optim state['step']): restore it when resuming from a checkpoint
 * (host counter and the device-resident counter the captured graphs read).  Both synchronise `stream`. */
int srl_learner_set_step(srl_learner_t* L, int64_t step, void* stream);
int64_t srl_learner_get_step(srl_learner_t* L, void* stream);

/* re-derive the packed bf16 operand copies from the fp32 master parameters now (optional: every forward does it).  With
 * use_lstm it also packs the [W_ih | W_hh] copy that srl_learner_forward_lstm_step reads, which only this call writes. */
int srl_learner_pack_weights(srl_learner_t* L, void* stream);

/* AtariNet.forward for n_rows*B frames: obs u8 [rows,B,4,84,84], reward f32 [rows,B], action i64 [rows,B]
 * -> policy_logits f32 [rows,B,A], baseline f32 [rows,B].  rows <= T+1. */
int srl_learner_forward(srl_learner_t* L, const uint8_t* obs, const float* reward, const int64_t* action, int rows,
                        float* policy_logits, float* baseline, void* stream);

/* forward + V-trace + losses + full backward.  Leaves SUM-reduced gradients (loss_fn.py sums) in `grads`
 * and {pg, baseline, entropy, total} in losses[4]; vs/pg_advantages (f32 [T,B]) may be NULL. */
int srl_learner_forward_backward(srl_learner_t* L, const uint8_t* obs, const float* reward, const uint8_t* done,
                                 const int64_t* action, const float* behavior_logits,
                                 float* losses, float* vs, float* pg_advantages, void* stream);

/* use_lstm variants (SURVEY.md §8 row a17).  h0/c0: initial LSTM state f32 [2,B,513+A] (create_rnn_state_buffers,
 * impala_atari.py:108-120); rows of the forward must be T+1.  hT/cT (may be NULL) receive the state after the last row. */
int srl_learner_forward_lstm(srl_learner_t* L, const uint8_t* obs, const float* reward, const uint8_t* done, const int64_t* action,
                             const float* h0, const float* c0, float* policy_logits, float* baseline, float* hT, float* cT, void* stream);
int srl_learner_forward_backward_lstm(srl_learner_t* L, const uint8_t* obs, const float* reward, const uint8_t* done,
                                      const int64_t* action, const float* behavior_logits, const float* h0, const float* c0,
                                      float* losses, float* vs, float* pg_advantages, void* stream);

/* One actor step of AtariNet(use_lstm=True) for the context's B environments (atari_model.py:91-143 with T = 1):
 * obs u8 [B,4,84,84], reward f32 [B], done u8 [B], action i64 [B], h_in/c_in f32 [2,B,H] -> policy_logits f32 [B,A],
 * baseline f32 [B], h_out/c_out f32 [2,B,H] (must not alias h_in/c_in).  The state is reset by done before the step.
 * H = 513 + A.  The LSTM weights are those of the last srl_learner_pack_weights (load them, then pack: the step reads a
 * packed bf16 copy that no forward re-derives); the biases are read from the fp32 parameters at call time.  Bad pointers are
 * rejected (SRL_EINVAL) before the context is used; a context without use_lstm is rejected too.  bf16 operands only. */
int srl_learner_forward_lstm_step(srl_learner_t* L, const uint8_t* obs, const float* reward, const uint8_t* done,
                                  const int64_t* action, const float* h_in, const float* c_in, float* policy_logits,
                                  float* baseline, float* h_out, float* c_out, void* stream);

/* The same step in two halves, for overlapping the gradient all-reduce with the backward pass:
 *   _begin : forward + V-trace/loss + head backward + the fc layer's backward.  On return (in stream order) the
 *            fc.weight / fc.bias segments of `grads` (95 % of the bytes) are final -> start their all-reduce.
 *   _finish: conv3 / conv2 / conv1 backward; afterwards the remaining segments are final.
 * srl_learner_forward_backward == _begin followed by _finish. */
int srl_learner_forward_backward_begin(srl_learner_t* L, const uint8_t* obs, const float* reward, const uint8_t* done,
                                       const int64_t* action, const float* behavior_logits,
                                       float* losses, float* vs, float* pg_advantages, void* stream);
int srl_learner_backward_finish(srl_learner_t* L, const uint8_t* obs, void* stream);

/* clip_grad_norm_(max_grad_norm) over `grads` (after the caller's all-reduce, if any) + optimizer step.  A NaN gradient makes the
 * norm and the clip coefficient NaN and poisons every weight, as clip_grad_norm_ + step does (max_grad_norm < 0: no clip, coefficient 1).
 * grad_norm_out: f32 [2] = {total L2 norm, clip coefficient} (may be NULL); f32 [3] = {..., lr of the step} once
 * srl_learner_set_lr_schedule has been called.  The bf16 operand copies of the weights
 * are re-derived at the start of the next srl_learner_forward* call. */
int srl_learner_apply_gradients(srl_learner_t* L, float* grad_norm_out, void* stream);

/* Data-parallel apply step over peer memory, replacing ncclAllReduce + srl_learner_apply_gradients (impala_atari.py:344-346
 * on every rank): reduce-scatter of the flat gradient through NVLink loads, global-norm clip, optimizer and all-gather in ONE
 * cooperative kernel (see optim.cu).  grads[i] / exchange[i] / ctl[i] (i < world) are rank i's gradient buffer, its
 * exchange buffer (4 * ceil(n/4 / world) + 4 floats: the reduced slice the peers pull) and its 1 KiB control block, all
 * mapped into this process (symmetric memory / CUDA IPC); grads[rank] must be the buffer given to srl_learner_create; the
 * control blocks start zeroed.  Every rank must call it once per step.  On return (stream order) the
 * local gradient buffer holds the SUM over ranks, as after ncclAllReduce. */
typedef struct {
  void* grads[8]; void* exchange[8]; void* ctl[8]; int rank; int world;
  void* grads_multicast;   /* NVLS multicast address of the gradient buffers (NULL: peer loads).  When set, the reduce-scatter is one
                            * multimem.ld_reduce per 16 bytes (the NVSwitch adds the copies) and the all-gather one multimem.st */
} srl_dp_peers_t;
int srl_learner_apply_gradients_dp(srl_learner_t* L, const srl_dp_peers_t* peers, float* grad_norm_and_coef_out, void* stream);

/* Weight-publish snapshot (impala_atari.py:348, actor_model.load_state_dict(learner_model.state_dict())): copies the flat fp32
 * parameters to `dst` (same layout, srl_param_layout elements) on `stream` -- unless losses[3] (the step's total loss, device
 * f32[4]; may be NULL = unconditional) is NaN/Inf, in which case `dst` keeps the last good weights (every finite loss copies).  The caller then copies
 * `dst` to the actors' host memory asynchronously while the next step already updates the live parameters. */
int srl_learner_snapshot_params(srl_learner_t* L, float* dst, const float* losses, void* stream);

/* borrow internal activations / operand copies for tests: name in {"xs","a1","a2","a3","a3t","h","logits","baseline",
 * "dlogits","dbaseline","dh","da3","da2","da1","wpack"}; returns device pointer + element count.  The fp32-accurate operand mode
 * (precision = 1) adds the low twins "a1_lo","a2_lo","a3_lo","dh_lo","da3_lo","da2_lo","da1_lo","wpack_lo" (SRL_ESTATE in the
 * bf16 mode).  h, logits, baseline, dlogits and dbaseline are f32, the rest bf16.  use_lstm contexts add the
 * actor step's bf16 operands: "lstm_step_xh" [2][B][2Hp] (per layer [x | m.h] of the last step, Hp = 576) and "lstm_step_w"
 * [2][4Hp][2Hp] (per layer [W_ih | W_hh], rows interleaved so one 128-row tile holds the 4 gates of 32 units; csrc/lstm.cu). */
int srl_learner_debug_buffer(srl_learner_t* L, const char* name, void** ptr, int64_t* count);

/* per-kernel timing of one learner step: when enabled every kernel launch of forward_backward /
 * apply_gradients is bracketed by cudaEventRecord on the caller's stream; profile_collect() synchronises
 * on those events and writes milliseconds per slot (-1 for slots not executed) to a HOST array of
 * srl_profile_slot_count() floats. */
int srl_learner_set_profiling(srl_learner_t* L, int enable);
int srl_profile_slot_count(void);
const char* srl_profile_slot_name(int slot);
int srl_learner_profile_collect(srl_learner_t* L, float* ms_out_host);

/* pin / unpin caller-owned HOST memory (trajectory ring slots: the pageable torch.stack + .to(device) of impala_atari.py:248-265
 * becomes direct DMA; actor parameters in shared memory: the target of the weight publish, impala_atari.py:348).  Registering a
 * range that a stale or enclosing registration already covers succeeds. */
int srl_host_register(void* ptr_host, int64_t bytes);
int srl_host_unregister(void* ptr_host);

/* asynchronous device-to-device copy on `stream` (used by tests to read the borrowed buffers) */
int srl_memcpy_d2d(void* dst, const void* src, int64_t bytes, void* stream);

/* ---- stand-alone encoder: the trainable AtariNet's conv/fc stack under autograd --------------------------------------------
 * replaces atari_model.py:91-107 (obs -> /255 -> conv1..3 -> fc -> ReLU -> [h, clamp(reward,-1,1), one_hot(action)]) and its
 * autograd; the LSTM core and the heads stay with the caller (scalerl_b200.algorithms.utils.atari_model.AtariNet).  The kernels
 * and the stream lanes are the learner's; every activation lives in two caller-owned blocks, so each forward keeps its own:
 *   saved   : written by the forward, read by its backward (activations + the packed weights the forward ran with);
 *   scratch : one call's temporaries (forward and backward alike; its contents do not outlive the call).
 * srl_encoder_sizes gives both blocks' bytes for a frame count and precision (0 = bf16 operands, 1 = fp32-accurate split operands, as
 * srl_config_t.precision).  Both blocks are 256-byte aligned, need no initialisation and must not overlap each other or any other argument.
 * A context holds only the lanes, their events and the precision: one per device, created on that device. */
typedef struct srl_encoder srl_encoder_t;
int srl_encoder_create(int precision, srl_encoder_t** out);
int srl_encoder_destroy(srl_encoder_t* E);
int srl_encoder_sizes(int frames, int precision, int64_t* saved_bytes, int64_t* scratch_bytes);
/* forward for `frames` <= 65536 frames: obs u8 [frames,4,84,84], reward f32 [frames], action i64 [frames] (clamped to [0,A)),
 * weights8 = {conv1.weight, conv1.bias, conv2.weight, conv2.bias, conv3.weight, conv3.bias, fc.weight, fc.bias} (f32, PyTorch layouts,
 * 16-byte aligned) -> core_out f32 [frames, 513+A] = [h (512), clamp(reward,-1,1), one_hot(action) (A)]. */
int srl_encoder_forward(srl_encoder_t* E, const uint8_t* obs, const float* reward, const int64_t* action, int frames, int A,
                        const float* const* weights8, void* saved, void* scratch, float* core_out, void* stream);
/* backward of the forward that filled `saved` (same frames, A and context precision): dcore f32 [frames, 513+A] (columns >= 512 are
 * not read) -> the 8 gradients of weights8's tensors, PyTorch layouts, 16-byte aligned, OVERWRITTEN (not accumulated). */
int srl_encoder_backward(srl_encoder_t* E, const float* dcore, int frames, int A, void* saved, void* scratch, float* const* grads8,
                         void* stream);

/* ---- LSTM core (AtariNet use_lstm=True; atari_model.py:52-55,109-120; SURVEY.md §8 row a17) -------------------------------
 * 2-layer LSTM(H, H), H = 513 + A, stepped with the state multiplied by (1 - done_t) before every step.
 * weights8 / grads8: 8 device pointers in nn.LSTM state_dict order {weight_ih_l0 [4H,H], weight_hh_l0 [4H,H], bias_ih_l0 [4H],
 * bias_hh_l0 [4H], *_l1 ...} (fp32, caller-owned); gradients are ACCUMULATED into grads8 (zero them before the step).
 * forward : core f32 [T1,B,H], done u8 [T1,B], h0/c0 f32 [2,B,H] -> out f32 [T1,B,H], hT/cT f32 [2,B,H] (may be NULL)
 * backward: dout f32 [T1-1,B,H] (rows 0..T1-2 only: the learner's bootstrap row T1-1 carries no gradient) -> dcore f32 [T1-1,B,H].
 *           The bias gradients are reduced without atomics (fixed 64-row chunks added in order): the same bits on every run.
 * Errors of these calls and of srl_lstm_core_* are reported by srl_last_error, as every other call's; srl_lstm_last_error returns
 * the same message (kept for existing hosts). */
typedef struct srl_lstm srl_lstm_t;
int srl_lstm_create(int T1, int B, int H, const float* const* weights8, float* const* grads8, srl_lstm_t** out);
int srl_lstm_destroy(srl_lstm_t* L);
int srl_lstm_forward(srl_lstm_t* L, const float* core, const uint8_t* done, const float* h0, const float* c0, float* out,
                     float* hT, float* cT, void* stream);
int srl_lstm_backward(srl_lstm_t* L, const float* dout, const uint8_t* done, float* dcore, void* stream);
const char* srl_lstm_last_error(void);
/* Address and element count of one of the context's device rows (tests only; no CUDA call), named as srl_lstm_core_debug_buffer's.
 * The backward covers the first (T1-1)*B rows, so "dgates" and "dx" have that many; "done" is unused (the caller passes its own). */
int srl_lstm_debug_buffer(srl_lstm_t* L, const char* name, int layer, void** ptr, int64_t* count);

/* ---- stand-alone LSTM core: the trainable AtariNet's use_lstm=True core under autograd ---------------------------------------
 * The same kernels as srl_lstm_*, on two caller-owned blocks as srl_encoder_*: `saved` is written by the forward and read by its
 * backward (layer inputs, m.h, h, gate activations, cell states, the packed weights the forward ran with, copies of done and of the
 * padded initial cell state); `scratch` holds one call's temporaries.  No context: tensor maps are encoded on the host per call
 * (legal under stream capture) on the current device.  H = 513 + A, A in [1, 31], 1 <= T1*B <= 65536 (T1 = 1 is one step).
 * Both blocks are 256-byte aligned, need no initialisation, and no output may overlap another argument.  Everything runs on `stream`.
 * forward : core f32 [T1,B,H], done u8 [T1,B], h0/c0 f32 [2,B,H], weights8 (srl_lstm_create order) -> out f32 [T1,B,H],
 *           hT/cT f32 [2,B,H] (the state after row T1-1).
 * backward: dout f32 [T1,B,H] (every row, the last included), dhT/dcT f32 [2,B,H] (gradients of hT/cT; NULL = zero)
 *           -> grads8 (the 8 tensors' gradients, OVERWRITTEN), dcore f32 [T1,B,H], dh0/dc0 f32 [2,B,H] (gradients of h0/c0; NULL = not
 *           wanted, which skips their extra GEMM).
 * debug_buffer (tests only; host arithmetic, no CUDA call): address and element count of one row of the blocks of a call with the same
 * T1, B, A.  Hp = H rounded up to 64, G = 4Hp, N1 = T1*B; per-layer rows take layer 0 or 1, every other row layer 0.
 *   saved:   "xin0" bf16 [N1][Hp] (layer 0's input; layer 1's is hbf of layer 0), per layer "hm" bf16 [N1][Hp] (m_t . h_{t-1}),
 *            "hbf" bf16 [N1][Hp] (h_t), "Wih"/"Whh" bf16 [4][Hp][Hp] (gate-major, zero padded), "WihT"/"WhhT" bf16 [Hp][G] (transposes),
 *            "gates" f32 [N1][4][Hp] (activations i, f, g, o), "cseq" f32 [N1][Hp] (c_t); "c_init" f32 [2][B][Hp] (columns [H, Hp) are
 *            never written), "done" u8 [N1].
 *   scratch: "gx" f32 [N1][G], "r" f32 [B][G], per layer "hseq" f32 [N1][Hp], "dgates" bf16 [N1][G]; "dx" f32 [N1][Hp],
 *            "dwpad" f32 [G][Hp], "dc"/"dhm" f32 [B][Hp], "bias_part" f32 [ceil(N1/64)][G].  After a backward, dgates of each layer and
 *            (layer 0's input gradient, padded) dx hold its results; the rest are the last step's temporaries. */
int srl_lstm_core_debug_buffer(int T1, int B, int A, void* saved, void* scratch, const char* name, int layer, void** ptr,
                               int64_t* count);
int srl_lstm_core_sizes(int T1, int B, int A, int64_t* saved_bytes, int64_t* scratch_bytes);
int srl_lstm_core_forward(const float* core, const uint8_t* done, const float* h0, const float* c0, int A, int T1, int B,
                          const float* const* weights8, void* saved, void* scratch, float* out, float* hT, float* cT, void* stream);
int srl_lstm_core_backward(const float* dout, const float* dhT, const float* dcT, int A, int T1, int B, void* saved, void* scratch,
                           float* const* grads8, float* dcore, float* dh0, float* dc0, void* stream);

/* ---- prioritized-replay sampler (BASELINE.json configs[3]; SURVEY.md §8f) ---------------------------------------------------
 * Device-resident float64 sum/min segment trees; replaces PrioritizedReplayBuffer's tree arithmetic
 * (scalerl/data/replay_buffer.py:305-381 over scalerl/data/segment_tree.py:7-196).  Index results are identical to the
 * reference's Python-float trees given identical leaf values.  srl_replay_* below stores transitions over such trees.
 * Errors are reported by srl_last_error; srl_per_last_error returns the same message (kept for existing hosts). */
typedef struct srl_per srl_per_t;
int srl_per_create(int64_t memory_size, double alpha, srl_per_t** out);
int srl_per_destroy(srl_per_t* P);
int64_t srl_per_size(const srl_per_t* P);
int64_t srl_per_capacity(const srl_per_t* P);
int srl_per_add(srl_per_t* P, int64_t n, void* stream);                                  /* _add x n  (replay_buffer.py:318-322) */
int srl_per_update_priorities(srl_per_t* P, const int64_t* idxs, const double* priorities, int64_t n, void* stream);   /* :346-351 */
/* pairs skipped so far by srl_per_update_priorities because idx was outside [0, size) or priority <= 0 (the reference asserts
 * both, replay_buffer.py:346-351), plus the non-finite priorities srl_replay_add_prioritized stored as max_priority^alpha;
 * synchronises `stream`; -1 on error */
int64_t srl_per_invalid_updates(srl_per_t* P, void* stream);
int srl_per_sample(srl_per_t* P, const double* uniforms, int batch, double beta, int64_t* idxs, double* weights64,
                   float* weights32, void* stream);                                      /* :353-381, uniforms f64 [batch] in [0,1) */
int srl_per_debug_trees(srl_per_t* P, double* sum_out, double* min_out, double* max_priority_out, void* stream);
const char* srl_per_last_error(void);
/* The stored count is also kept on the device, written by the add kernel: srl_per_sample and srl_per_update_priorities read it when
 * their kernels run, so a captured sample or update sees every add made before the graph replays. */

/* ---- prioritized replay memory: n-step transitions on the device, sampled and gathered there -------------------------------
 * PrioritizedReplayBuffer (scalerl/data/replay_buffer.py:132-381) with its storage on the GPU: a ring of memory_size transitions,
 * state / next_state u8 [M,4,84,84], action i64 [M], reward f32 [M], done u8 [M], whose slot i is leaf i of the memory's own sampler
 * (srl_replay_per).  An n_step-deep window of raw vector steps per env folds into n-step transitions as _get_n_step_info does
 * (:230-273): state and action of the oldest step, reward r0 + r1*g1 + r2*g2 ... in fp32 (g_k = fp32(gamma^k) in double, every product
 * and sum rounded separately), stopping at the first done, whose step gives next_state and done.  Every call is stream-ordered. */
typedef struct srl_replay srl_replay_t;
/* memory_size in [2, 2^30], num_envs in [1, min(65536, memory_size)], n_step in [1, 32], gamma finite, alpha the trees' exponent.
 * Allocates memory_size * 56,461 B plus the window (a failed allocation names the bytes asked for).  Synchronous. */
int srl_replay_create(int64_t memory_size, int num_envs, int n_step, double gamma, double alpha, srl_replay_t** out);
int srl_replay_destroy(srl_replay_t* R);
int64_t srl_replay_size(const srl_replay_t* R);         /* stored transitions (len of the reference's memory) */
srl_per_t* srl_replay_per(srl_replay_t* R);              /* its trees: srl_apex_learner_step's `per`, srl_per_update_priorities */
/* one vector env step of num_envs envs: state / next_state u8 [E,4,84,84], action i64 [E], reward f32 [E], done u8 [E] (device or host
 * memory, copied on `stream`).  Once n_step steps are staged, E transitions enter the ring at slots (ptr + e) mod memory_size in env
 * order (replay_buffer.py:197-218, 319-323) with priority max_priority^alpha. */
int srl_replay_add(srl_replay_t* R, const uint8_t* state, const int64_t* action, const float* reward, const uint8_t* next_state,
                   const uint8_t* done, void* stream);
/* srl_per_sample with beta read from the device (beta_dev f64 [1], so a replayed graph sees every change), then srl_replay_gather of the
 * sampled idxs: uniforms f64 [batch] in [0,1), outputs state / next_state u8 [batch,4,84,84] (16-byte aligned), action i64, reward f32,
 * done u8, idxs i64, weights f32 [batch] (may be NULL).  Needs size >= 2 when called; no host synchronisation, capturable. */
int srl_replay_sample(srl_replay_t* R, const double* uniforms, int batch, const double* beta_dev, uint8_t* state, int64_t* action,
                      float* reward, uint8_t* next_state, uint8_t* done, int64_t* idxs, float* weights, void* stream);
/* copies ring slots idxs i64 [n] (device) into the outputs, as srl_replay_sample's; a slot outside [0, memory_size) leaves its rows */
int srl_replay_gather(srl_replay_t* R, const int64_t* idxs, int64_t n, uint8_t* state, int64_t* action, float* reward, uint8_t* next_state,
                      uint8_t* done, void* stream);

/* ---- frame replay memory: srl_replay_* with each 84x84 frame stored once -------------------------------------------------------
 * The transitions, fold, trees, sampling and outputs of srl_replay_*, bit for bit for the same adds, with the frame stacks kept as
 * handles into a FIFO pool of frame_capacity u8 [84,84] frames (frame of 64-bit sequence number s at s mod frame_capacity).  An add
 * compares each env's 8 incoming frames (state 0..3, next_state 0..3) byte for byte with the env's earlier frames of the call and with
 * its previous next_state frames, reuses the sequence number of an equal one and numbers the rest in env order; an Atari stream that
 * continues an episode adds one frame per env step.  Frames it overwrites retire every ring slot that references them: a retired slot
 * has sum-tree leaf 0 and min-tree leaf +inf (never sampled, outside p_min), leaves the gather's output rows as they were, is skipped by
 * srl_per_update_priorities without counting as invalid, and lives again when an add writes its slot.  It only saves memory when the
 * stacks of the stream share frames.  Every call is stream-ordered. */
typedef struct srl_frame_replay srl_frame_replay_t;
/* srl_replay_create's arguments and limits, and frame_capacity in [8 num_envs (n_step + 1), 2^32] frames (the lower bound keeps the
 * staging window's frames from being overwritten; memory_size + memory_size / 8 + 8 num_envs (n_step + 4) retires nothing while
 * episodes average 32 steps or more).  Allocates frame_capacity * 7,056 B plus 94 B per slot and the window.  Synchronous. */
int srl_frame_replay_create(int64_t memory_size, int num_envs, int n_step, double gamma, double alpha, int64_t frame_capacity,
                            srl_frame_replay_t** out);
int srl_frame_replay_destroy(srl_frame_replay_t* R);
int64_t srl_frame_replay_size(const srl_frame_replay_t* R);   /* slots written, retired ones included (len of the reference's memory) */
srl_per_t* srl_frame_replay_per(srl_frame_replay_t* R);        /* its trees, with the retired mask attached */
/* srl_replay_add: state / next_state u8 [E,4,84,84] (device or host memory, copied on `stream`), action i64, reward f32, done u8 [E] */
int srl_frame_replay_add(srl_frame_replay_t* R, const uint8_t* state, const int64_t* action, const float* reward, const uint8_t* next_state,
                         const uint8_t* done, void* stream);
/* srl_replay_sample and srl_replay_gather, each stack rebuilt from its 4 frames; a retired slot leaves its rows as they were */
int srl_frame_replay_sample(srl_frame_replay_t* R, const double* uniforms, int batch, const double* beta_dev, uint8_t* state, int64_t* action,
                            float* reward, uint8_t* next_state, uint8_t* done, int64_t* idxs, float* weights, void* stream);
int srl_frame_replay_gather(srl_frame_replay_t* R, const int64_t* idxs, int64_t n, uint8_t* state, int64_t* action, float* reward,
                            uint8_t* next_state, uint8_t* done, void* stream);
/* frames written to the pool since creation, and slots retired since creation; each synchronises `stream`; -1 on error */
int64_t srl_frame_replay_frames_allocated(srl_frame_replay_t* R, void* stream);
int64_t srl_frame_replay_retired(srl_frame_replay_t* R, void* stream);

/* ---- Ape-X learner step: a prioritized (double) DQN update on the encoder (BASELINE.json configs[3]) --------------------------
 * replaces the learner statements of the reference's Ape-X Learner.train (scalerl/algorithms/apex/worker.py:134-161) and, with
 * double DQN, clipping and the target cadence, DQNAgent.learn (scalerl/algorithms/dqn/dqn_agent.py:136-190).  The Q network is
 * Nature DQN: AtariNet's conv1..3 + fc + ReLU (atari_model.py:30-47,91-101) followed by q = Linear(512, A), A in [1, 31], or, with
 * `dueling`, the dueling head of Wang et al. 2016 (eq. 9) on the same 512 fc features: V = value(h) = Linear(512, 1), Adv =
 * advantage(h) = Linear(512, A), Q = V + Adv - mean_a Adv.  Both heads read the shared fc output (the paper's Atari network has two
 * separate 512-unit fc streams): the encoder is the same for both.  With `num_atoms` = K > 0 the head is categorical (C51,
 * Bellemare et al. 2017): q = Linear(512, A K), row a K + k atom k of action a, p(s)[a] = softmax over the action's K logits, Q(s, a) =
 * sum_k z_k p_k on the support z_k = v_min + k dz, dz = (v_max - v_min) / (K - 1) rounded once to fp32.  With `num_quantiles` = N > 0
 * the head is the quantile head (QR-DQN, Dabney et al. 2018): q = Linear(512, A N), row a N + i quantile i of action a at the midpoint
 * tau^_i = (2 i + 1) / (2 N), Q(s, a) = (sum_i theta_{a,i}) / N.  With `dist_dueling` = 1 either of these heads is Rainbow's dueling
 * head per atom or quantile (Hessel et al. 2018), W = K or N rows per action: v = value(h) = Linear(512, W), adv = advantage(h) =
 * Linear(512, A W), rows[a W + k] = (v[k] + adv[a W + k]) - (1/A) sum_a' adv[a' W + k], the advantage mean summed over a' in order and
 * divided once.  The step composes W_eff and b_eff of these rows from value and advantage (online and target, from the parameters as they
 * are when it runs), runs the categorical or quantile update on them unchanged, and splits the rows' gradients back into g_v[k] =
 * sum_a g[a W + k] and g_adv[a W + k] = g[a W + k] - (1/A) sum_a' g[a' W + k].
 * srl_replay_* stores and folds n-step transitions (pass gamma^n for them, and srl_replay_per as `per`); srl_apex_actor_* acts and computes
 * their initial priorities.
 * Parameters in state_dict order {conv1.weight, conv1.bias, conv2.weight, conv2.bias, conv3.weight, conv3.bias, fc.weight, fc.bias,
 * q.weight [A,512], q.bias [A]}; srl_apex_param_layout returns the flat buffer's floats and each tensor's offset / count (int64[10]).
 * The dueling head's state_dict order is {conv1..3, fc, value.weight [1,512], value.bias [1], advantage.weight [A,512],
 * advantage.bias [A]} (int64[12], srl_apex_param_layout_ex); value.weight lies directly before advantage.weight.
 * The categorical head keeps the 10 plain names with q.weight [A K, 512] and q.bias [A K] (srl_apex_param_layout_cat), and so does the
 * quantile head with q.weight [A N, 512] and q.bias [A N] (srl_apex_param_layout_quantile).  The distributional dueling head has the
 * dueling head's 12 names with value [W, 512], [W] and advantage [A W, 512], [A W] (srl_apex_param_layout_dist_dueling).
 * Every head, with or without noise, has one layout rule (srl_apex_param_layout_noisy's): in memory, each segment padded to 4
 * floats, come the conv tensors, fc's bias, the head weights and the head biases (noisy: the head biases first), then fc's weight,
 * each group by (mu before sigma, layer).  Params, grads, both Adam states and the target copy share the layout. */
typedef struct srl_apex_learner srl_apex_learner_t;
typedef struct srl_apex_config {
  int32_t B;                 /* transitions per step, 1 <= B <= 65536                                        */
  int32_t A;                 /* actions, [1, 31]                                                             */
  int32_t precision;         /* encoder operands, as srl_config_t.precision: 0 = bf16, 1 = fp32-accurate split */
  int32_t double_dqn;        /* 1: a* = argmax of the online network at s' (dqn_agent.py:155-160)              */
  float gamma;               /* discount (gamma^n for n-step transitions)                                    */
  float max_grad_norm;       /* clip_grad_norm_ threshold (dqn_agent.py:178-181), > 0; +inf: no clip (coef 1) */
  float learning_rate, adam_beta1, adam_beta2, adam_eps;   /* torch.optim.Adam (apex/worker.py:132)            */
  float priority_eps;        /* priority = |q - y| + priority_eps (in double), >= 0                           */
  int32_t dueling;           /* 0: q = Linear(512, A); 1: the dueling head Q = V + Adv - mean(Adv)             */
  int32_t num_atoms;         /* 0: a scalar Q head; K in [2, 64]: the categorical head (not with dueling = 1)  */
  float v_min, v_max;        /* the categorical support [v_min, v_max], finite, v_min < v_max (read when num_atoms > 0) */
  int32_t noisy;             /* 0: plain layers; 1: noisy fc and head layers (srl_apex_param_layout_noisy)        */
  uint64_t noise_seed;       /* the Philox key of the noise (read when noisy = 1)                                */
  int32_t num_quantiles;     /* 0: no quantile head; N in [2, 256]: the quantile head (not with dueling = 1 or num_atoms > 0) */
  float kappa;               /* the quantile Huber threshold, finite and > 0 (read when num_quantiles > 0; QR-DQN-1: 1)      */
  int32_t dist_dueling;      /* 0; 1: the categorical or quantile head as dueling rows (not with dueling = 1)             */
} srl_apex_config_t;
int64_t srl_apex_param_layout(int A, int64_t* offsets10, int64_t* counts10);
/* the layout of either head: dueling 0 -> 10 tensors (srl_apex_param_layout's), 1 -> 12; -1 with srl_last_error set for A outside
 * [1, 31] or dueling outside {0, 1} */
int64_t srl_apex_param_layout_ex(int A, int dueling, int64_t* offsets12, int64_t* counts12);
/* the 10-tensor layout with q.weight [A num_atoms, 512] and q.bias [A num_atoms] (num_atoms 0: srl_apex_param_layout's); -1 with
 * srl_last_error set for A outside [1, 31] or num_atoms outside {0} and [2, 64] */
int64_t srl_apex_param_layout_cat(int A, int num_atoms, int64_t* offsets10, int64_t* counts10);
/* The layout of every head, with or without noisy networks (Fortunato et al. 2018, factorised Gaussian noise): noisy = 0 gives
 * srl_apex_param_layout_ex / _cat's (dueling and num_atoms > 0 together are refused); noisy = 1 replaces fc and each head layer
 * <l> by <l>.weight_mu, <l>.weight_sigma, <l>.bias_mu, <l>.bias_sigma in that order: {conv1..3 (6), fc (4), q (4)} = 14 tensors,
 * or {conv1..3, fc, value (4), advantage (4)} = 18 with the dueling head.  Each noisy layer computes
 *   y = (mu_w + sigma_w (.) eps_w) x + mu_b + sigma_b (.) eps_b,  eps_w = f(eps_out) f(eps_in)^T,  eps_b = f(eps_out),  f(x) = sgn(x) sqrt|x|
 * In memory the biases come first, then the head weights (value.weight_mu directly before advantage.weight_mu, and the same for
 * sigma), then fc.weight_mu and fc.weight_sigma, as the rule above.  -> the buffer's floats, or -1 with srl_last_error set */
int64_t srl_apex_param_layout_noisy(int A, int dueling, int num_atoms, int noisy, int64_t* offsets18, int64_t* counts18);
/* The layout of every head: srl_apex_param_layout_noisy's with num_quantiles = N in [2, 256] for the quantile head (q.weight [A N, 512],
 * q.bias [A N]; not with dueling = 1 or num_atoms > 0), 0 for the others.  -> the buffer's floats, or -1 with srl_last_error set */
int64_t srl_apex_param_layout_quantile(int A, int dueling, int num_atoms, int num_quantiles, int noisy, int64_t* offsets18,
                                       int64_t* counts18);
/* The layout of every head: srl_apex_param_layout_quantile's with dist_dueling = 1 for the distributional dueling head (num_atoms > 0
 * or num_quantiles > 0, not dueling = 1): value [W, 512] and advantage [A W, 512] with their biases in the dueling head's places, so
 * value.weight lies directly before advantage.weight (noisy: the mu rows, and the sigma rows).  -> the buffer's floats, or -1 with
 * srl_last_error set */
int64_t srl_apex_param_layout_dist_dueling(int A, int dueling, int num_atoms, int num_quantiles, int dist_dueling, int noisy,
                                           int64_t* offsets18, int64_t* counts18);
/* params / grads / exp_avg / exp_avg_sq / target_params: caller-owned flat f32 device buffers of srl_apex_param_layout floats,
 * 16-byte aligned and disjoint.  The context owns the encoder's blocks (one saved block for the forward over s, one for the
 * forwards over s', their scratch) and the tail's buffers.  Synchronous. */
int srl_apex_learner_create(const srl_apex_config_t* cfg, float* params, float* grads, float* exp_avg, float* exp_avg_sq,
                            float* target_params, srl_apex_learner_t** out);
int srl_apex_learner_destroy(srl_apex_learner_t* L);
/* One learner step on B transitions (apex/memory.py:7-8): obs / next_obs u8 [B,4,84,84], action i64 [B], reward f32 [B],
 * done u8/bool [B], weights f32 [B] (importance weights; NULL = 1), idxs i64 [B] with per (both NULL, or both set).
 *   q = Q(s)[a];  y = r + gamma Q_t(s')[a*] (1 - d), a* = argmax Q_t(s') or, double_dqn, argmax Q(s')   (worker.py:148-150)
 *   loss = mean(w (q - y)^2)                                                                             (worker.py:156-157)
 *   priority = |q - y| + priority_eps from the pre-update weights -> the sampler's trees, last occurrence of an idx wins (:152-154)
 * The categorical head (num_atoms = K > 0) replaces the squared TD error by the distributional update of Bellemare et al. 2017:
 *   a* as above on the expected Q;  m = the projection of p_t(s')[a*] moved to clamp(r + gamma (1 - d) z_j, v_min, v_max) onto the
 *   support (Algorithm 1, j ascending);  ce = -sum_k m_k log p(s)[a, k];  loss = mean(w ce);  priority = max(KL(m || p(s)[a]), 0) +
 *   priority_eps (Hessel et al. 2018).  q holds sum_k z_k p(s)[a, k], y holds sum_k z_k m_k.
 * The quantile head (num_quantiles = N > 0) replaces it by the quantile Huber loss of Dabney et al. 2018 (eq. 10):
 *   a* as above on Q = mean_i theta_i;  T_j = r + gamma theta_t(s')[a*, j] (T_j = r when d = 1 or gamma = 0: s' is not read);
 *   u_ij = T_j - theta(s)[a, i];  rho_ij = |tau^_i - 1{u_ij < 0}| L_kappa(u_ij) / kappa, L_kappa the Huber loss;  loss_n = (1 / N)
 *   sum_i sum_j rho_ij;  loss = mean(w loss_n);  priority = loss_n + priority_eps.  q holds Q(s, a), y holds mean_j T_j.
 *   clip_grad_norm_(max_grad_norm), torch.optim.Adam step with the step count kept on the device       (dqn_agent.py:172-182)
 * With noisy = 1 update k (the device step count before the update) first draws the noise of both networks: standard normals from
 * Philox4x32-10 keyed by noise_seed, counted by (k, network), Box-Muller.  The online network's one draw per layer serves Q(s) and the
 * double-DQN choice at s'; the target network's draw is independent.  The step runs on the composed weights mu + sigma (.) eps; their
 * gradients are the mu gradients, and the sigma gradients are dW (.) eps and db (.) f(eps_out), before the clip and Adam.
 * stats_out: f32 [3] device = {loss, gradient norm, clip coefficient} (may be NULL).  No host synchronisation; capturable. */
int srl_apex_learner_step(srl_apex_learner_t* L, const uint8_t* obs, const int64_t* action, const float* reward, const uint8_t* next_obs,
                          const uint8_t* done, const float* weights, const int64_t* idxs, srl_per_t* per, float* stats_out, void* stream);
/* target_params = tau * params + (1 - tau) * target_params, each product and the sum rounded separately (soft_target_update,
 * utils/model_utils.py:29-32; dqn_agent.py:185-190): tau = 1 copies exactly.  tau in [0, 1]. */
int srl_apex_learner_update_target(srl_apex_learner_t* L, float tau, void* stream);
/* Adam's step count (torch.optim state['step']) for a resumed run: writes the device counter; synchronises `stream` */
int srl_apex_learner_set_step(srl_apex_learner_t* L, int64_t step, void* stream);
/* Q(obs) with the online parameters for n >= 1 frames: obs u8 [n,4,84,84] -> q_out f32 [n,A] (predict / get_action).  Runs on its own
 * encoder context and blocks, so it may run on another stream than srl_apex_learner_step without touching the step's buffers; it reads
 * the parameters as they are when it runs (order it with the step on one stream for a given parameter version).  Calls of it on two
 * streams at once share its blocks and must be ordered. */
int srl_apex_learner_q_values(srl_apex_learner_t* L, const uint8_t* obs, int n, float* q_out, void* stream);
/* borrow the step's buffers for tests: "core", "core_next" (double DQN only), "core_next_target" f32 [B,514] (the encoder's core rows;
 * h = columns < 512), "dcore" f32 [B,514], "q", "y" f32 [B], "priorities" f64 [B], "loss" f32 [1], "step" i32 [1] (device step count),
 * and the bf16 activations the forward over s saved, in the learner's layouts (srl_learner_debug_buffer): "a1", "a2", "a3".
 * The categorical head adds "logits", "logits_next" (double DQN only), "logits_next_target" and "dlogits" f32 [B,A*K], "m" f32 [B,K]
 * (the projected targets) and "ce" f32 [B] (the cross-entropies); its "y" is sum_k z_k m_k.  The quantile head adds "theta",
 * "theta_next" (double DQN only), "theta_next_target" and "dtheta" f32 [B,A*N] (the quantiles and their gradient), "target_quantiles"
 * f32 [B,N] and "qr_loss" f32 [B] (the per-transition losses).  The distributional dueling head adds the rows the step composed,
 * "rows_weight_online" / "rows_weight_target" f32 [A*W,512] and "rows_bias_online" / "rows_bias_target" f32 [A*W], and their
 * gradients "rows_weight_grad" f32 [A*W,512] and "rows_bias_grad" f32 [A*W] (W = K or N).
 * Noisy networks add, per network <n> = "online" or "target", the last step's "normals_<n>" (the standard normals) and "noise_<n>"
 * (f of them) f32 [NN] = [fc in 3136 | fc out 512 | head in 512 (dueling: value's, then advantage's) | head out R (dueling: value's 1,
 * then advantage's A)], R = the head's rows (A, A K, or A + 1), and the composed weights "fc_weight_<n>" [512,3136], "fc_bias_<n>"
 * [512], "head_weight_<n>" [R,512], "head_bias_<n>" ([R]; dueling: the value bias [1]) and "head_adv_bias_<n>" (dueling: [A]).
 * srl_apex_learner_q_values reads the mean weights mu (NoisyLinear's eval mode). */
int srl_apex_learner_debug_buffer(srl_apex_learner_t* L, const char* name, void** ptr, int64_t* count);

/* ---- Ape-X actor: per-env epsilon-greedy acting and actor-computed initial priorities (apex/worker.py:59-79, apex/memory.py:43-64) --
 * A forward-only Q network for num_envs envs on a caller-owned flat f32 parameter snapshot (srl_apex_param_layout order, 16-byte
 * aligned; the actor reads it when its kernels run, so the caller refreshes it with one device copy from the learner's parameters).
 * The context owns one encoder context, encoder blocks for num_envs frames, core rows for 2 * num_envs frames and a device draw counter;
 * no optimizer state, gradients or target copy.  Its calls share those buffers: order them on one stream.  Synchronous create. */
typedef struct srl_apex_actor srl_apex_actor_t;
/* A in [1, 31], num_envs in [1, 65536], precision as srl_apex_config_t.precision, seed: the key of the actor's random numbers */
int srl_apex_actor_create(int A, int num_envs, int precision, uint64_t seed, const float* params, srl_apex_actor_t** out);
/* the same with the head kind: dueling 0 (q = Linear(512, A), srl_apex_actor_create's) or 1 (the dueling head; params in
 * srl_apex_param_layout_ex(A, 1) order) */
int srl_apex_actor_create_ex(int A, int num_envs, int precision, int dueling, uint64_t seed, const float* params, srl_apex_actor_t** out);
/* the same with the categorical head: num_atoms in [2, 64] (0: srl_apex_actor_create's plain head), the support [v_min, v_max] as
 * srl_apex_config_t's; params in srl_apex_param_layout_cat(A, num_atoms) order.  Its Q values are the expectations sum_k z_k p_k and its
 * priorities max(KL(m || p(s)[a]), 0) + priority_eps with the snapshot as online and target network (srl_apex_learner_step's bits) */
int srl_apex_actor_create_cat(int A, int num_envs, int precision, int num_atoms, float v_min, float v_max, uint64_t seed, const float* params,
                              srl_apex_actor_t** out);
/* the same for every head: dueling, num_atoms, v_min, v_max as srl_apex_config_t's, and noisy (0 or 1); params in
 * srl_apex_param_layout_noisy(A, dueling, num_atoms, noisy) order.  A noisy actor keeps one noise draw (Philox keyed by seed, counted by
 * a device noise counter, shared by all envs): create draws the first, every act draws a new one before its forward, and q_values and
 * the prioritized add compose the kept draw with the snapshot as it is when they run. */
int srl_apex_actor_create_noisy(int A, int num_envs, int precision, int dueling, int num_atoms, float v_min, float v_max, int noisy,
                                uint64_t seed, const float* params, srl_apex_actor_t** out);
/* the same with the quantile head: num_quantiles and kappa as srl_apex_config_t's (num_quantiles 0: srl_apex_actor_create_noisy's
 * head); params in srl_apex_param_layout_quantile(A, dueling, num_atoms, num_quantiles, noisy) order.  Its Q values are the quantile
 * means and its priorities the quantile Huber loss + priority_eps with the snapshot as online and target network
 * (srl_apex_learner_step's bits) */
int srl_apex_actor_create_quantile(int A, int num_envs, int precision, int dueling, int num_atoms, float v_min, float v_max, int num_quantiles,
                                   float kappa, int noisy, uint64_t seed, const float* params, srl_apex_actor_t** out);
/* the same with dist_dueling as srl_apex_config_t's (0: srl_apex_actor_create_quantile's head); params in
 * srl_apex_param_layout_dist_dueling(A, dueling, num_atoms, num_quantiles, dist_dueling, noisy) order.  Every act, q_values and
 * prioritized add composes the head rows from the snapshot as it is then (after the noise, when noisy), as srl_apex_learner_step does */
int srl_apex_actor_create_dist_dueling(int A, int num_envs, int precision, int dueling, int num_atoms, float v_min, float v_max,
                                       int num_quantiles, float kappa, int dist_dueling, int noisy, uint64_t seed, const float* params,
                                       srl_apex_actor_t** out);
int srl_apex_actor_destroy(srl_apex_actor_t* X);
/* obs u8 [E,4,84,84], epsilons f32 [E] (device) -> actions i64 [E]: with probability epsilons[e] a uniform action, else the first
 * argmax of Q(obs[e]) (torch.argmax's pick).  The random numbers are Philox4x32-10 keyed by seed, counted by (draw, env); the launch
 * advances the device draw counter, so a captured call draws new numbers on every replay.  No host synchronisation; capturable. */
int srl_apex_actor_act(srl_apex_actor_t* X, const uint8_t* obs, const float* epsilons, int64_t* actions, void* stream);
/* Q(obs) with the snapshot for n >= 1 frames: obs u8 [n,4,84,84] -> q_out f32 [n,A] */
int srl_apex_actor_q_values(srl_apex_actor_t* X, const uint8_t* obs, int n, float* q_out, void* stream);
/* borrow the actor's buffers for tests: "core" f32 [2E,514] (rows 0..E-1: the last act or the states of the last prioritized add,
 * rows E..2E-1: its next states) and, categorical head only, "logits" f32 [2E,A*K] of the same rows (quantile head: "theta"
 * f32 [2E,A*N]).  A noisy actor adds its kept draw
 * "normals" and "noise" and the weights its last call composed, "fc_weight", "fc_bias", "head_weight", "head_bias" and (dueling)
 * "head_adv_bias", in the layouts of srl_apex_learner_debug_buffer's.  The distributional dueling head adds the rows its last call
 * composed, "rows_weight" f32 [A*W,512] and "rows_bias" f32 [A*W] */
int srl_apex_actor_debug_buffer(srl_apex_actor_t* X, const char* name, void** ptr, int64_t* count);
/* srl_replay_add, then, for the E transitions the call completes, their initial priorities computed by `actor` (built for the memory's
 * num_envs) instead of max_priority:  p = |Q(s)[a] - y| + priority_eps,  y = R + fp32(gamma^n_step) (1 - d) max_a Q(s')  with the
 * arithmetic of srl_apex_learner_step's target and priority (the same bits for the same weights).  R, a and d are the fold's; s is the
 * oldest staged step's state, s' the newest step's next_state (only read when d = 0).  Leaves ptr.. = p^alpha, max_priority =
 * max(max_priority, p); a non-finite p is stored as max_priority^alpha and counted by srl_per_invalid_updates.  priority_eps finite,
 * > 0.  While the window fills nothing runs beyond the copy. */
int srl_replay_add_prioritized(srl_replay_t* R, srl_apex_actor_t* actor, const uint8_t* state, const int64_t* action, const float* reward,
                               const uint8_t* next_state, const uint8_t* done, float priority_eps, void* stream);
/* srl_replay_add_prioritized on the frame replay memory: s is the oldest staged step's states, rebuilt from their frames when n_step > 1 */
int srl_frame_replay_add_prioritized(srl_frame_replay_t* R, srl_apex_actor_t* actor, const uint8_t* state, const int64_t* action,
                                     const float* reward, const uint8_t* next_state, const uint8_t* done, float priority_eps, void* stream);

/* ---- R2D2 learner step: a recurrent Q network trained on stored-state sequences (Kapturowski et al. 2019) -----------------------
 * The Q network is AtariNet(use_lstm=True)'s encoder and 2-layer LSTM core (srl_encoder_*, srl_lstm_core_*: the row [relu(fc(x)) (512),
 * clamp(r_{t-1}, -1, 1), one_hot(a_{t-1}) (A)], H = 513 + A, the state multiplied by (1 - done_t) before step t) followed by a Q head on
 * the core output: q = Linear(H, A), or with `dueling` value = Linear(H, 1), advantage = Linear(H, A), Q = V + Adv - mean_a Adv (Wang et
 * al. 2016, eq. 9; the mean summed in action order).  bf16 encoder and LSTM operands (the LSTM core has no split mode).
 * Parameters in state_dict order {conv1.weight, conv1.bias, ..., fc.bias, rnn_layer.weight_ih_l0, weight_hh_l0, bias_ih_l0, bias_hh_l0,
 * *_l1, q.weight [A,H], q.bias [A]} (18 tensors), or with the dueling head {..., value.weight [1,H], value.bias [1], advantage.weight
 * [A,H], advantage.bias [A]} (20); in memory in that order, each segment padded to 4 floats (16-byte aligned).  Params, grads, both
 * Adam states and the target copy share the layout.  -> the buffer's floats, or -1 with srl_last_error set (A outside [1, 31],
 * dueling outside {0, 1}). */
int64_t srl_r2d2_param_layout(int A, int dueling, int64_t* offsets20, int64_t* counts20);
typedef struct srl_r2d2_learner srl_r2d2_learner_t;
typedef struct srl_r2d2_config {
  int32_t B;                 /* sequences per step                                                                      */
  int32_t A;                 /* actions, [1, 31]                                                                        */
  int32_t burn_in;           /* rows run without gradient before the trained rows, >= 0 (R2D2 section 3: 40)           */
  int32_t T;                 /* trained rows per sequence, >= 1 (80)                                                    */
  int32_t n_step;            /* n of the n-step return, >= 1 (5); (burn_in + T + n_step) * B <= 65536                    */
  float gamma;               /* discount per step, [0, 1] (0.997); the kernel forms gamma^k itself                      */
  int32_t dueling;           /* 0: q = Linear(H, A); 1: the dueling head                                                */
  int32_t value_rescaling;   /* 1: h(x) = sign(x)(sqrt(|x| + 1) - 1) + eps x on the targets (Pohlen et al. 2018); 0: identity */
  float rescale_eps;         /* eps of h, finite and > 0 when value_rescaling (1e-3)                                    */
  float priority_eta;        /* eta of the sequence priority, [0, 1] (0.9)                                              */
  float priority_eps;        /* added to every priority, finite and >= 0                                                */
  float max_grad_norm;       /* clip_grad_norm_ threshold, > 0; +inf: no clip                                           */
  float learning_rate, adam_beta1, adam_beta2, adam_eps;   /* torch.optim.Adam (1e-4, 0.9, 0.999, 1e-3)                 */
} srl_r2d2_config_t;
/* params / grads / exp_avg / exp_avg_sq / target_params: caller-owned flat f32 device buffers of srl_r2d2_param_layout floats, 16-byte
 * aligned and disjoint.  The context owns the encoder and LSTM blocks of the step and of the q-value forwards.  Synchronous. */
int srl_r2d2_learner_create(const srl_r2d2_config_t* cfg, float* params, float* grads, float* exp_avg, float* exp_avg_sq,
                            float* target_params, srl_r2d2_learner_t** out);
int srl_r2d2_learner_destroy(srl_r2d2_learner_t* L);
/* One learner step on B stored sequences of L = burn_in + T + n_step rows, time-major: frame u8 [L,B,4,84,84], last_action i64 [L,B],
 * reward f32 [L,B], done u8/bool [L,B]; h0 / c0 f32 [2,B,H] the stored recurrent state before row 0; weights f32 [B] (NULL = 1); idxs
 * i64 [B] with per (both NULL, or both set).  Row t holds s_t, the action a_{t-1} and reward r_t that led to it, and done_t (the step
 * into row t ended an episode); the transition of row t is (s_t, a_t = last_action[t+1], reward[t+1], done[t+1]).
 *   burn-in (section 3): rows [0, burn_in) through the online network from (h0, c0), no gradient; the trained rows [burn_in, burn_in + T)
 *     continue from that state; the target network runs all L rows from (h0, c0); the n bootstrap rows get no gradient
 *   a* = first argmax_a Q_online(s_{t+n});  m = the first k in 1..n with done[t+k] (or none)
 *   y_t = h(sum_{k=1}^{min(n,m)} gamma^{k-1} reward[t+k] + [no m] gamma^n h^-1(Q_target(s_{t+n}, a*)))   (section 2, the n-step
 *     double-Q target with value rescaling; evaluated in double, rounded once to fp32)
 *   delta_t = Q_online(s_t, a_t) - y_t;  loss = (1 / (B T)) sum_b w_b sum_t delta_t^2
 *   priority_b = eta max_t |delta_t| + (1 - eta) mean_t |delta_t| + priority_eps (section 2) -> the sampler's trees (last idx wins)
 *   clip_grad_norm_(max_grad_norm) and a torch.optim.Adam step with the step count kept on the device.
 * stats_out: f32 [3] device = {loss, gradient norm, clip coefficient} (may be NULL).  No host synchronisation; capturable. */
int srl_r2d2_learner_step(srl_r2d2_learner_t* L, const uint8_t* frame, const int64_t* last_action, const float* reward, const uint8_t* done,
                          const float* h0, const float* c0, const float* weights, const int64_t* idxs, srl_per_t* per, float* stats_out,
                          void* stream);
/* Q values of the online network over T1 rows of N columns from the state (h0, c0): frame u8 [T1,N,4,84,84], last_action i64 [T1,N],
 * reward f32 [T1,N], done u8 [T1,N], h0 / c0 f32 [2,N,H] -> q_out f32 [T1,N,A], hT / cT f32 [2,N,H] the state after row T1 - 1 (may
 * not overlap h0 / c0).  T1 = 1 is one acting step.  N in [1, min(L B, 2048)].  Runs on its own encoder context and blocks, so it may
 * run on another stream than the step; calls of it on two streams at once share those blocks and must be ordered. */
int srl_r2d2_learner_q_values(srl_r2d2_learner_t* L, const uint8_t* frame, const int64_t* last_action, const float* reward, const uint8_t* done,
                              int T1, int N, const float* h0, const float* c0, float* q_out, float* hT, float* cT, void* stream);
/* target_params = tau * params + (1 - tau) * target_params (srl_apex_learner_update_target's arithmetic); tau in [0, 1] */
int srl_r2d2_learner_update_target(srl_r2d2_learner_t* L, float tau, void* stream);
/* Adam's step count for a resumed run: writes the device counter; synchronises `stream` */
int srl_r2d2_learner_set_step(srl_r2d2_learner_t* L, int64_t step, void* stream);
/* borrow the step's buffers for tests: "core" f32 [L*B,H] (the last encoder forward's rows: the target's), "out_online" f32
 * [(T+n)*B,H] (the LSTM output of rows burn_in..L-1), "out_target" f32 [L*B,H], "h_burn_in" / "c_burn_in" f32 [2,B,H] (burn_in > 0),
 * "q_online" f32 [(T+n)*B,A], "q_target" f32 [T*B,A] (rows burn_in+n..L-1), "dq" f32 [T*B,A], "dout" / "dcore" f32 [(T+n)*B,H] (the
 * head's and the LSTM core's input gradients), "q_taken", "y", "delta" f32 [T*B], "priorities" f64 [B], "loss" f32 [1], "step" i32 [1] */
int srl_r2d2_learner_debug_buffer(srl_r2d2_learner_t* L, const char* name, void** ptr, int64_t* count);

/* ---- trajectory ring -> time-major batch (the stacking step of ImpalaTrainer.get_batch, impala_atari.py:248-251) -----------
 * staging: B trajectory slots on the DEVICE, each one contiguous record of slot_bytes holding every key of create_buffers
 * (impala_atari.py:135-147) for T+1 steps; offsets6_host (HOST array) = byte offsets of {obs u8[T+1,4,84,84], reward f32[T+1],
 * done u8[T+1], action i64[T+1], policy_logits f32[T+1,A], episode_return f32[T+1]} inside a slot.
 * Outputs: the time-major batch tensors [T+1,B,...] (episode_return may be NULL). */
int srl_unpack_slots(const uint8_t* staging, int64_t slot_bytes, const int64_t* offsets6_host, int T, int B, int A,
                     uint8_t* obs, float* reward, uint8_t* done, int64_t* action, float* policy_logits, float* episode_return,
                     void* stream);

/* ---- stand-alone optimizer ops (flat f32 buffers of n elements) ------------------------------------------
 * srl_grad_norm_clip_coef: coef[0] = ||g||_2, coef[1] = min(1, max_norm/(||g||+1e-6)); scratch f32[>=1028].  max_norm < 0 or +inf:
 * no clip (coefficient 1).  A NaN norm gives a NaN coefficient, as torch.nn.utils.clip_grad_norm_ does, so one NaN gradient poisons
 * every clipped gradient; an Inf one gives the coefficient 0.  The fused steps (srl_learner_apply_gradients[_dp],
 * srl_apex_learner_step) clip the same way. */
int srl_grad_norm_clip_coef(const float* grads, int64_t n, float max_norm, float* coef, float* scratch, void* stream);
int srl_rmsprop_step(float* params, const float* grads, float* square_avg, int64_t n, const float* coef,
                     float lr, float alpha, float eps, void* stream);
int srl_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n, const float* coef,
                  float lr, float beta1, float beta2, float eps, int step, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SCALERL_B200_H_ */
