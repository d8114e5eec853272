/* scalerl_b200 test hooks -- C ABI of libscalerl_b200_testhooks.so (NOT shipped in the product library).
 * Unit-test entry points for the sm_90a building blocks of the learner kernels.  Return value: 0 on success, a
 * cudaError_t (> 0) or -1 for a bad argument; srl_test_last_error() holds the message. */
#ifndef SCALERL_B200_TESTHOOKS_H_
#define SCALERL_B200_TESTHOOKS_H_
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif
const char* srl_test_last_error(void);
/* descriptor experiment: operand windows that start at an arbitrary 128-byte row of a SWIZZLE_128B tile.
 * kmajor (mn_major=0): A bf16 [160,64], B bf16 [64,64]  -> D[128,64] = A[shift:shift+128] . B^T
 * mnmajor (=1)       : A bf16 [96,128], B bf16 [96,64]  -> D[128,64] = A[shift:shift+64]^T . B[shift:shift+64]   (shift <= 32) */
int srl_test_shifted_operand(const void* A, const void* B, float* D, int shift, int mn_major, int base_offset_mode, void* stream);
/* fills the shared memory of every SM with quiet-NaN bit patterns (kernels must never depend on stale smem) */
int srl_test_poison_smem(void* stream);
/* programmatic-dependent-launch self test; every out[0..nblk) must read 1 (flag, out: device int buffers) */
int srl_test_pdl(int* flag, int* out, int nblk, unsigned delay_ns, void* stream);
/* where srl_encoder_forward / srl_encoder_backward put a named row of their saved and scratch blocks (both as srl_encoder_sizes sized
 * them for `frames` and `precision`): the same carving of the same table (kernels.h encoder_rows).  name: xs, a1, a2, a3, h, wpack,
 * dh, da3, da2, da1, wgrad_part or a3t.  *hi receives the row's address, *lo its low twin's (NULL in the bf16 mode and for rows
 * without one), *count its elements. */
int srl_test_encoder_row(int frames, int precision, const char* name, void* saved, void* scratch, void** hi, void** lo, int64_t* count);
/* one fused clip + optimizer step (the cooperative kernel srl_learner_apply_gradients and srl_apex_learner_step run) on flat f32
 * device buffers of any n >= 1.  optimizer 0 = RMSprop: s0 = square_avg, a = alpha (b, s1 unused); 1 = Adam: s0 = exp_avg,
 * s1 = exp_avg_sq, a, b = beta1, beta2.  coef f32[3] receives {norm, clip coefficient, lr of the step (but for constant-lr RMSprop
 * without momentum)}; scratch f32[>= 596] the block partials.  The step count is *dstep + 1 (dstep NULL: step >= 1), stored back to
 * *dstep.  schedule 0 = constant lr, 1 = linear (lr_end >= 0, frames_per_step > 0, total_frames > 0); momentum_buf (RMSprop only,
 * NULL: none) with momentum >= 0.  p, g, s0, s1, momentum_buf 16-byte aligned.  blocks (may be NULL) receives the grid launched,
 * variant (may be NULL) the parameters of the clip_optim_kernel<OPT, SCHED, MOM> template launched: 4 OPT + 2 SCHED + MOM. */
int srl_test_clip_optim(int optimizer, float* p, float* g, float* s0, float* s1, int64_t n, float max_norm, float* coef, float* scratch,
                        float lr, float a, float b, float eps, int step, int* dstep, int schedule, float lr_end, double frames_per_step,
                        double total_frames, float* momentum_buf, float momentum, int* blocks, int* variant, void* stream);
#ifdef __cplusplus
}
#endif
#endif
