// Test-only entry points (include/scalerl_b200_testhooks.h), built into libscalerl_b200_testhooks.so -- NOT part of the
// product library.  They exercise the building blocks the product kernels rely on, in isolation: K-major / MN-major
// SWIZZLE_128B wgmma operand descriptors that start at an arbitrary 128-byte row of a swizzled tile (the "resident
// window" trick of igemm_res.cuh), programmatic dependent launch, a shared-memory poisoner (kernels must never
// depend on stale shared memory), and the fused clip + optimizer step of optim.cu at any size (the learners only run it
// on their own parameter counts).
#include <stdlib.h>
#include <string.h>
#include "../../include/scalerl_b200_testhooks.h"
#include "errors.h"
#include "kernels.h"

using namespace srl;

extern "C" const char* srl_test_last_error(void) { return error_message(); }

namespace srl {
// the hooks library is self-contained: its own copies of the launch switches declared in kernels.h
bool pdl_active() {
  static const bool env_on = [] { const char* e = getenv("SRL_PDL"); return !e || atoi(e) != 0; }();
  return env_on;
}
void pdl_set_active(bool) {}
}  // namespace srl

extern "C" int srl_test_shifted_operand(const void* A, const void* B, float* D, int shift, int mn_major, int base_offset_mode, void* stream) {
  REQ(A && B && D && shift >= 0 && shift <= 32, "test_shifted_operand: bad argument");
  CU(test_shift(A, B, D, shift, mn_major, base_offset_mode, (cudaStream_t)stream), "test_shifted_operand");
  return 0;
}
extern "C" int srl_test_pdl(int* flag, int* out, int nblk, unsigned delay_ns, void* stream) {
  REQ(flag && out && nblk > 0, "test_pdl: bad argument");
  CU(test_pdl(flag, out, nblk, delay_ns, (cudaStream_t)stream), "test_pdl");
  return 0;
}
extern "C" int srl_test_poison_smem(void* stream) {
  CU(test_poison_smem((cudaStream_t)stream), "test_poison_smem");
  return 0;
}

extern "C" int srl_test_encoder_row(int frames, int precision, const char* name, void* saved, void* scratch, void** hi, void** lo,
                                    int64_t* count) {
  REQ(name && saved && scratch && hi && lo && count, "test_encoder_row: NULL argument");
  REQ(frames >= 1 && frames <= MAX_FRAMES, "test_encoder_row: frames=%d must be in [1, %d]", frames, MAX_FRAMES);
  REQ(precision == 0 || precision == 1, "test_encoder_row: precision=%d must be 0 (bf16 operands) or 1 (fp32-accurate split operands)",
      precision);
  EncoderBuffers b = {};
  WsRow t[ENC_ROWS];
  encoder_rows(b, frames, frames, t);
  int i = 0;
  while (i < ENC_ROWS && !(t[i].name && strcmp(t[i].name, name) == 0)) ++i;
  REQ(i < ENC_ROWS, "test_encoder_row: unknown row '%s'", name);
  CU(carve_blocks(t, ENC_ROWS, ENC_SAVED_ROWS, precision == 1, saved, scratch), "test_encoder_row");
  *hi = *t[i].hi;
  *lo = precision == 1 && t[i].lo ? *t[i].lo : nullptr;
  *count = t[i].count;
  return 0;
}

extern "C" int srl_test_clip_optim(int optimizer, float* p, float* g, float* s0, float* s1, int64_t n, float max_norm, float* coef,
                                   float* scratch, float lr, float a, float b, float eps, int step, int* dstep, int schedule, float lr_end,
                                   double frames_per_step, double total_frames, float* momentum_buf, float momentum, int* blocks,
                                   int* variant, void* stream) {
  REQ(optimizer == 0 || optimizer == 1, "test_clip_optim: optimizer=%d must be 0 (RMSprop) or 1 (Adam)", optimizer);
  REQ(p && g && s0 && coef && scratch && (optimizer == 0 || s1), "test_clip_optim: NULL pointer");
  REQ(n >= 1, "test_clip_optim: n=%lld must be >= 1", (long long)n);
  REQ(dstep || step >= 1, "test_clip_optim: step=%d must be >= 1 without a device step count", step);
  REQ(schedule == SCHED_CONSTANT || schedule == SCHED_LINEAR, "test_clip_optim: unknown schedule %d", schedule);
  REQ(schedule == SCHED_CONSTANT || (lr_end >= 0.f && frames_per_step > 0.0 && total_frames > 0.0),
      "test_clip_optim: the linear schedule needs lr_end >= 0, frames_per_step > 0 and total_frames > 0");
  REQ(!momentum_buf || (optimizer == 0 && momentum >= 0.f), "test_clip_optim: momentum is an RMSprop option, >= 0");
  REQ(!misaligned(p, 16) && !misaligned(g, 16) && !misaligned(s0, 16) && !misaligned(s1, 16) && !misaligned(momentum_buf, 16),
      "test_clip_optim: buffers must be 16-byte aligned");
  OptExtra x;
  x.schedule = schedule;
  x.lr_end = lr_end;
  x.frames_per_step = frames_per_step;
  x.total_frames = schedule == SCHED_LINEAR ? total_frames : 1.0;
  x.buf = momentum_buf;
  x.momentum = momentum_buf ? momentum : 0.f;
  const OptStep o = {optimizer, p, g, s0, optimizer == 1 ? s1 : nullptr, n, max_norm, coef, scratch, lr, a, optimizer == 1 ? b : 0.f, eps,
                     step, dstep, x};
  CU(launch_clip_optim(o, (cudaStream_t)stream, blocks, variant), "test_clip_optim");
  return 0;
}
