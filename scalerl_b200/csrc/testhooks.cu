// Test-only entry points (include/scalerl_b200_testhooks.h), built into libscalerl_b200_testhooks.so -- NOT part of the
// product library.  They exercise the building blocks the product kernels rely on, in isolation: K-major / MN-major
// SWIZZLE_128B wgmma operand descriptors that start at an arbitrary 128-byte row of a swizzled tile (the "resident
// window" trick of igemm_res.cuh), programmatic dependent launch, and a shared-memory poisoner (kernels must never
// depend on stale shared memory).
#include <stdlib.h>
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

