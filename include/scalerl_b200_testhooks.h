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
#ifdef __cplusplus
}
#endif
#endif
