// Common device helpers for the sm_90a kernels: mbarrier, proxy fences, wgmma (fence / commit / wait, the accumulator row
// hand-off), wgmma shared-memory descriptors, bf16 packing.
// Hand-written inline PTX; descriptor bit layouts follow the PTX ISA "wgmma matrix descriptor" table.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include "wgmma.cuh"

#define SRL_DEVINL __device__ __forceinline__

#ifndef SRL_SPIN_LIMIT
#define SRL_SPIN_LIMIT (1u << 24)   // bounded mbarrier spin: a broken pipeline traps instead of hanging the GPU
#endif

namespace srl {

SRL_DEVINL uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// ------------------------------------------------------------------------------------------
// mbarrier
// ------------------------------------------------------------------------------------------
SRL_DEVINL void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
SRL_DEVINL void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
SRL_DEVINL void mbar_arrive(uint64_t* bar) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
SRL_DEVINL void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
SRL_DEVINL bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
SRL_DEVINL void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > SRL_SPIN_LIMIT) { __trap(); }
  }
}

// Programmatic dependent launch (PDL).  A kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may start
// while its stream predecessor is still running: everything before pdl_wait() (barrier init, descriptor
// prefetch, loads of data that was complete long before the predecessor started) overlaps the predecessor's tail;
// pdl_wait() returns once the predecessor grid has completed and its memory is visible.  pdl_launch() lets the NEXT
// kernel in the stream begin its own prologue.  Both are no-ops for a kernel launched without the attribute.
// Diagnostics build (SRL_DEFINES=SRL_KSTAMP, tests/diag/diag_timeline.py): thread 0 of block 0 of every kernel appends {kernel id, %globaltimer at
// entry, %globaltimer when its stream predecessor had completed} to a buffer -- the in-graph timeline of a step, which no profiler here can
// show (ncu serialises the launches, per-kernel CUDA events break the programmatic dependencies).  Never defined in the product build.
#ifdef SRL_KSTAMP
static __device__ unsigned long long* g_kstamp = nullptr;      // one copy per translation unit: kstamp_set_<unit>() (kernels.h)
SRL_DEVINL unsigned long long kstamp_now() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
SRL_DEVINL void kstamp_put(int kid, unsigned long long t0) {
  if (g_kstamp && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) {
    const unsigned long long t1 = kstamp_now(), i = atomicAdd(g_kstamp, 1ull);
    if (i < 2000) { g_kstamp[1 + 3 * i] = (unsigned long long)kid; g_kstamp[2 + 3 * i] = t0; g_kstamp[3 + 3 * i] = t1; }
  }
}
#define SRL_KSTAMP_SETTER(fn) void fn(unsigned long long* q) { cudaMemcpyToSymbol(g_kstamp, &q, sizeof q); }
#else
#define SRL_KSTAMP_SETTER(fn) void fn(unsigned long long*) {}
#endif
// kid: the kernel's id in the diagnostics timeline (ignored by the product build)
SRL_DEVINL void pdl_wait(int kid = 0) {
#ifdef SRL_KSTAMP
  const unsigned long long t0 = kstamp_now();
#endif
  asm volatile("griddepcontrol.wait;" ::: "memory");
#ifdef SRL_KSTAMP
  if (kid) kstamp_put(kid, t0);
#else
  (void)kid;
#endif
}
SRL_DEVINL void pdl_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// 16-byte shared-memory load through the shared pipe (LDS), never a generic LD: keeps it in order with mbarrier operations
SRL_DEVINL uint4 lds128(uint32_t saddr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(saddr) : "memory");
  return v;
}
SRL_DEVINL void sts_volatile_f32(uint32_t saddr, float v) { asm volatile("st.volatile.shared.f32 [%0], %1;" ::"r"(saddr), "f"(v) : "memory"); }

// generic-proxy smem writes -> visible to the async proxy (wgmma / TMA reads)
SRL_DEVINL void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA): accumulators live in the registers of the issuing warpgroup
// ------------------------------------------------------------------------------------------
// one lane of the (converged) warp: the form the compiler recognises as 'exactly one thread' for the TMA issue paths
SRL_DEVINL uint32_t elect_one_sync() {
  uint32_t pred;
  __syncwarp();      // elect.sync needs the full warp converged
  asm volatile("{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.u32 %0, 1, 0, P;\n\t}" : "=r"(pred));
  return pred;
}
SRL_DEVINL void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
SRL_DEVINL void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
SRL_DEVINL void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// every committed group but the newest has completed: the MMAs of the next k-block can be issued while the last one retires
SRL_DEVINL void wg_wait_prev() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }
// Per-warpgroup register budgets (setmaxnreg, .sync.aligned: every warp of the warpgroup executes it).  A CTA's warps are dealt
// round-robin to the four SM sub-partitions of 16384 registers each, so per-thread counts summed over one warp of every role
// must stay <= 512.  The TMA producer gives registers back, the warpgroups holding wgmma accumulators take them.
template <int N> SRL_DEVINL void reg_release() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> SRL_DEVINL void reg_claim() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
// keeps the compiler from moving accumulator reads / writes across wgmma.wait_group
template <int N>
SRL_DEVINL void wg_fence_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
SRL_DEVINL void named_bar(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

// D[128 x N] += A[128 x 16] * B[N x 16]^T for one warpgroup: two m64 halves, d[0] = rows 0..63, d[1] = rows 64..127.
// a_hi: descriptor distance (16-byte units) from the rows-0..63 A tile to the rows-64..127 one.
template <int N, int TA, int TB>
SRL_DEVINL void wg_mma128(float (&d)[2][N / 2], uint64_t ad, uint32_t a_hi, uint64_t bd, uint32_t accumulate) {
  Wgmma<N, TA, TB>::mma(d[0], ad, bd, accumulate);
  Wgmma<N, TA, TB>::mma(d[1], ad + a_hi, bd, accumulate);
}

// Row hand-off of a 128 x N accumulator held by one warpgroup (wgmma fragment layout) to the row-per-thread epilogues: thread
// `wt` (0..127) receives row wt, columns 16c..16c+15, in v.  Goes through `img` (2 x 128 rows x 20 floats of shared memory,
// WG_IMG_BYTES, private to the warpgroup; the two halves alternate so one barrier per chunk suffices).  bar: named barrier id.
// ONE_BUF: `img` is half that size (WG_IMG_BYTES / 2) and every chunk pays a second barrier.
// deepest pipeline (<= want stages of `per` bytes) that fits the 227 KB shared-memory budget beside `fixed` bytes
constexpr int fit_stages(int want, int fixed, int per) {
  int s = want;
  while (s > 1 && fixed + s * per > 232448) --s;
  return s;
}
constexpr int WG_IMG_STRIDE = 20;                        // 16 columns + 4: conflict-free 16-byte row reads
constexpr int WG_IMG_BYTES = 2 * 128 * WG_IMG_STRIDE * 4;
// wg_acc_rows16: the same for two separate 64 x N accumulators d0 (rows 0..63) and d1 (rows 64..127).
template <int N, bool ONE_BUF = false>
SRL_DEVINL void wg_acc_rows16(const float (&d0)[N / 2], const float (&d1)[N / 2], int c, float* img, int wt, int bar, float (&v)[16]) {
  float* buf = ONE_BUF ? img : img + (c & 1) * 128 * WG_IMG_STRIDE;
  if (ONE_BUF) named_bar(bar, 128);                      // the previous chunk has been read by every thread
  const int w = wt >> 5, l = wt & 31;
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int jj = 0; jj < 2; ++jj)
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int row = 64 * h + 16 * w + (l >> 2) + 8 * rr, i = 4 * (2 * c + jj) + 2 * rr;
        const float (&d)[N / 2] = h ? d1 : d0;
        *reinterpret_cast<float2*>(buf + row * WG_IMG_STRIDE + 8 * jj + 2 * (l & 3)) = make_float2(d[i], d[i + 1]);
      }
  named_bar(bar, 128);
  const float4* q = reinterpret_cast<const float4*>(buf + wt * WG_IMG_STRIDE);
#pragma unroll
  for (int j = 0; j < 4; ++j) { const float4 x = q[j]; v[4 * j] = x.x; v[4 * j + 1] = x.y; v[4 * j + 2] = x.z; v[4 * j + 3] = x.w; }
}
template <int N, bool ONE_BUF = false>
SRL_DEVINL void wg_acc_row16(const float (&d)[2][N / 2], int c, float* img, int wt, int bar, float (&v)[16]) {
  wg_acc_rows16<N, ONE_BUF>(d[0], d[1], c, img, wt, bar, v);
}

// ------------------------------------------------------------------------------------------
// descriptors
// ------------------------------------------------------------------------------------------
// wgmma shared-memory matrix descriptor, SWIZZLE_128B. byte offsets are encoded >>4.
//   K-major  tile: rows (M/N index) of 128 B (64 bf16 along K); 8-row groups 1024 B apart  -> SBO=1024, LBO=16 (ignored)
//   MN-major tile: rows (K index)   of 128 B (64 bf16 along M/N); 8-row groups 1024 B apart -> SBO=1024,
//                  LBO = byte distance between successive 64-element M/N blocks
// The swizzle is a function of the absolute shared-memory address (as TMA writes it), so a descriptor may start at any
// 128-byte row of a 1024-byte-aligned tile (tests/test_gpu_parity.py::test_shifted_operand_descriptors).
SRL_DEVINL uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;   // SWIZZLE_128B
  return d;
}
// the same descriptor for a SWIZZLE_64B tile (rows of 64 B, 8-row groups 512 B apart)
SRL_DEVINL uint64_t make_smem_desc_sw64(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return (make_smem_desc(saddr, lbo_bytes, sbo_bytes) & ~((uint64_t)3 << 62)) | ((uint64_t)2 << 62);
}

// 128B-swizzle: 16-byte chunk c (0..7) of 128-byte row r lands at chunk position c ^ (r & 7)
SRL_DEVINL uint32_t swz128(uint32_t row, uint32_t chunk) { return row * 128u + ((chunk ^ (row & 7u)) << 4); }
// 64B-swizzle: 16-byte chunk c (0..3) of 64-byte row r lands at chunk position c ^ ((r >> 1) & 3)   (address bits [4:5] ^= bits [7:8])
SRL_DEVINL uint32_t swz64(uint32_t row, uint32_t chunk) { return row * 64u + ((chunk ^ ((row >> 1) & 3u)) << 4); }

// ------------------------------------------------------------------------------------------
// small numeric helpers
// ------------------------------------------------------------------------------------------
SRL_DEVINL uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
SRL_DEVINL float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
SRL_DEVINL float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xFFFF0000u); }

// 16-byte vector reduction: 4 fp32 adds in one L2 atomic transaction (sm_90+)
SRL_DEVINL void red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
SRL_DEVINL void red_add_16(float* dst, const float (&v)[16], float scale = 1.0f) {
#pragma unroll
  for (int j = 0; j < 16; j += 4) red_add_v4(dst + j, v[j] * scale, v[j + 1] * scale, v[j + 2] * scale, v[j + 3] * scale);
}

// Action index of a trajectory element, clamped to [0, A-1]: the reference's F.one_hot / gather raise on an out-of-range
// action (atari_model.py:104, vtrace.py:35-40); a kernel cannot raise, so it must at least never index out of bounds
// (the host side offers the raising check: B200ImpalaLearner(validate_inputs=True)).
SRL_DEVINL int ld_action(const int64_t* p, int A) {
  const long long a = __ldg(reinterpret_cast<const long long*>(p));
  return a < 0 ? 0 : (a >= A ? A - 1 : (int)a);
}

// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC 2011): four 32-bit words of counter c under key k.
// The Ape-X actor's epsilon-greedy draws and the noisy networks' noise (noisy.cu) use it.
SRL_DEVINL uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u; k.y += 0xBB67AE85u;
  }
  return c;
}

SRL_DEVINL float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// The ticket of a two-level deterministic reduction (the IMPALA and DQN loss tails): scratch[0] counts the blocks that have
// published their partials.  One thread per block calls it after its stores; true in the block that published last, which then
// sums the partials in its kernel's fixed order and re-arms the ticket (scratch[0] = 0).
SRL_DEVINL bool take_ticket(float* scratch) {
  __threadfence();
  return atomicAdd(reinterpret_cast<unsigned*>(scratch), 1u) == gridDim.x - 1;
}

}  // namespace srl
