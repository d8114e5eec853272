// clip_grad_norm_ (impala_atari.py:344-345) + RMSprop (impala_atari.py:99-105,346) / Adam:
//   * the stand-alone norm and update kernels of the C ABI (srl_grad_norm_clip_coef, srl_rmsprop_step, srl_adam_step)
//   * the learner's clip + optimizer step as one cooperative kernel, single-GPU and data-parallel
//   * the weight-publish snapshot
#include "common.cuh"
#include "kernels.h"
#include <cooperative_groups.h>
#include <type_traits>
namespace cg = cooperative_groups;
#ifndef SRL_TRY
#define SRL_TRY(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return e_; } while (0)
#endif

namespace srl {

// ------------------------------------------------------------------------------------------------
// shared math: every kernel below computes the norm, the clip coefficient and the update with these
// ------------------------------------------------------------------------------------------------
// scratch[4 + b] holds block b's partial sum of squares (scratch[0]: grad_sumsq_kernel's ticket)
// thread 0 stores the block's sum of s: warp sums, then the WARPS warp sums in warp order (red: WARPS floats of shared memory)
template <int WARPS>
SRL_DEVINL void block_partial(float s, float* red, float* scratch) {
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < WARPS; ++w) t += red[w];
    scratch[4 + blockIdx.x] = t;
  }
}
// sum of the partials of blocks [0, count) in double, by one warp in a fixed order (deterministic); every lane returns it.
// The partials were written by other blocks: they are read from L2.
SRL_DEVINL double sum_partials(const float* scratch, unsigned count) {
  double t = 0.0;
  for (unsigned k = threadIdx.x; k < count; k += 32) t += (double)__ldcg(scratch + 4 + k);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  return t;
}
// torch.nn.utils.clip_grad_norm_: the gradients are scaled by min(1, max_norm / (||g|| + 1e-6)); max_norm < 0 and max_norm = +inf
// do not clip (coefficient exactly 1).  A NaN norm gives a NaN coefficient, as torch's clamp(max=1) does, so a NaN anywhere in the
// gradients poisons every weight (fminf would return the non-NaN operand, 1, and step every other weight as if nothing happened).
SRL_DEVINL float clip_coef(float norm, float max_norm) {
  if (!(max_norm >= 0.f) || isinf(max_norm)) return 1.0f;
  const float c = max_norm / (norm + 1e-6f);
  return c < 1.0f || isnan(c) ? c : 1.0f;
}

// one element of torch.optim.RMSprop(centered=False) on the clipped gradient gk: v = a v + (1-a) gk^2, then
// MOM: m = mu m + gk / (sqrt(v) + eps), p -= lr m;  else: p -= lr gk / (sqrt(v) + eps).
template <bool MOM>
SRL_DEVINL void rmsprop_elem(float& p, float& v, float& m, float gk, float lr, float a, float eps, float mu) {
  v = a * v + (1.f - a) * gk * gk;
  if (MOM) {
    m = mu * m + gk / (sqrtf(v) + eps);
    p = p - lr * m;
  } else {
    p = p - lr * (gk / (sqrtf(v) + eps));
  }
}
template <bool MOM>
SRL_DEVINL void rmsprop_v4(float4& pp, float4& vv, float4& mm, const float4& gg, float c, float lr, float a, float eps, float mu) {
  float* P = &pp.x; float* V = &vv.x; float* M = &mm.x; const float* G = &gg.x;
#pragma unroll
  for (int k = 0; k < 4; ++k) rmsprop_elem<MOM>(P[k], V[k], M[k], G[k] * c, lr, a, eps, mu);
}

// torch.optim.Adam's bias corrections of the 1-based step t: 1 / (1 - b1^t) and 1 / sqrt(1 - b2^t)
struct AdamBias { float inv_bc1, inv_sqrt_bc2; };
SRL_DEVINL AdamBias adam_bias(float b1, float b2, int t) {
  return {1.0f / (float)(1.0 - pow((double)b1, (double)t)), 1.0f / sqrtf((float)(1.0 - pow((double)b2, (double)t)))};
}
// one element of torch.optim.Adam on the clipped gradient gk: m = b1 m + (1-b1) gk ; v = b2 v + (1-b2) gk^2 ;
// p -= (lr/bc1) m / (sqrt(v)/sqrt(bc2) + eps).  The argument order is the order of the callers' loads (g, m, v, p), which the
// schedule of the fused kernels follows.
SRL_DEVINL void adam_elem(float gk, float& m, float& v, float& p, float lr, float b1, float b2, float eps, const AdamBias& bc) {
  const float mk = b1 * m + (1.f - b1) * gk;
  const float vk = b2 * v + (1.f - b2) * gk * gk;
  m = mk; v = vk;
  p = p - (lr * bc.inv_bc1) * (mk / (sqrtf(vk) * bc.inv_sqrt_bc2 + eps));
}

// lr of the 1-based step t: SCHED_LINEAR = max(lr (1 - min((t-1) F, Ftot) / Ftot), lr_end) -- torchbeast's LambdaLR
// (scheduler.step() after optimizer.step(): step 1 runs at lr) with the floor of the reference's LinearDecayScheduler.
// The whole expression is evaluated in double and rounded once, so the host's closed form gives the same float.
SRL_DEVINL float scheduled_lr(float lr, int t, const OptExtra& x) {
  const double f = 1.0 - fmin((double)(t - 1) * x.frames_per_step, x.total_frames) / x.total_frames;
  return (float)fmax((double)lr * f, (double)x.lr_end);
}

// ------------------------------------------------------------------------------------------------
// stand-alone kernels (C ABI)
// ------------------------------------------------------------------------------------------------
// coef[0] = ||g||_2 ; coef[1] = the clip coefficient.  scratch: [0] ticket (uint), [4 .. 4+grid) block partials; the last block to
// take a ticket adds the partials.
__global__ void __launch_bounds__(256) grad_sumsq_kernel(const float* __restrict__ g, int64_t n, float max_norm, float* __restrict__ coef,
                                                         float* __restrict__ scratch) {
  float s = 0.f;
  const int64_t n4 = n >> 2;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 v = __ldg(g4 + i);
    s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) { const float v = g[n4 * 4 + threadIdx.x]; s += v * v; }
  __shared__ float red[8];
  __shared__ bool is_last;
  block_partial<8>(s, red, scratch);
  if (threadIdx.x == 0) {
    __threadfence();
    is_last = atomicAdd(reinterpret_cast<unsigned*>(scratch), 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (is_last && threadIdx.x < 32) {
    __threadfence();
    const double t = sum_partials(scratch, gridDim.x);
    if (threadIdx.x == 0) {
      const float norm = (float)sqrt(t);
      coef[0] = norm;
      coef[1] = clip_coef(norm, max_norm);
      *reinterpret_cast<unsigned*>(scratch) = 0u;
    }
  }
}

// torch.optim.RMSprop(momentum=0, centered=False) with g pre-scaled by coef[1] (coef == nullptr: unscaled)
__global__ void __launch_bounds__(256) rmsprop_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ v, int64_t n,
                                                      const float* __restrict__ coef, float lr, float alpha, float eps) {
  const float c = coef ? __ldg(coef + 1) : 1.0f;
  const int64_t n4 = n >> 2;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 pp = reinterpret_cast<float4*>(p)[i], vv = reinterpret_cast<float4*>(v)[i], mm = {};
    const float4 gg = __ldg(reinterpret_cast<const float4*>(g) + i);
    rmsprop_v4<false>(pp, vv, mm, gg, c, lr, alpha, eps, 0.f);
    reinterpret_cast<float4*>(p)[i] = pp;
    reinterpret_cast<float4*>(v)[i] = vv;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const int64_t i = n4 * 4 + threadIdx.x;
    float m = 0.f;
    rmsprop_elem<false>(p[i], v[i], m, g[i] * c, lr, alpha, eps, 0.f);
  }
}

// torch.optim.Adam with g pre-scaled by coef[1] (coef == nullptr: unscaled); step = the 1-based step count
__global__ void __launch_bounds__(256) adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                   float* __restrict__ v, int64_t n, const float* __restrict__ coef, float lr, float b1,
                                                   float b2, float eps, int step) {
  const float c = coef ? __ldg(coef + 1) : 1.0f;
  const AdamBias bc = adam_bias(b1, b2, step);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    adam_elem(g[i] * c, m[i], v[i], p[i], lr, b1, b2, eps, bc);
}

cudaError_t launch_grad_norm(const float* g, int64_t n, float max_norm, float* coef, float* scratch, cudaStream_t st) {
  int blocks = (int)((n / 4 + 255) / 256);
  if (blocks > 592) blocks = 592;
  if (blocks < 1) blocks = 1;
  grad_sumsq_kernel<<<blocks, 256, 0, st>>>(g, n, max_norm, coef, scratch);
  return cudaGetLastError();
}
static int ew_blocks(int64_t n) { int64_t b = (n / 4 + 255) / 256; return (int)(b < 1 ? 1 : (b > 1184 ? 1184 : b)); }
cudaError_t launch_rmsprop(float* p, const float* g, float* v, int64_t n, const float* coef, float lr, float alpha, float eps,
                           cudaStream_t st) {
  rmsprop_kernel<<<ew_blocks(n), 256, 0, st>>>(p, g, v, n, coef, lr, alpha, eps);
  return cudaGetLastError();
}
cudaError_t launch_adam(float* p, const float* g, float* m, float* v, int64_t n, const float* coef, float lr, float b1, float b2, float eps,
                        int step, cudaStream_t st) {
  adam_kernel<<<ew_blocks(n * 4), 256, 0, st>>>(p, g, m, v, n, coef, lr, b1, b2, eps, step);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// clip_grad_norm_ + optimizer step as ONE cooperative kernel (impala_atari.py:344-346): phase 1 sums g^2 (block partials
// in a fixed slot each), grid barrier, every block adds the partials in the same fixed order (deterministic, identical
// in all blocks), phase 2 applies the clipped update (g is re-read from L2).  OPT 0 = RMSprop, 1 = Adam; SCHED = the
// learning-rate schedule (OptExtra); MOM = RMSprop momentum.  Every variant but the constant-lr, no-momentum one writes the
// step's lr to coef[2].
// ------------------------------------------------------------------------------------------------
template <int OPT, int SCHED, bool MOM>
__global__ void __launch_bounds__(512) clip_optim_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ s0,
                                                         float* __restrict__ s1, int64_t n, float max_norm, float* __restrict__ coef,
                                                         float* __restrict__ scratch, float lr, float a, float b, float eps, int step,
                                                         int* __restrict__ dstep, const OptExtra x) {
  static_assert(!(MOM && OPT != 0), "momentum is an RMSprop option");
  cg::grid_group grid = cg::this_grid();
  pdl_wait(52);    // (cooperative launch, no attribute: returns at once; names the kernel in the diagnostics timeline)
  const int64_t n4 = n >> 2, stride = (int64_t)gridDim.x * blockDim.x, i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int t = dstep ? *dstep + 1 : step;          // 1-based step count: Adam bias correction; counted for RMSprop too (checkpoints)
  const float lr_t = SCHED == SCHED_LINEAR ? scheduled_lr(lr, t, x) : lr;
  float* __restrict__ mb = x.buf;                   // MOM: the momentum buffer
  // The thread's first HOLD float4 of g (and, for RMSprop, of p and the state) stay in registers across the grid barrier: phase 2 then
  // starts from registers instead of paying a second round of L2 / HBM latency (the grid covers n with <= HOLD items per thread).
  constexpr int HOLD = 2;
  float4 gh[HOLD], ph[HOLD], vh[HOLD], mh[HOLD];
  float s = 0.f;
#pragma unroll
  for (int h = 0; h < HOLD; ++h) {
    const int64_t i = i0 + h * stride;
    if (i < n4) {
      gh[h] = reinterpret_cast<const float4*>(g)[i];
      if (OPT == 0) { ph[h] = reinterpret_cast<const float4*>(p)[i]; vh[h] = reinterpret_cast<const float4*>(s0)[i]; }
      if (MOM) mh[h] = reinterpret_cast<const float4*>(mb)[i];
    }
  }
#pragma unroll
  for (int h = 0; h < HOLD; ++h)
    if (i0 + h * stride < n4) s += gh[h].x * gh[h].x + gh[h].y * gh[h].y + gh[h].z * gh[h].z + gh[h].w * gh[h].w;
  for (int64_t i = i0 + HOLD * stride; i < n4; i += stride) {
    const float4 v = reinterpret_cast<const float4*>(g)[i];
    s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) { const float v = g[n4 * 4 + threadIdx.x]; s += v * v; }
  __shared__ float red[16];
  __shared__ float c_sh;
  block_partial<16>(s, red, scratch);
  grid.sync();
  if (threadIdx.x < 32) {
    const double tsum = sum_partials(scratch, gridDim.x);
    if (threadIdx.x == 0) {
      const float norm = (float)sqrt(tsum);
      const float c = clip_coef(norm, max_norm);
      c_sh = c;
      if (blockIdx.x == 0) {
        coef[0] = norm; coef[1] = c;
        if (SCHED != SCHED_CONSTANT || MOM) coef[2] = lr_t;
        if (dstep) *dstep = t;
      }
    }
  }
  __syncthreads();
  const float c = c_sh;
  const float mu = x.momentum;
  float m1 = 0.f;                                   // !MOM: the unused momentum slot of the scalar tail
  if (OPT == 0) {
#pragma unroll
    for (int h = 0; h < HOLD; ++h) {
      const int64_t i = i0 + h * stride;
      if (i < n4) {
        float4 pp = ph[h], vv = vh[h], mm = MOM ? mh[h] : float4{};
        rmsprop_v4<MOM>(pp, vv, mm, gh[h], c, lr_t, a, eps, mu);
        reinterpret_cast<float4*>(p)[i] = pp;
        reinterpret_cast<float4*>(s0)[i] = vv;
        if (MOM) reinterpret_cast<float4*>(mb)[i] = mm;
      }
    }
    for (int64_t i = i0 + HOLD * stride; i < n4; i += stride) {
      float4 pp = reinterpret_cast<float4*>(p)[i], vv = reinterpret_cast<float4*>(s0)[i], mm = MOM ? reinterpret_cast<float4*>(mb)[i] : float4{};
      const float4 gg = reinterpret_cast<const float4*>(g)[i];
      rmsprop_v4<MOM>(pp, vv, mm, gg, c, lr_t, a, eps, mu);
      reinterpret_cast<float4*>(p)[i] = pp;
      reinterpret_cast<float4*>(s0)[i] = vv;
      if (MOM) reinterpret_cast<float4*>(mb)[i] = mm;
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
      const int64_t i = n4 * 4 + threadIdx.x;
      float* m = MOM ? mb + i : &m1;
      rmsprop_elem<MOM>(p[i], s0[i], *m, g[i] * c, lr_t, a, eps, mu);
    }
  } else {
    const AdamBias bc = adam_bias(a, b, t);
    for (int64_t i = i0; i < n; i += stride) adam_elem(g[i] * c, s0[i], s1[i], p[i], lr_t, a, b, eps, bc);
  }
}

// ------------------------------------------------------------------------------------------------
// Data-parallel apply step as ONE cooperative kernel over peer memory (NVLink / NVSwitch loads), no NCCL on the data path:
//   barrier 1 (every rank finished its backward)
//   phase 1   reduce-scatter: rank r sums slice r of the flat gradient over all ranks (NVLink loads from the peers' buffers,
//             rank order) into its exchange buffer rs[r] (and in place), accumulating the slice's sum of squares
//   barrier 2 (all slices reduced, per-slice sums of squares published to every rank)
//   phase 2   all-gather by pull fused with clip_grad_norm_ + RMSprop/Adam: every rank reads each reduced slice from its
//             owner's exchange buffer (so all replicas see the same bits), keeps a copy in its gradient buffer, and updates
//             its own replica of the parameters
// No closing barrier: the exchange buffers are separate from the gradient buffers, so the next backward may start while a
// slow peer is still pulling; rs[r] is rewritten only after the next barrier 1, which that peer reaches after this kernel.
// (Measured at N = 2: pulling beats pushing the reduced slice into every rank -- the system-scope fence after remote
// stores waits 3-10 us for their acknowledgements.)
// The gradient buffers and the control blocks are symmetric-memory allocations mapped into every rank
// (torch.distributed._symmetric_memory); ctl[p] is rank p's control block: words [0,8) = barrier epochs written by each
// source rank, [8,16) = per-slice sums of squares (float bits) written by each source rank, [32] = local epoch counter.
// Cross-GPU waits are bounded (30 s of globaltimer, then trap): a lost peer becomes a CUDA error, not a hang.
// ------------------------------------------------------------------------------------------------
SRL_DEVINL float4 ld_sys_v4(const float* p) {
  float4 v;
  asm volatile("ld.volatile.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
SRL_DEVINL float ld_sys_f32(const float* p) {
  float v;
  asm volatile("ld.volatile.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
  return v;
}
SRL_DEVINL void st_release_sys(unsigned* p, unsigned v) { asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
SRL_DEVINL void st_relaxed_sys(unsigned* p, unsigned v) { asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
SRL_DEVINL unsigned ld_acquire_sys(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
SRL_DEVINL unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
SRL_DEVINL void st_sys_v4(float* p, const float4& v) {
  asm volatile("st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
// NVLS (NVLink SHARP) multicast accesses: `p` is an address inside a multicast mapping of a symmetric buffer.  ld_reduce returns
// the SUM over every rank's copy, computed in the switch (one request instead of world-1 peer loads); st writes every copy.
SRL_DEVINL float4 multimem_ld_reduce_v4(const float* p) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
SRL_DEVINL float multimem_ld_reduce_f32(const float* p) {
  float v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
  return v;
}
SRL_DEVINL void multimem_st_v4(float* p, const float4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
SRL_DEVINL void multimem_st_f32(float* p, float v) { asm volatile("multimem.st.relaxed.sys.global.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory"); }

// cross-GPU barrier, split in two: one block signals every rank, EVERY block waits on the local flags (thread q < world
// waits for rank q).  Waits are bounded: 30 s of globaltimer, then trap.
// fence = true when this block wrote remote memory that the flag publishes (the release store is cumulative over what the
// thread observed through the block / grid barriers, but remote relaxed stores of another thread are fenced explicitly)
SRL_DEVINL void dp_signal(const DpPeers& P, unsigned epoch, bool fence) {      // threads q < world of one block
  if ((int)threadIdx.x < P.world) {
    if (fence) __threadfence_system();
    st_release_sys(P.ctl[threadIdx.x] + P.rank, epoch);
  }
}
SRL_DEVINL void dp_wait(const DpPeers& P, unsigned epoch) {        // all threads of a block
  if ((int)threadIdx.x < P.world) {
    const unsigned* mine = P.ctl[P.rank] + threadIdx.x;
    const unsigned long long t0 = global_ns();
    unsigned spins = 0;
    while ((int)(ld_acquire_sys(mine) - epoch) < 0) {
      if ((++spins & 0x3FFu) == 0 && global_ns() - t0 > 30000000000ull) __trap();     // the timer is read every 1024 polls
    }
  }
  __syncthreads();
}


// NVLS = true (the symmetric gradient buffer has a multicast mapping, P.mc_g): phase 1 is ONE multimem.ld_reduce per float4 of
// the rank's slice (the switch adds the world copies) followed by a multimem.st that writes the sum into EVERY rank's gradient
// buffer; after barrier 2 each rank holds the complete reduced gradient locally, so phase 2 is the plain single-GPU clip +
// optimizer pass -- no peer pulls, no exchange buffer.  An element is read and then overwritten only by its slice's owner, so
// the in-place broadcast cannot race with another rank's reduction.  All replicas consume the owner's bits: bit-identical.
// OPT, SCHED and MOM as for clip_optim_kernel.
template <int OPT, bool NVLS, int SCHED, bool MOM>
__global__ void __launch_bounds__(512) dp_clip_optim_kernel(float* __restrict__ p, float* g, float* __restrict__ s0, float* __restrict__ s1,
                                                            int64_t n, float max_norm, float* coef, float* scratch, float lr, float a,
                                                            float b, float eps, int step, int* dstep, const DpPeers P, const OptExtra x) {
  static_assert(!(MOM && OPT != 0), "momentum is an RMSprop option");
  cg::grid_group grid = cg::this_grid();
  const int64_t n4 = n >> 2, stride = (int64_t)gridDim.x * blockDim.x, i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int W = P.world, R = P.rank;
  const int64_t chunk = (n4 + W - 1) / W, lo = R * chunk, hi = min(n4, lo + chunk);
  const int t = dstep ? *reinterpret_cast<volatile int*>(dstep) + 1 : step;
  const float lr_t = SCHED == SCHED_LINEAR ? scheduled_lr(lr, t, x) : lr;
  float* __restrict__ mb = x.buf;                   // MOM: the momentum buffer (local, like the parameters)
  const unsigned e0 = reinterpret_cast<volatile unsigned*>(P.ctl[R])[32];     // epoch base (rewritten after the grid barrier)
  // ---- barrier 1: every rank's backward is complete
  if (blockIdx.x == 0) dp_signal(P, e0 + 1, false);      // the gradients were written by earlier kernels: already at L2
  dp_wait(P, e0 + 1);
  // ---- phase 1: reduce my slice over all ranks (rank order); the result goes to my exchange buffer rs (read by the peers
  //      in phase 2) and, in place, to my gradient buffer
  float s = 0.f;
  float* rs_mine = P.rs[R];
  if constexpr (NVLS) {
    constexpr int PF = 4;                                  // PF switch reductions in flight per thread
    for (int64_t ib = lo + i0; ib < hi; ib += PF * stride) {
      float4 acc[PF];
#pragma unroll
      for (int u = 0; u < PF; ++u) { const int64_t i = ib + u * stride; if (i < hi) acc[u] = multimem_ld_reduce_v4(P.mc_g + 4 * i); }
#pragma unroll
      for (int u = 0; u < PF; ++u) {
        const int64_t i = ib + u * stride;
        if (i < hi) {
          multimem_st_v4(P.mc_g + 4 * i, acc[u]);          // every rank's gradient buffer (mine included) receives the sum
          s += acc[u].x * acc[u].x + acc[u].y * acc[u].y + acc[u].z * acc[u].z + acc[u].w * acc[u].w;
        }
      }
    }
    if (R == W - 1 && blockIdx.x == 0 && (int64_t)threadIdx.x < (n & 3)) {
      const int64_t i = n4 * 4 + threadIdx.x;
      const float acc = multimem_ld_reduce_f32(P.mc_g + i);
      multimem_st_f32(P.mc_g + i, acc);
      s += acc * acc;
    }
    // no per-thread system fence here (it cost a full NVLink round trip per step, ~8 us at N = 8): the grid barrier below orders
    // every thread's multimem.st before block 0's fence.sys + st.release of barrier 2, and fence cumulativity (PTX memory model)
    // carries those writes to the acquiring peers -- the same rule the peer-load variant relies on for its exchange buffer
  } else {
    for (int64_t i = lo + i0; i < hi; i += stride) {
      float4 acc = ld_sys_v4(P.g[0] + 4 * i);
      for (int q = 1; q < W; ++q) {
        const float4 v = ld_sys_v4(P.g[q] + 4 * i);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
      reinterpret_cast<float4*>(rs_mine)[i - lo] = acc;
      reinterpret_cast<float4*>(g)[i] = acc;
      s += acc.x * acc.x + acc.y * acc.y + acc.z * acc.z + acc.w * acc.w;
    }
    if (R == W - 1 && blockIdx.x == 0 && (int64_t)threadIdx.x < (n & 3)) {     // the n % 4 tail belongs to the last slice
      const int64_t i = n4 * 4 + threadIdx.x;
      float acc = ld_sys_f32(P.g[0] + i);
      for (int q = 1; q < W; ++q) acc += ld_sys_f32(P.g[q] + i);
      rs_mine[4 * chunk + threadIdx.x] = acc;
      g[i] = acc;
      s += acc * acc;
    }
  }
  __shared__ float red[16];
  __shared__ float c_sh;
  // the slice stores are local: the grid barrier makes them visible at L2, which is where the peers' NVLink loads land
  block_partial<16>(s, red, scratch);
  grid.sync();
  // ---- barrier 2: all slices pushed everywhere, per-slice sums of squares published
  if (blockIdx.x == 0) {
    if (threadIdx.x < 32) {
      const double tsum = sum_partials(scratch, gridDim.x);
      if (threadIdx.x == 0) {
        for (int q = 0; q < W; ++q) st_relaxed_sys(P.ctl[q] + 8 + R, __float_as_uint((float)tsum));
        reinterpret_cast<volatile unsigned*>(P.ctl[R])[32] = e0 + 2;          // every block has read e0 / dstep (grid barrier above)
        if (dstep) *dstep = t;
      }
    }
    __syncthreads();
    dp_signal(P, e0 + 2, true);
  }
  dp_wait(P, e0 + 2);
  if (threadIdx.x == 0) {
    double tot = 0.0;
    for (int q = 0; q < W; ++q) tot += (double)__uint_as_float(reinterpret_cast<volatile unsigned*>(P.ctl[R])[8 + q]);
    const float norm = (float)sqrt(tot);
    const float c = clip_coef(norm, max_norm);      // identical in every block of every rank
    c_sh = c;
    if (blockIdx.x == 0) {
      coef[0] = norm; coef[1] = c;
      if (SCHED != SCHED_CONSTANT || MOM) coef[2] = lr_t;
    }
  }
  __syncthreads();
  const float c = c_sh;
  const float mu = x.momentum;
  // ---- phase 2: clip + optimizer on my replica; the gradient buffer is local and fully reduced now
  const AdamBias bc = OPT == 1 ? adam_bias(a, b, t) : AdamBias{0.f, 0.f};
  // the pulls of up to DP_PF iterations are issued before any of them is used: one NVLink round trip, not one per iteration
  constexpr int DP_PF = 4;
  for (int64_t ib = i0; ib < n4; ib += DP_PF * stride) {
    float4 gpre[DP_PF];
#pragma unroll
    for (int u = 0; u < DP_PF; ++u) {
      const int64_t i = ib + u * stride;
      if (i < n4) {
        const int owner = (int)min((int64_t)(W - 1), i / chunk);
        // NVLS: the owner's multimem.st already put the sum into my buffer (written by a peer: read past L1 with ld.volatile)
        gpre[u] = NVLS ? ld_sys_v4(g + 4 * i)
                       : (owner == R ? reinterpret_cast<const float4*>(g)[i] : ld_sys_v4(P.rs[owner] + 4 * (i - owner * chunk)));
      }
    }
#pragma unroll
    for (int u = 0; u < DP_PF; ++u) {
      const int64_t i = ib + u * stride;
      if (i >= n4) break;
      const float4 gg = gpre[u];
      if (!NVLS && (int)min((int64_t)(W - 1), i / chunk) != R) reinterpret_cast<float4*>(g)[i] = gg;       // keep a copy: all-gather
      float4 pp = reinterpret_cast<float4*>(p)[i], vv = reinterpret_cast<float4*>(s0)[i];
      if (OPT == 0) {
        float4 mm = MOM ? reinterpret_cast<float4*>(mb)[i] : float4{};
        rmsprop_v4<MOM>(pp, vv, mm, gg, c, lr_t, a, eps, mu);
        if (MOM) reinterpret_cast<float4*>(mb)[i] = mm;
      } else {
        // adam_elem's arithmetic, written out: through the helper the compiler contracts b v + (1-b) g^2 into the other FMA here,
        // which changes the rounding of exp_avg_sq
        float* Pp = &pp.x; float* V = &vv.x; const float* G = &gg.x;
        float4 ww = reinterpret_cast<float4*>(s1)[i];
        float* Wv = &ww.x;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float gk = G[k] * c;
          V[k] = a * V[k] + (1.f - a) * gk;                    // exp_avg
          Wv[k] = b * Wv[k] + (1.f - b) * gk * gk;             // exp_avg_sq
          Pp[k] = Pp[k] - (lr_t * bc.inv_bc1) * (V[k] / (sqrtf(Wv[k]) * bc.inv_sqrt_bc2 + eps));
        }
        reinterpret_cast<float4*>(s1)[i] = ww;
      }
      reinterpret_cast<float4*>(p)[i] = pp;
      reinterpret_cast<float4*>(s0)[i] = vv;
    }
  }
  if (blockIdx.x == 0 && (int64_t)threadIdx.x < (n & 3)) {
    const int64_t i = n4 * 4 + threadIdx.x;
    float gv;
    if (NVLS) gv = ld_sys_f32(g + i);
    else if (R == W - 1) gv = g[i];
    else { gv = ld_sys_f32(P.rs[W - 1] + 4 * chunk + threadIdx.x); g[i] = gv; }
    const float gk = gv * c;
    if (OPT == 0) {
      float m1 = 0.f;                               // !MOM: the unused momentum slot
      rmsprop_elem<MOM>(p[i], s0[i], MOM ? mb[i] : m1, gk, lr_t, a, eps, mu);
    } else {
      adam_elem(gk, s0[i], s1[i], p[i], lr_t, a, b, eps, bc);
    }
  }
  // no closing barrier: after barrier 2 no rank touches another rank's memory until the next step's barrier 1
}

// Weight-publish snapshot (impala_atari.py:348): dst = src when the step's total loss is finite, else dst keeps the last good
// weights -- so the asynchronous D2H that follows never hands poisoned parameters to the actors.
__global__ void __launch_bounds__(256) snapshot_if_finite_kernel(float4* __restrict__ dst, const float4* __restrict__ src, int64_t n4,
                                                                 const float* __restrict__ losses) {
  if (losses) {
    const float t = losses[3];
    if (!isfinite(t)) return;                    // NaN or Inf: keep the previous snapshot
  }
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) dst[i] = __ldg(src + i);
}
cudaError_t launch_snapshot_if_finite(float* dst, const float* src, int64_t n, const float* losses, cudaStream_t st) {
  const int64_t n4 = n >> 2;        // flat parameter buffers are padded to multiples of 4 floats
  int blocks = (int)((n4 + 255) / 256);
  if (blocks > 132 * 8) blocks = 132 * 8;
  if (blocks < 1) blocks = 1;
  snapshot_if_finite_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<float4*>(dst), reinterpret_cast<const float4*>(src), n4, losses);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// launchers of the fused steps
// ------------------------------------------------------------------------------------------------
// blocks of a cooperative optimizer launch: enough 512-thread blocks to cover n with one float4 per thread, at most what can be
// co-resident and at most 592 (scratch holds 592 partials).  Occupancy is queried once per device and kernel.
template <auto KERNEL>
static cudaError_t coop_blocks(int64_t n, int* blocks_out) {
  static int per_sm_dev[64] = {}, sms_dev[64] = {};      // per device and kernel: one process may drive several GPUs
  int dev = 0;
  SRL_TRY(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
  if (!per_sm_dev[dev]) {
    int sm_count = 0, occ = 0;
    SRL_TRY(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev));
    SRL_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, KERNEL, 512, 0));
    if (occ < 1) return cudaErrorLaunchOutOfResources;
    sms_dev[dev] = sm_count; per_sm_dev[dev] = occ;
  }
  const int per_sm = per_sm_dev[dev], sms = sms_dev[dev];
  int64_t need = (n / 4 + 511) / 512;
  int blocks = (int)(need < 1 ? 1 : need);
  int cap = per_sm * sms; if (cap > 592) cap = 592;
  if (blocks > cap) blocks = cap;
  *blocks_out = blocks;
  return cudaSuccess;
}
template <auto KERNEL>
static cudaError_t launch_coop(int64_t n, void** args, cudaStream_t st, int* blocks_out = nullptr) {
  int blocks = 0;
  SRL_TRY(coop_blocks<KERNEL>(n, &blocks));
  if (blocks_out) *blocks_out = blocks;
  return cudaLaunchCooperativeKernel((const void*)KERNEL, dim3(blocks), dim3(512), args, 0, st);
}
// calls f(OPT, SCHED, MOM), as std::integral_constants, for the variant of the step: RMSprop with or without momentum, or Adam,
// each under the constant or the linear schedule
template <class F>
static cudaError_t with_variant(int optimizer, const OptExtra& x, F f) {
  using Rms = std::integral_constant<int, 0>;
  using Adam = std::integral_constant<int, 1>;
  using Const = std::integral_constant<int, SCHED_CONSTANT>;
  using Lin = std::integral_constant<int, SCHED_LINEAR>;
  const bool lin = x.schedule == SCHED_LINEAR;
  if (optimizer == 1) return lin ? f(Adam(), Lin(), std::false_type()) : f(Adam(), Const(), std::false_type());
  if (x.buf) return lin ? f(Rms(), Lin(), std::true_type()) : f(Rms(), Const(), std::true_type());
  return lin ? f(Rms(), Lin(), std::false_type()) : f(Rms(), Const(), std::false_type());
}

cudaError_t launch_clip_optim(const OptStep& o, cudaStream_t st, int* blocks, int* variant) {
  OptStep a = o;        // addressable copies of the kernel arguments
  void* args[] = {&a.p, &a.g, &a.s0, &a.s1, &a.n, &a.max_norm, &a.coef, &a.scratch, &a.lr, &a.a, &a.b, &a.eps, &a.step, &a.dstep, &a.x};
  return with_variant(o.optimizer, o.x, [&](auto O, auto S, auto M) {
    if (variant) *variant = 4 * decltype(O)::value + 2 * decltype(S)::value + (decltype(M)::value ? 1 : 0);
    return launch_coop<clip_optim_kernel<O, S, M>>(o.n, args, st, blocks);
  });
}
cudaError_t launch_dp_clip_optim(const OptStep& o, const DpPeers& P, cudaStream_t st) {
  OptStep a = o;
  DpPeers q = P;
  void* args[] = {&a.p, &a.g, &a.s0, &a.s1, &a.n, &a.max_norm, &a.coef, &a.scratch, &a.lr, &a.a, &a.b, &a.eps, &a.step, &a.dstep, &q, &a.x};
  return with_variant(o.optimizer, o.x, [&](auto O, auto S, auto M) {
    return P.mc_g ? launch_coop<dp_clip_optim_kernel<O, true, S, M>>(o.n, args, st)
                  : launch_coop<dp_clip_optim_kernel<O, false, S, M>>(o.n, args, st);
  });
}

SRL_KSTAMP_SETTER(kstamp_set_optim)

}  // namespace srl
