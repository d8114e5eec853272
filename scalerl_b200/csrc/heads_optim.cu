// fp32 CUDA-core kernels around the encoder:
//   * policy / baseline heads forward + backward (atari_model.py:104-107,126-127 and their autograd)
//   * bias-gradient column sums over bf16 dY
//   * clip_grad_norm_ (impala_atari.py:344-345) + RMSprop (impala_atari.py:99-105,346) / Adam update
#include "common.cuh"
#include "kernels.h"
#include <cooperative_groups.h>
namespace cg = cooperative_groups;
#ifndef SRL_TRY
#define SRL_TRY(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return e_; } while (0)
#endif

namespace srl {

constexpr int HEAD_MAX_A = 32;

// ------------------------------------------------------------------------------------------------
// heads forward: one warp per frame.  core = [h(512), clamp(reward,-1,1), one_hot(action)(A)]
// ------------------------------------------------------------------------------------------------
// Block = 256 threads = 2 frames x 4 warps; warp w of a frame owns features [128w, 128w+128), 4 per lane (float4 loads).
__global__ void __launch_bounds__(256) head_fwd_kernel(const float* __restrict__ hpart, int nsplit, const float* __restrict__ bfc,
                                                       float* __restrict__ h, const float* __restrict__ reward,
                                                       const int64_t* __restrict__ action, const float* __restrict__ Wp,
                                                       const float* __restrict__ bp, const float* __restrict__ Wb,
                                                       const float* __restrict__ bb, int N, int A, float* __restrict__ logits,
                                                       float* __restrict__ baseline) {
  pdl_wait(46);    // launched with programmatic stream serialization: see common.cuh
  pdl_launch();
  __shared__ float part[2][4][HEAD_MAX_A + 1];
  const int lane = threadIdx.x & 31, warp = (threadIdx.x >> 5) & 3, f = threadIdx.x >> 7;
  const int n = blockIdx.x * 2 + f;
  const int CORE = 513 + A;
  const int j = warp * 128 + lane * 4;
  if (n < N) {
    // fc epilogue: reduce the split-K partials in fixed order, + bias, ReLU (atari_model.py:100-101)
    float4 x = __ldg(reinterpret_cast<const float4*>(hpart + (size_t)n * 512 + j));
    for (int k = 1; k < nsplit; ++k) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(hpart + ((size_t)k * N + n) * 512 + j));
      x.x += t.x; x.y += t.y; x.z += t.z; x.w += t.w;
    }
    const float4 b4 = __ldg(reinterpret_cast<const float4*>(bfc + j));
    x.x = fmaxf(x.x + b4.x, 0.f); x.y = fmaxf(x.y + b4.y, 0.f); x.z = fmaxf(x.z + b4.z, 0.f); x.w = fmaxf(x.w + b4.w, 0.f);
    *reinterpret_cast<float4*>(h + (size_t)n * 512 + j) = x;
    for (int a = 0; a <= A; ++a) {
      const float* w = (a < A ? Wp + (size_t)a * CORE : Wb) + j;     // rows are not 16-byte aligned (CORE is odd): scalar loads
      float s = x.x * __ldg(w) + x.y * __ldg(w + 1) + x.z * __ldg(w + 2) + x.w * __ldg(w + 3);
      s = warp_sum(s);
      if (lane == 0) part[f][warp][a] = s;
    }
  }
  __syncthreads();
  if (n < N && warp == 0 && lane <= A) {
    const int a = lane;
    const float* w = a < A ? Wp + (size_t)a * CORE : Wb;
    const float r = fminf(fmaxf(__ldg(reward + n), -1.f), 1.f);
    const int act = ld_action(action + n, A);
    float s = (part[f][0][a] + part[f][1][a]) + (part[f][2][a] + part[f][3][a]);
    s += __ldg(w + 512) * r + __ldg(w + 513 + act) + (a < A ? __ldg(bp + a) : __ldg(bb));
    if (a < A) logits[(size_t)n * A + a] = s; else baseline[n] = s;
  }
}

// dh[n][j] = (sum_a dlogits[n][a] Wp[a][j] + dV[n] Wb[j]) * (h[n][j] > 0)  -> bf16 (operand of the fc dgrad/wgrad GEMMs)
__global__ void __launch_bounds__(128) head_bwd_dh_kernel(const float* __restrict__ dlogits, const float* __restrict__ dbaseline,
                                                          const float* __restrict__ h, const float* __restrict__ Wp,
                                                          const float* __restrict__ Wb, int N, int A, __nv_bfloat16* __restrict__ dh,
                                                          __nv_bfloat16* __restrict__ dh_lo) {
  pdl_wait(47);    // launched with programmatic stream serialization: see common.cuh
  pdl_launch();
  const int n = blockIdx.x;
  const int j = blockIdx.y * 128 + threadIdx.x;
  const int CORE = 513 + A;
  float s = __ldg(dbaseline + n) * __ldg(Wb + j);
  for (int a = 0; a < A; ++a) s = fmaf(__ldg(dlogits + (size_t)n * A + a), __ldg(Wp + (size_t)a * CORE + j), s);
  if (!(__ldg(h + (size_t)n * 512 + j) > 0.f)) s = 0.f;
  const __nv_bfloat16 hi = __float2bfloat16_rn(s);
  dh[(size_t)n * 512 + j] = hi;
  if (dh_lo) dh_lo[(size_t)n * 512 + j] = __float2bfloat16_rn(s - __bfloat162float(hi));     // fp32-accurate operand mode
}

// head weight/bias gradients: thread = one column j of `core` (j == CORE is the bias "ones" column), blockIdx.y = a group of
// consecutive slabs of frames.  Each group writes its A+1 partial sums to part[group][a][j]; head_wgrad_reduce_kernel adds the
// groups in a fixed order, so the gradients are the same bits on every run (no float atomics).
constexpr int HEAD_SLAB = 16;   // frames per slab
__global__ void __launch_bounds__(128) head_wgrad_kernel(const float* __restrict__ dlogits, const float* __restrict__ dbaseline,
                                                         const float* __restrict__ h, const float* __restrict__ reward,
                                                         const int64_t* __restrict__ action, int N, int A, int slabs_per_group,
                                                         float* __restrict__ part) {
  pdl_wait(48);    // (side stream, no attribute: returns at once; names the kernel in the diagnostics timeline)
  __shared__ float sd[HEAD_SLAB][HEAD_MAX_A + 1];
  __shared__ float sr[HEAD_SLAB];
  __shared__ int sa[HEAD_SLAB];
  const int j = blockIdx.x * 128 + threadIdx.x;
  const int CORE = 513 + A;
  const int nslab = (N + HEAD_SLAB - 1) / HEAD_SLAB;
  const int s0 = blockIdx.y * slabs_per_group, s1 = min(nslab, s0 + slabs_per_group);
  float acc[HEAD_MAX_A + 1];
#pragma unroll
  for (int a = 0; a <= HEAD_MAX_A; ++a) acc[a] = 0.f;
  for (int sl = s0; sl < s1; ++sl) {
    const int n0 = sl * HEAD_SLAB, cnt = min(HEAD_SLAB, N - n0);
    __syncthreads();                 // the previous slab's shared rows have been read
    for (int i = threadIdx.x; i < HEAD_SLAB * (A + 1); i += 128) {   // rows past the ragged end are ZERO (0 * stale smem could be NaN)
      const int r = i / (A + 1), a = i - r * (A + 1);
      sd[r][a] = r < cnt ? (a < A ? __ldg(dlogits + (size_t)(n0 + r) * A + a) : __ldg(dbaseline + n0 + r)) : 0.f;
    }
    if (threadIdx.x < cnt) {
      sr[threadIdx.x] = fminf(fmaxf(__ldg(reward + n0 + threadIdx.x), -1.f), 1.f);
      sa[threadIdx.x] = ld_action(action + n0 + threadIdx.x, A);
    }
    __syncthreads();
    if (j > CORE) continue;
    float c[HEAD_SLAB];
#pragma unroll
    for (int r = 0; r < HEAD_SLAB; ++r) {       // all loads of the slab are independent: HEAD_SLAB requests in flight
      float v = 0.f;
      if (r < cnt) {
        if (j < 512) v = __ldg(h + (size_t)(n0 + r) * 512 + j);
        else if (j == 512) v = sr[r];
        else if (j < CORE) v = (sa[r] == j - 513) ? 1.f : 0.f;
        else v = 1.f;
      }
      c[r] = v;
    }
#pragma unroll
    for (int a = 0; a <= HEAD_MAX_A; ++a) {
      if (a > A) break;
#pragma unroll
      for (int r = 0; r < HEAD_SLAB; ++r) acc[a] = fmaf(sd[r][a], c[r], acc[a]);
    }
  }
  if (j > CORE) return;
#pragma unroll
  for (int a = 0; a <= HEAD_MAX_A; ++a)
    if (a <= A) part[((size_t)blockIdx.y * (A + 1) + a) * (CORE + 1) + j] = acc[a];
}
// sums the groups' partials in group order and adds them into the pre-zeroed head gradients
__global__ void __launch_bounds__(256) head_wgrad_reduce_kernel(const float* __restrict__ part, int groups, int A, float* __restrict__ gWp,
                                                                float* __restrict__ gbp, float* __restrict__ gWb, float* __restrict__ gbb) {
  const int CORE = 513 + A, n = (A + 1) * (CORE + 1);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = 0.f;
  for (int g = 0; g < groups; ++g) s += __ldg(part + (size_t)g * n + i);
  const int a = i / (CORE + 1), j = i - a * (CORE + 1);
  if (a < A) { if (j < CORE) gWp[(size_t)a * CORE + j] += s; else gbp[a] += s; }
  else       { if (j < CORE) gWb[j] += s; else gbb[0] += s; }
}

// ------------------------------------------------------------------------------------------------
// optimizer
// ------------------------------------------------------------------------------------------------
// coef[0] = ||g||_2 ; coef[1] = min(1, max_norm / (||g|| + 1e-6))     (torch.nn.utils.clip_grad_norm_)
// scratch: [0] ticket (uint), [4 .. 4+grid) block partials
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
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += red[w];
    scratch[4 + blockIdx.x] = t;
    __threadfence();
    is_last = atomicAdd(reinterpret_cast<unsigned*>(scratch), 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (is_last && threadIdx.x < 32) {   // fixed-order parallel sum of the block partials (deterministic)
    __threadfence();
    double t = 0.0;
    for (unsigned k = threadIdx.x; k < gridDim.x; k += 32) t += (double)reinterpret_cast<volatile float*>(scratch)[4 + k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (threadIdx.x == 0) {
      const float norm = (float)sqrt(t);
      coef[0] = norm;
      coef[1] = max_norm >= 0.f ? fminf(max_norm / (norm + 1e-6f), 1.0f) : 1.0f;
      *reinterpret_cast<unsigned*>(scratch) = 0u;
    }
  }
}

// torch.optim.RMSprop(momentum=0, centered=False): v = alpha v + (1-alpha) g^2 ; p -= lr g / (sqrt(v) + eps); g pre-scaled by coef[1]
__global__ void __launch_bounds__(256) rmsprop_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ v, int64_t n,
                                                      const float* __restrict__ coef, float lr, float alpha, float eps) {
  const float c = coef ? __ldg(coef + 1) : 1.0f;
  const int64_t n4 = n >> 2;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 pp = reinterpret_cast<float4*>(p)[i], vv = reinterpret_cast<float4*>(v)[i];
    const float4 gg = __ldg(reinterpret_cast<const float4*>(g) + i);
    float* P = &pp.x; float* V = &vv.x; const float* G = &gg.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float gk = G[k] * c;
      V[k] = alpha * V[k] + (1.f - alpha) * gk * gk;
      P[k] = P[k] - lr * (gk / (sqrtf(V[k]) + eps));
    }
    reinterpret_cast<float4*>(p)[i] = pp;
    reinterpret_cast<float4*>(v)[i] = vv;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const int64_t i = n4 * 4 + threadIdx.x;
    const float gk = g[i] * c;
    v[i] = alpha * v[i] + (1.f - alpha) * gk * gk;
    p[i] = p[i] - lr * (gk / (sqrtf(v[i]) + eps));
  }
}

// torch.optim.Adam: m = b1 m + (1-b1) g ; v = b2 v + (1-b2) g^2 ; p -= (lr/bc1) m / (sqrt(v)/sqrt(bc2) + eps)
// The 1-based step count is read from device memory (dstep, incremented by adam_step_inc_kernel) so that a captured
// CUDA graph replays with the right bias correction; dstep == nullptr uses the host-provided `step`.
__global__ void adam_step_inc_kernel(int* dstep) { *dstep += 1; }
__global__ void __launch_bounds__(256) adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                   float* __restrict__ v, int64_t n, const float* __restrict__ coef, float lr, float b1,
                                                   float b2, float eps, int step, const int* __restrict__ dstep) {
  const float c = coef ? __ldg(coef + 1) : 1.0f;
  const int t = dstep ? *dstep : step;
  const float inv_bc1 = 1.0f / (float)(1.0 - pow((double)b1, (double)t));
  const float inv_sqrt_bc2 = 1.0f / sqrtf((float)(1.0 - pow((double)b2, (double)t)));
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float gk = g[i] * c;
    const float mk = b1 * m[i] + (1.f - b1) * gk;
    const float vk = b2 * v[i] + (1.f - b2) * gk * gk;
    m[i] = mk; v[i] = vk;
    p[i] = p[i] - (lr * inv_bc1) * (mk / (sqrtf(vk) * inv_sqrt_bc2 + eps));
  }
}

// ------------------------------------------------------------------------------------------------
// LSTM path (use_lstm): the heads read the LSTM output X [N][H] (H = 513 + A) instead of [h, reward, one-hot]
// ------------------------------------------------------------------------------------------------
// core[n] = [relu(sum_s hpart + bfc) (512), clamp(reward,-1,1), one_hot(action) (A)]  (atari_model.py:100-107); also stores h
__global__ void __launch_bounds__(128) core_build_kernel(const float* __restrict__ hpart, int nsplit, const float* __restrict__ bfc,
                                                         const float* __restrict__ reward, const int64_t* __restrict__ action, int N, int A,
                                                         float* __restrict__ h, float* __restrict__ core) {
  const int n = blockIdx.x, H = 513 + A;
  for (int j = threadIdx.x; j < H; j += 128) {
    float v;
    if (j < 512) {
      v = __ldg(hpart + (size_t)n * 512 + j);
      for (int k = 1; k < nsplit; ++k) v += __ldg(hpart + ((size_t)k * N + n) * 512 + j);
      v = fmaxf(v + __ldg(bfc + j), 0.f);
      h[(size_t)n * 512 + j] = v;
    } else if (j == 512) {
      v = fminf(fmaxf(__ldg(reward + n), -1.f), 1.f);
    } else {
      v = (ld_action(action + n, A) == j - 513) ? 1.f : 0.f;
    }
    core[(size_t)n * H + j] = v;
  }
}
// logits[n][a] = X[n] . Wp[a] + bp[a];  baseline[n] = X[n] . Wb + bb      (one warp per frame)
__global__ void __launch_bounds__(256) head_dense_fwd_kernel(const float* __restrict__ X, const float* __restrict__ Wp, const float* __restrict__ bp,
                                                             const float* __restrict__ Wb, const float* __restrict__ bb, int N, int A,
                                                             float* __restrict__ logits, float* __restrict__ baseline) {
  const int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (n >= N) return;
  const int H = 513 + A;
  for (int a = 0; a <= A; ++a) {
    const float* w = a < A ? Wp + (size_t)a * H : Wb;
    float s = 0.f;
    for (int j = lane; j < H; j += 32) s = fmaf(__ldg(X + (size_t)n * H + j), __ldg(w + j), s);
    s = warp_sum(s);
    if (lane == 0) { if (a < A) logits[(size_t)n * A + a] = s + __ldg(bp + a); else baseline[n] = s + __ldg(bb); }
  }
}
// dX[n][j] = sum_a dlogits[n][a] Wp[a][j] + dV[n] Wb[j];  head weight/bias gradients accumulated atomically (slabs of 16 frames)
__global__ void __launch_bounds__(128) head_dense_bwd_kernel(const float* __restrict__ X, const float* __restrict__ dlogits,
                                                             const float* __restrict__ dbaseline, const float* __restrict__ Wp,
                                                             const float* __restrict__ Wb, int N, int A, float* __restrict__ dX,
                                                             float* __restrict__ gWp, float* __restrict__ gbp, float* __restrict__ gWb,
                                                             float* __restrict__ gbb) {
  __shared__ float sd[16][HEAD_MAX_A + 1];
  const int H = 513 + A, j = blockIdx.x * 128 + threadIdx.x;
  const int n0 = blockIdx.y * 16, cnt = min(16, N - n0);
  for (int i = threadIdx.x; i < HEAD_SLAB * (A + 1); i += 128) {   // rows past the ragged end are ZERO (0 * stale smem could be NaN)
    const int r = i / (A + 1), a = i - r * (A + 1);
    sd[r][a] = r < cnt ? (a < A ? __ldg(dlogits + (size_t)(n0 + r) * A + a) : __ldg(dbaseline + n0 + r)) : 0.f;
  }
  __syncthreads();
  if (j > H) return;
  float acc[HEAD_MAX_A + 1];
#pragma unroll
  for (int a = 0; a <= HEAD_MAX_A; ++a) acc[a] = 0.f;
  for (int r = 0; r < cnt; ++r) {
    const float x = j < H ? __ldg(X + (size_t)(n0 + r) * H + j) : 1.f;     // j == H: the bias "ones" column
    float dx = 0.f;
#pragma unroll
    for (int a = 0; a < HEAD_MAX_A; ++a)
      if (a < A) { acc[a] = fmaf(sd[r][a], x, acc[a]); if (j < H) dx = fmaf(sd[r][a], __ldg(Wp + (size_t)a * H + j), dx); }
    acc[HEAD_MAX_A] = fmaf(sd[r][A], x, acc[HEAD_MAX_A]);
    if (j < H) dX[(size_t)(n0 + r) * H + j] = dx + sd[r][A] * __ldg(Wb + j);
  }
#pragma unroll
  for (int a = 0; a < HEAD_MAX_A; ++a)
    if (a < A) { if (j < H) atomicAdd(gWp + (size_t)a * H + j, acc[a]); else atomicAdd(gbp + a, acc[a]); }
  if (j < H) atomicAdd(gWb + j, acc[HEAD_MAX_A]); else atomicAdd(gbb, acc[HEAD_MAX_A]);
}
// dh[n][j] = bf16(dcore[n][j] * (h[n][j] > 0)), j < 512 (the reward / one-hot columns of core have no parameters below them)
__global__ void __launch_bounds__(128) dcore_to_dh_kernel(const float* __restrict__ dcore, const float* __restrict__ h, int A,
                                                          __nv_bfloat16* __restrict__ dh) {
  const int n = blockIdx.x, H = 513 + A;
  for (int j = threadIdx.x; j < 512; j += 128) {
    const float v = __ldg(h + (size_t)n * 512 + j) > 0.f ? __ldg(dcore + (size_t)n * H + j) : 0.f;
    dh[(size_t)n * 512 + j] = __float2bfloat16_rn(v);
  }
}

cudaError_t launch_core_build(const float* hpart, int nsplit, const float* bfc, const float* reward, const int64_t* action, int N, int A, float* h,
                              float* core, cudaStream_t st) {
  core_build_kernel<<<N, 128, 0, st>>>(hpart, nsplit, bfc, reward, action, N, A, h, core);
  return cudaGetLastError();
}
cudaError_t launch_head_dense_fwd(const float* X, const float* Wp, const float* bp, const float* Wb, const float* bb, int N, int A, float* logits,
                                  float* baseline, cudaStream_t st) {
  head_dense_fwd_kernel<<<(N + 7) / 8, 256, 0, st>>>(X, Wp, bp, Wb, bb, N, A, logits, baseline);
  return cudaGetLastError();
}
cudaError_t launch_head_dense_bwd(const float* X, const float* dlogits, const float* dbaseline, const float* Wp, const float* Wb, int N, int A,
                                  float* dX, float* gWp, float* gbp, float* gWb, float* gbb, cudaStream_t st) {
  const int H = 513 + A;
  head_dense_bwd_kernel<<<dim3((H + 1 + 127) / 128, (N + 15) / 16), 128, 0, st>>>(X, dlogits, dbaseline, Wp, Wb, N, A, dX, gWp, gbp, gWb, gbb);
  return cudaGetLastError();
}
cudaError_t launch_dcore_to_dh(const float* dcore, const float* h, int N, int A, __nv_bfloat16* dh, cudaStream_t st) {
  dcore_to_dh_kernel<<<N, 128, 0, st>>>(dcore, h, A, dh);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// trajectory-slot unpack: B slots (one contiguous record per actor rollout, all keys of create_buffers,
// impala_atari.py:135-147) copied host->device as they lie, then scattered into the time-major [T+1, B, ...] batch.
// grid = (T+1, B): one block moves one 28,224-byte frame with 16-byte vectors; thread 0 moves the scalars.
// ------------------------------------------------------------------------------------------------
struct SlotOffsets { int64_t obs, reward, done, action, policy_logits, episode_return; };
__global__ void __launch_bounds__(256) unpack_slots_kernel(const uint8_t* __restrict__ staging, int64_t slot_bytes, SlotOffsets o, int B, int A,
                                                           uint8_t* __restrict__ obs, float* __restrict__ reward, uint8_t* __restrict__ done,
                                                           int64_t* __restrict__ action, float* __restrict__ logits,
                                                           float* __restrict__ episode_return) {
  const int t = blockIdx.x, b = blockIdx.y;
  const uint8_t* slot = staging + (size_t)b * slot_bytes;
  const uint4* src = reinterpret_cast<const uint4*>(slot + o.obs + (size_t)t * 28224);
  uint4* dst = reinterpret_cast<uint4*>(obs + ((size_t)t * B + b) * 28224);
  for (int i = threadIdx.x; i < 1764; i += 256) dst[i] = __ldg(src + i);
  const size_t n = (size_t)t * B + b;
  if (threadIdx.x == 0) {
    reward[n] = reinterpret_cast<const float*>(slot + o.reward)[t];
    done[n] = (slot + o.done)[t];
    action[n] = reinterpret_cast<const int64_t*>(slot + o.action)[t];
    if (episode_return) episode_return[n] = reinterpret_cast<const float*>(slot + o.episode_return)[t];
  }
  if (threadIdx.x >= 32 && threadIdx.x < 32 + A) logits[n * A + threadIdx.x - 32] = reinterpret_cast<const float*>(slot + o.policy_logits)[t * A + threadIdx.x - 32];
}

cudaError_t launch_unpack_slots(const uint8_t* staging, int64_t slot_bytes, const int64_t* off6, int T, int B, int A, uint8_t* obs, float* reward,
                                uint8_t* done, int64_t* action, float* logits, float* episode_return, cudaStream_t st) {
  SlotOffsets o{off6[0], off6[1], off6[2], off6[3], off6[4], off6[5]};
  unpack_slots_kernel<<<dim3(T + 1, B), 256, 0, st>>>(staging, slot_bytes, o, B, A, obs, reward, done, action, logits, episode_return);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
cudaError_t launch_head_fwd(const float* hpart, int nsplit, const float* bfc, float* h, const float* reward, const int64_t* action,
                            const float* Wp, const float* bp, const float* Wb, const float* bb, int N, int A, float* logits,
                            float* baseline, cudaStream_t st) {
  if (N <= 0) return cudaSuccess;
  return launch_chain(head_fwd_kernel, dim3((N + 1) / 2), dim3(256), 0, st, hpart, nsplit, bfc, h, reward, action, Wp, bp, Wb, bb, N, A, logits, baseline);
  return cudaGetLastError();
}
cudaError_t launch_head_bwd(const float* dlogits, const float* dbaseline, const float* h, const float* reward, const int64_t* action,
                            const float* Wp, const float* Wb, int N, int A, __nv_bfloat16* dh, float* gWp, float* gbp, float* gWb,
                            float* gbb, float* part, cudaStream_t st, cudaStream_t st_wgrad, bool do_dh, __nv_bfloat16* dh_lo) {
  if (N <= 0) return cudaSuccess;
  if (do_dh) SRL_TRY(launch_chain(head_bwd_dh_kernel, dim3(N, 4), dim3(128), 0, st, dlogits, dbaseline, h, Wp, Wb, N, A, dh, dh_lo));
  const int CORE = 513 + A;
  // the head weight gradients only feed the optimizer: they may run on a side stream (st_wgrad) beside the fc backward
  const int nslab = (N + HEAD_SLAB - 1) / HEAD_SLAB, spg = (nslab + HEAD_GROUPS - 1) / HEAD_GROUPS, groups = (nslab + spg - 1) / spg;
  head_wgrad_kernel<<<dim3((CORE + 1 + 127) / 128, groups), 128, 0, st_wgrad>>>(dlogits, dbaseline, h, reward, action, N, A, spg, part);
  head_wgrad_reduce_kernel<<<((A + 1) * (CORE + 1) + 255) / 256, 256, 0, st_wgrad>>>(part, groups, A, gWp, gbp, gWb, gbb);
  return cudaGetLastError();
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
                        int step, int* dstep, cudaStream_t st) {
  if (dstep) adam_step_inc_kernel<<<1, 1, 0, st>>>(dstep);
  adam_kernel<<<ew_blocks(n * 4), 256, 0, st>>>(p, g, m, v, n, coef, lr, b1, b2, eps, step, dstep);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// clip_grad_norm_ + optimizer step as ONE cooperative kernel (impala_atari.py:344-346): phase 1 sums g^2 (block partials
// in a fixed slot each), grid barrier, every block adds the partials in the same fixed order (deterministic, identical
// in all blocks), phase 2 applies the clipped update (g is re-read from L2).  OPT 0 = RMSprop, 1 = Adam.
// ------------------------------------------------------------------------------------------------
template <int OPT>
__global__ void __launch_bounds__(512) clip_optim_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ s0,
                                                         float* __restrict__ s1, int64_t n, float max_norm, float* __restrict__ coef,
                                                         float* __restrict__ scratch, float lr, float a, float b, float eps, int step,
                                                         int* __restrict__ dstep) {
  cg::grid_group grid = cg::this_grid();
  pdl_wait(52);    // (cooperative launch, no attribute: returns at once; names the kernel in the diagnostics timeline)
  const int64_t n4 = n >> 2, stride = (int64_t)gridDim.x * blockDim.x, i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int t = dstep ? *dstep + 1 : step;          // 1-based step count: Adam bias correction; counted for RMSprop too (checkpoints)
  // The thread's first HOLD float4 of g (and, for RMSprop, of p and the state) stay in registers across the grid barrier: phase 2 then
  // starts from registers instead of paying a second round of L2 / HBM latency (the grid covers n with <= HOLD items per thread).
  constexpr int HOLD = 2;
  float4 gh[HOLD], ph[HOLD], vh[HOLD];
  float s = 0.f;
#pragma unroll
  for (int h = 0; h < HOLD; ++h) {
    const int64_t i = i0 + h * stride;
    if (i < n4) {
      gh[h] = reinterpret_cast<const float4*>(g)[i];
      if (OPT == 0) { ph[h] = reinterpret_cast<const float4*>(p)[i]; vh[h] = reinterpret_cast<const float4*>(s0)[i]; }
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
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float tsum = 0.f;
    for (int w = 0; w < 16; ++w) tsum += red[w];
    scratch[4 + blockIdx.x] = tsum;
  }
  grid.sync();
  if (threadIdx.x < 32) {
    double tsum = 0.0;
    for (unsigned k = threadIdx.x; k < gridDim.x; k += 32) tsum += (double)__ldcg(scratch + 4 + k);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) tsum += __shfl_xor_sync(0xffffffffu, tsum, o);
    if (threadIdx.x == 0) {
      const float norm = (float)sqrt(tsum);
      const float c = max_norm >= 0.f ? fminf(max_norm / (norm + 1e-6f), 1.0f) : 1.0f;
      c_sh = c;
      if (blockIdx.x == 0) {
        coef[0] = norm; coef[1] = c;
        if (dstep) *dstep = t;
      }
    }
  }
  __syncthreads();
  const float c = c_sh;
  if (OPT == 0) {
#pragma unroll
    for (int h = 0; h < HOLD; ++h) {
      const int64_t i = i0 + h * stride;
      if (i < n4) {
        float4 pp = ph[h], vv = vh[h];
        const float4 gg = gh[h];
        float* P = &pp.x; float* V = &vv.x; const float* G = &gg.x;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float gk = G[k] * c;
          V[k] = a * V[k] + (1.f - a) * gk * gk;
          P[k] = P[k] - lr * (gk / (sqrtf(V[k]) + eps));
        }
        reinterpret_cast<float4*>(p)[i] = pp;
        reinterpret_cast<float4*>(s0)[i] = vv;
      }
    }
    for (int64_t i = i0 + HOLD * stride; i < n4; i += stride) {
      float4 pp = reinterpret_cast<float4*>(p)[i], vv = reinterpret_cast<float4*>(s0)[i];
      const float4 gg = reinterpret_cast<const float4*>(g)[i];
      float* P = &pp.x; float* V = &vv.x; const float* G = &gg.x;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float gk = G[k] * c;
        V[k] = a * V[k] + (1.f - a) * gk * gk;
        P[k] = P[k] - lr * (gk / (sqrtf(V[k]) + eps));
      }
      reinterpret_cast<float4*>(p)[i] = pp;
      reinterpret_cast<float4*>(s0)[i] = vv;
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
      const int64_t i = n4 * 4 + threadIdx.x;
      const float gk = g[i] * c;
      s0[i] = a * s0[i] + (1.f - a) * gk * gk;
      p[i] = p[i] - lr * (gk / (sqrtf(s0[i]) + eps));
    }
  } else {
    const float inv_bc1 = 1.0f / (float)(1.0 - pow((double)a, (double)t));
    const float inv_sqrt_bc2 = 1.0f / sqrtf((float)(1.0 - pow((double)b, (double)t)));
    for (int64_t i = i0; i < n; i += stride) {
      const float gk = g[i] * c;
      const float mk = a * s0[i] + (1.f - a) * gk;
      const float vk = b * s1[i] + (1.f - b) * gk * gk;
      s0[i] = mk; s1[i] = vk;
      p[i] = p[i] - (lr * inv_bc1) * (mk / (sqrtf(vk) * inv_sqrt_bc2 + eps));
    }
  }
}

SRL_KSTAMP_SETTER(kstamp_set_heads)

template <int OPT>
static cudaError_t launch_clip_optim_t(float* p, float* g, float* s0, float* s1, int64_t n, float max_norm, float* coef, float* scratch,
                                       float lr, float a, float b, float eps, int step, int* dstep, cudaStream_t st) {
  static int per_sm_dev[64] = {}, sms_dev[64] = {};      // per device: one process may drive several GPUs
  int dev = 0;
  SRL_TRY(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
  if (!per_sm_dev[dev]) {
    int sm_count = 0, occ = 0;
    SRL_TRY(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev));
    SRL_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, clip_optim_kernel<OPT>, 512, 0));
    if (occ < 1) return cudaErrorLaunchOutOfResources;
    sms_dev[dev] = sm_count; per_sm_dev[dev] = occ;
  }
  const int per_sm = per_sm_dev[dev], sms = sms_dev[dev];
  int64_t need = (n / 4 + 511) / 512;
  int blocks = (int)(need < 1 ? 1 : need);
  int cap = per_sm * sms; if (cap > 592) cap = 592;          // scratch holds 592 partials
  if (blocks > cap) blocks = cap;
  void* args[] = {&p, &g, &s0, &s1, &n, &max_norm, &coef, &scratch, &lr, &a, &b, &eps, &step, &dstep};
  return cudaLaunchCooperativeKernel((const void*)clip_optim_kernel<OPT>, dim3(blocks), dim3(512), args, 0, st);
}
cudaError_t launch_clip_optim(int optimizer, float* p, float* g, float* s0, float* s1, int64_t n, float max_norm, float* coef,
                              float* scratch, float lr, float a, float b, float eps, int step, int* dstep, cudaStream_t st) {
  return optimizer == 0 ? launch_clip_optim_t<0>(p, g, s0, s1, n, max_norm, coef, scratch, lr, a, b, eps, step, dstep, st)
                        : launch_clip_optim_t<1>(p, g, s0, s1, n, max_norm, coef, scratch, lr, a, b, eps, step, dstep, st);
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
template <int OPT, bool NVLS>
__global__ void __launch_bounds__(512) dp_clip_optim_kernel(float* __restrict__ p, float* g, float* __restrict__ s0, float* __restrict__ s1,
                                                            int64_t n, float max_norm, float* coef, float* scratch, float lr, float a,
                                                            float b, float eps, int step, int* dstep, const DpPeers P) {
  cg::grid_group grid = cg::this_grid();
  const int64_t n4 = n >> 2, stride = (int64_t)gridDim.x * blockDim.x, i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int W = P.world, R = P.rank;
  const int64_t chunk = (n4 + W - 1) / W, lo = R * chunk, hi = min(n4, lo + chunk);
  const int t = dstep ? *reinterpret_cast<volatile int*>(dstep) + 1 : step;
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
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float tsum = 0.f;
    for (int w = 0; w < 16; ++w) tsum += red[w];
    scratch[4 + blockIdx.x] = tsum;
    // the slice stores are local: the grid barrier makes them visible at L2, which is where the peers' NVLink loads land
  }
  grid.sync();
  // ---- barrier 2: all slices pushed everywhere, per-slice sums of squares published
  if (blockIdx.x == 0) {
    if (threadIdx.x < 32) {
      double tsum = 0.0;
      for (unsigned k = threadIdx.x; k < gridDim.x; k += 32) tsum += (double)__ldcg(scratch + 4 + k);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) tsum += __shfl_xor_sync(0xffffffffu, tsum, o);
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
    const float c = max_norm >= 0.f ? fminf(max_norm / (norm + 1e-6f), 1.0f) : 1.0f;     // identical in every block of every rank
    c_sh = c;
    if (blockIdx.x == 0) { coef[0] = norm; coef[1] = c; }
  }
  __syncthreads();
  const float c = c_sh;
  // ---- phase 2: clip + optimizer on my replica; the gradient buffer is local and fully reduced now
  float inv_bc1 = 0.f, inv_sqrt_bc2 = 0.f;
  if (OPT == 1) {
    inv_bc1 = 1.0f / (float)(1.0 - pow((double)a, (double)t));
    inv_sqrt_bc2 = 1.0f / sqrtf((float)(1.0 - pow((double)b, (double)t)));
  }
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
      float* Pp = &pp.x; float* V = &vv.x; const float* G = &gg.x;
      if (OPT == 0) {
  #pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float gk = G[k] * c;
          V[k] = a * V[k] + (1.f - a) * gk * gk;
          Pp[k] = Pp[k] - lr * (gk / (sqrtf(V[k]) + eps));
        }
      } else {
        float4 ww = reinterpret_cast<float4*>(s1)[i];
        float* Wv = &ww.x;
  #pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float gk = G[k] * c;
          V[k] = a * V[k] + (1.f - a) * gk;                    // exp_avg
          Wv[k] = b * Wv[k] + (1.f - b) * gk * gk;             // exp_avg_sq
          Pp[k] = Pp[k] - (lr * inv_bc1) * (V[k] / (sqrtf(Wv[k]) * inv_sqrt_bc2 + eps));
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
      s0[i] = a * s0[i] + (1.f - a) * gk * gk;
      p[i] = p[i] - lr * (gk / (sqrtf(s0[i]) + eps));
    } else {
      const float mk = a * s0[i] + (1.f - a) * gk, vk = b * s1[i] + (1.f - b) * gk * gk;
      s0[i] = mk; s1[i] = vk;
      p[i] = p[i] - (lr * inv_bc1) * (mk / (sqrtf(vk) * inv_sqrt_bc2 + eps));
    }
  }
  // no closing barrier: after barrier 2 no rank touches another rank's memory until the next step's barrier 1
}

template <int OPT, bool NVLS>
static cudaError_t launch_dp_clip_optim_t(float* p, float* g, float* s0, float* s1, int64_t n, float max_norm, float* coef, float* scratch,
                                          float lr, float a, float b, float eps, int step, int* dstep, DpPeers P, cudaStream_t st) {
  static int per_sm_dev[64] = {}, sms_dev[64] = {};      // per device: one process may drive several GPUs
  int dev = 0;
  SRL_TRY(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
  if (!per_sm_dev[dev]) {
    int sm_count = 0, occ = 0;
    SRL_TRY(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev));
    SRL_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, (dp_clip_optim_kernel<OPT, NVLS>), 512, 0));
    if (occ < 1) return cudaErrorLaunchOutOfResources;
    sms_dev[dev] = sm_count; per_sm_dev[dev] = occ;
  }
  const int per_sm = per_sm_dev[dev], sms = sms_dev[dev];
  int64_t need = (n / 4 + 511) / 512;
  int blocks = (int)(need < 1 ? 1 : need);
  int cap = per_sm * sms; if (cap > 592) cap = 592;
  if (blocks > cap) blocks = cap;
  void* args[] = {&p, &g, &s0, &s1, &n, &max_norm, &coef, &scratch, &lr, &a, &b, &eps, &step, &dstep, &P};
  return cudaLaunchCooperativeKernel((const void*)dp_clip_optim_kernel<OPT, NVLS>, dim3(blocks), dim3(512), args, 0, st);
}
// Weight-publish snapshot (impala_atari.py:348): dst = src when the step's total loss is finite, else dst keeps the last good
// weights -- so the asynchronous D2H that follows never hands poisoned parameters to the actors.
__global__ void __launch_bounds__(256) snapshot_if_finite_kernel(float4* __restrict__ dst, const float4* __restrict__ src, int64_t n4,
                                                                 const float* __restrict__ losses) {
  if (losses) {
    const float t = losses[3];
    if (!(fabsf(t) <= 3.0e38f)) return;          // NaN or Inf: keep the previous snapshot
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

cudaError_t launch_dp_clip_optim(int optimizer, float* p, float* g, float* s0, float* s1, int64_t n, float max_norm, float* coef,
                                 float* scratch, float lr, float a, float b, float eps, int step, int* dstep, const DpPeers& P,
                                 cudaStream_t st) {
  if (P.mc_g)
    return optimizer == 0 ? launch_dp_clip_optim_t<0, true>(p, g, s0, s1, n, max_norm, coef, scratch, lr, a, b, eps, step, dstep, P, st)
                          : launch_dp_clip_optim_t<1, true>(p, g, s0, s1, n, max_norm, coef, scratch, lr, a, b, eps, step, dstep, P, st);
  return optimizer == 0 ? launch_dp_clip_optim_t<0, false>(p, g, s0, s1, n, max_norm, coef, scratch, lr, a, b, eps, step, dstep, P, st)
                        : launch_dp_clip_optim_t<1, false>(p, g, s0, s1, n, max_norm, coef, scratch, lr, a, b, eps, step, dstep, P, st);
}

}  // namespace srl
