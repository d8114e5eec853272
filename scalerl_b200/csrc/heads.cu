// fp32 CUDA-core kernels around the encoder:
//   * policy / baseline heads forward + backward (atari_model.py:104-107,126-127 and their autograd)
//   * the heads of the LSTM path (use_lstm) and the assembly of its input
//   * the trajectory-slot unpack
#include "common.cuh"
#include "kernels.h"
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
// dh[n][j] = bf16(dcore[n][j] * (h[n][j] > 0)), j < 512 (the reward / one-hot columns of core have no parameters below them);
// dh_lo (when not null) = the low twin bf16(v - bf16(v)) of the fp32-accurate operand mode
__global__ void __launch_bounds__(128) dcore_to_dh_kernel(const float* __restrict__ dcore, const float* __restrict__ h, int A,
                                                          __nv_bfloat16* __restrict__ dh, __nv_bfloat16* __restrict__ dh_lo) {
  const int n = blockIdx.x, H = 513 + A;
  for (int j = threadIdx.x; j < 512; j += 128) {
    const float v = __ldg(h + (size_t)n * 512 + j) > 0.f ? __ldg(dcore + (size_t)n * H + j) : 0.f;
    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
    dh[(size_t)n * 512 + j] = hi;
    if (dh_lo) dh_lo[(size_t)n * 512 + j] = __float2bfloat16_rn(v - __bfloat162float(hi));
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
cudaError_t launch_dcore_to_dh(const float* dcore, const float* h, int N, int A, __nv_bfloat16* dh, cudaStream_t st, __nv_bfloat16* dh_lo) {
  dcore_to_dh_kernel<<<N, 128, 0, st>>>(dcore, h, A, dh, dh_lo);
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

SRL_KSTAMP_SETTER(kstamp_set_heads)

}  // namespace srl
