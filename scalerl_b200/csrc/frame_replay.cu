// GPU prioritized replay memory that stores each 84x84 frame once (Ape-X path): the transitions, sampling and outputs of replay.cu, with
// the frame stacks replaced by handles into a FIFO pool of frames.  In an Atari stream consecutive stacks share three of their four
// frames and next_state of step t is state of step t + 1, so a stream that continues an episode adds one 7,056-byte frame per env step
// where replay.cu stores two 28,224-byte stacks.
//   pool:  frame_capacity (F) frames; the frame of 64-bit sequence number s lives at s mod F, and s is live while s >= head - F.
//   slot:  ring slot i (leaf i of the memory's sampler) holds the 8 sequence numbers of its state and next_state stacks, the oldest of
//          them, and action, reward and done as replay.cu stores them.  The staging window holds handles; the fold copies handles.
// An add dedups the step's 8 incoming frames per env byte for byte (frame_dedup_kernel), numbers the new ones by an exclusive scan in env
// order (frame_assign_kernel), retires every slot whose oldest frame the new ones overwrite (frame_retire_scan_kernel + per_retire),
// writes the new frames (frame_place_kernel) and folds (frame_fold_kernel, replay.cu's reward and done arithmetic).  Gathers rebuild
// each stack from its 4 frame addresses.  All of it is HBM-bound byte movement on 16-byte vectors, no tensor cores.
#include <math.h>
#include <new>
#include "common.cuh"
#include "errors.h"
#include "kernels.h"
#include "replay.cuh"
#include "../../include/scalerl_b200.h"

namespace srl {

constexpr int64_t FRAME_BYTES = 84 * 84;                   // one u8 frame: 7,056 B
constexpr int FRAME_VEC = (int)(FRAME_BYTES / 16);         // 441 16-byte vectors
constexpr int HANDLES = 8;                                 // frames of a (state, next_state) pair: state 0..3, then next_state 0..3
constexpr int DEDUP_THREADS = 256;
constexpr int PLACE_THREADS = 448;                         // one vector per thread
constexpr int FOLD_THREADS_F = 256;
constexpr int RETIRE_THREADS = 256, RETIRE_BLOCKS = 1056;
constexpr int FG_THREADS = 256, FG_VPT = 2;                // 16-byte vectors per thread, all loaded before any is stored
constexpr int FG_CHUNKS = (ROW_PAIR_VEC + FG_THREADS * FG_VPT - 1) / (FG_THREADS * FG_VPT);   // CTAs per transition
constexpr int64_t SEQ_NONE = INT64_MAX;                    // the oldest frame of a slot never written

// device-resident counters of the pool
struct FrameState {
  int64_t head;                    // frames written since creation: the sequence number of the next new frame
  int64_t limit;                   // head - F after the current add's frames: frames below it are overwritten
  unsigned long long n_retire;     // slots the current add retires (the first n_retire entries of the retire list)
  unsigned long long retired;      // slots retired since creation
};

// The transition fields: the ring ([M] rows, h [M][8]) and the staging window ([n_step][E] rows, h [n_step][E][8]; oldest unused).
struct FrameSlots {
  int64_t* h;
  int64_t* oldest;
  int64_t* action;
  float* reward;
  uint8_t* done;
};

// frame j (0..7) of env e's incoming (state, next_state) pair in the staging buffers [E][4][441] each
__device__ __forceinline__ const uint4* staged_frame(const uint4* stage_s, const uint4* stage_ns, int e, int j) {
  return (j < 4 ? stage_s : stage_ns) + ((int64_t)e * 4 + (j & 3)) * FRAME_VEC;
}

// byte equality of two frames, by the whole block (every thread gets the answer)
__device__ __forceinline__ bool frames_equal(const uint4* __restrict__ a, const uint4* __restrict__ b) {
  bool diff = false;
  for (int i = threadIdx.x; i < FRAME_VEC; i += blockDim.x) {
    const uint4 u = a[i], v = b[i];
    diff |= (u.x != v.x) | (u.y != v.y) | (u.z != v.z) | (u.w != v.w);
  }
  return !__syncthreads_or(diff);
}

// Block e: each of the env's 8 incoming frames, in order, is compared byte for byte with
//   1. the frames of this call already placed for the env (state 0..3, then next_state 0..3): the first equal one gives its handle;
//   2. else the env's previous next_state frames (prev_h, NULL on the first add), newest first, each only while it is sure to outlive
//      this step's stay in the window: s >= head + 8 E n_step - F (the adds the window spans write at most 8 E frames each);
//   3. else the frame is new.
// ref[e][j] = the reused sequence number, or -(k + 1) for the env's k-th new frame; count[e] = the env's new frames.  A frame equal to an
// earlier frame of this call that was itself a reuse finds the same handle in step 2, so step 1 only compares with new frames.
__global__ void __launch_bounds__(DEDUP_THREADS) frame_dedup_kernel(const uint4* __restrict__ stage_s, const uint4* __restrict__ stage_ns,
                                                                    const uint4* __restrict__ pool, int64_t F, const int64_t* __restrict__ prev_h,
                                                                    const FrameState* __restrict__ st, int E, int n_step, int64_t* __restrict__ ref,
                                                                    int* __restrict__ count) {
  const int e = blockIdx.x;
  __shared__ int64_t sref[HANDLES];
  const int64_t keep_from = st->head + (int64_t)HANDLES * E * n_step - F;
  int fresh = 0;
  for (int j = 0; j < HANDLES; ++j) {
    const uint4* x = staged_frame(stage_s, stage_ns, e, j);
    int64_t r = 0;
    bool found = false;
    for (int c = 0; c < j && !found; ++c)
      if (sref[c] < 0 && frames_equal(x, staged_frame(stage_s, stage_ns, e, c))) { r = sref[c]; found = true; }
    if (prev_h)
      for (int k = 3; k >= 0 && !found; --k) {
        const int64_t s = prev_h[(int64_t)e * HANDLES + 4 + k];
        if (s >= keep_from && frames_equal(x, pool + (s % F) * FRAME_VEC)) { r = s; found = true; }
      }
    if (!found) r = -(++fresh);
    if (threadIdx.x == 0) { sref[j] = r; ref[(int64_t)e * HANDLES + j] = r; }
    __syncthreads();
  }
  if (threadIdx.x == 0) count[e] = fresh;
}

// One block: the env's first new frame gets sequence number head + (new frames of envs 0 .. e-1), an exclusive scan in env order, so
// the pool's layout does not depend on scheduling.  Writes this step's window handles, then head, limit and the retire count.
__global__ void __launch_bounds__(1024) frame_assign_kernel(const int64_t* __restrict__ ref, const int* __restrict__ count, int E, int64_t F,
                                                            FrameState* __restrict__ st, int64_t* __restrict__ win_h) {
  __shared__ int64_t warp_sum[32];
  __shared__ int64_t carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t head = st->head;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int o = 0; o < E; o += 1024) {
    const int e = o + threadIdx.x;
    const int64_t c = e < E ? count[e] : 0;
    int64_t x = c;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int64_t y = __shfl_up_sync(0xffffffffu, x, d);
      if (lane >= d) x += y;
    }
    if (lane == 31) warp_sum[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int64_t w = warp_sum[lane];
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int64_t y = __shfl_up_sync(0xffffffffu, w, d);
        if (lane >= d) w += y;
      }
      warp_sum[lane] = w;
    }
    __syncthreads();
    const int64_t base = head + carry + (warp ? warp_sum[warp - 1] : 0) + x - c;
    if (e < E)
      for (int j = 0; j < HANDLES; ++j) {
        const int64_t r = ref[(int64_t)e * HANDLES + j];
        win_h[(int64_t)e * HANDLES + j] = r >= 0 ? r : base - r - 1;
      }
    __syncthreads();
    if (threadIdx.x == 0) carry += warp_sum[31];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    st->head = head + carry;
    st->limit = head + carry - F;
    st->n_retire = 0;
  }
}

// every live slot whose oldest frame lies below the limit joins the retire list (its order is irrelevant: per_retire's trees are a
// function of the set)
__global__ void __launch_bounds__(RETIRE_THREADS) frame_retire_scan_kernel(const int64_t* __restrict__ oldest, const uint8_t* __restrict__ retired,
                                                                           int64_t M, FrameState* __restrict__ st, int64_t* __restrict__ list) {
  const int64_t limit = st->limit;
  if (limit <= 0) return;                                  // nothing overwritten yet
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < M; s += (int64_t)gridDim.x * blockDim.x)
    if (oldest[s] < limit && !retired[s]) {
      list[atomicAdd(&st->n_retire, 1ull)] = s;
      atomicAdd(&st->retired, 1ull);
    }
}

// block (e, j): the env's frame j into the pool at its sequence number, if it is new
__global__ void __launch_bounds__(PLACE_THREADS) frame_place_kernel(const uint4* __restrict__ stage_s, const uint4* __restrict__ stage_ns,
                                                                    const int64_t* __restrict__ ref, const int64_t* __restrict__ win_h, int64_t F,
                                                                    uint4* __restrict__ pool) {
  const int e = blockIdx.x, j = blockIdx.y;
  if (ref[(int64_t)e * HANDLES + j] >= 0) return;
  const uint4* src = staged_frame(stage_s, stage_ns, e, j);
  uint4* dst = pool + (win_h[(int64_t)e * HANDLES + j] % F) * FRAME_VEC;
  if (threadIdx.x < FRAME_VEC) dst[threadIdx.x] = src[threadIdx.x];
}

// One n-step transition per env (one thread each) at ring slot (ptr + e) mod M: fold_reward_done's reward and done, the state handles
// of the oldest step and the next_state handles of the step the fold stopped at, and the oldest of the 8.
__global__ void __launch_bounds__(FOLD_THREADS_F) frame_fold_kernel(FrameSlots win, FrameSlots ring, int E, int n_step, int oldest,
                                                                    GammaPowers gp, int64_t ptr, int64_t M) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  float r;
  uint8_t d;
  const int stop = fold_reward_done(win.reward, win.done, E, e, n_step, oldest, gp, &r, &d);
  const int64_t slot = (ptr + e) % M;
  const int64_t* hs = win.h + ((int64_t)oldest * E + e) * HANDLES;
  const int64_t* hn = win.h + ((int64_t)stop * E + e) * HANDLES + 4;
  int64_t lo = SEQ_NONE;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int64_t a = hs[k], b = hn[k];
    ring.h[slot * HANDLES + k] = a;
    ring.h[slot * HANDLES + 4 + k] = b;
    lo = min(lo, min(a, b));
  }
  ring.oldest[slot] = lo;
  ring.action[slot] = win.action[(int64_t)oldest * E + e];
  ring.reward[slot] = r;
  ring.done[slot] = d;
}

// out row b = ring slot idxs[b] (blockIdx.x = b), each stack rebuilt from its 4 frames; blockIdx.y splits the row pair.  A slot outside
// [0, M) or retired leaves its output row as it was.
__global__ void __launch_bounds__(FG_THREADS) frame_gather_kernel(const uint4* __restrict__ pool, int64_t F, const int64_t* __restrict__ ring_h,
                                                                  const int64_t* __restrict__ ring_action, const float* __restrict__ ring_reward,
                                                                  const uint8_t* __restrict__ ring_done, const uint8_t* __restrict__ retired,
                                                                  int64_t M, const int64_t* __restrict__ idxs, uint4* __restrict__ out_s,
                                                                  uint4* __restrict__ out_ns, int64_t* __restrict__ action, float* __restrict__ reward,
                                                                  uint8_t* __restrict__ done) {
  __shared__ int64_t base[HANDLES];
  const int b = blockIdx.x;
  const int64_t slot = idxs[b];
  if (slot < 0 || slot >= M || retired[slot]) return;
  if (threadIdx.x < HANDLES) base[threadIdx.x] = (ring_h[slot * HANDLES + threadIdx.x] % F) * FRAME_VEC;
  __syncthreads();
  const int i0 = blockIdx.y * FG_THREADS * FG_VPT + threadIdx.x;
  uint4 v[FG_VPT];
#pragma unroll
  for (int k = 0; k < FG_VPT; ++k) {
    const int i = i0 + k * FG_THREADS;
    if (i < ROW_PAIR_VEC) {
      const int f = i / FRAME_VEC;
      v[k] = pool[base[f] + i - f * FRAME_VEC];
    }
  }
#pragma unroll
  for (int k = 0; k < FG_VPT; ++k) {
    const int i = i0 + k * FG_THREADS;
    if (i < OBS_VEC) out_s[(int64_t)b * OBS_VEC + i] = v[k];
    else if (i < ROW_PAIR_VEC) out_ns[(int64_t)b * OBS_VEC + i - OBS_VEC] = v[k];
  }
  if (blockIdx.y == 0 && threadIdx.x == 0) {
    action[b] = ring_action[slot];
    reward[b] = ring_reward[slot];
    done[b] = ring_done[slot];
  }
}

// stack row e (blockIdx.x) = the 4 frames of h[e * 8 + 0..3] (the state handles of a window step), u8 [E,4,84,84]
__global__ void __launch_bounds__(FG_THREADS) frame_stacks_kernel(const uint4* __restrict__ pool, int64_t F, const int64_t* __restrict__ h,
                                                                  uint4* __restrict__ out) {
  const int e = blockIdx.x;
  const int i = blockIdx.y * FG_THREADS + threadIdx.x;
  if (i >= OBS_VEC) return;
  const int f = i / FRAME_VEC;
  out[(int64_t)e * OBS_VEC + i] = pool[(h[(int64_t)e * HANDLES + f] % F) * FRAME_VEC + i - f * FRAME_VEC];
}

// a slot never written: handles 0 (a gather of it reads pool frame 0, never outside the pool), oldest SEQ_NONE (never retired), live
__global__ void frame_init_kernel(int64_t* h, int64_t* oldest, uint8_t* retired, int64_t M, FrameState* st, int64_t F) {
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < M; s += (int64_t)gridDim.x * blockDim.x) {
    for (int k = 0; k < HANDLES; ++k) h[s * HANDLES + k] = 0;
    oldest[s] = SEQ_NONE;
    retired[s] = 0;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *st = FrameState{0, -F, 0ull, 0ull};
}

}  // namespace srl
using namespace srl;

struct srl_frame_replay {
  srl_per_t* per;
  int64_t memory_size, frame_capacity;
  int num_envs, n_step;
  GammaPowers gp;
  float gamma_n;                   // fp32(gamma^n_step), as srl_replay's
  int64_t steps;                   // vector steps added so far (host-known: adds are host calls)
  void* arena;
  uint4 *pool, *stage_s, *stage_ns, *scratch;
  FrameSlots ring, win;
  uint8_t* retired;
  int64_t *ref, *retire_list;
  int* count;
  FrameState* st;
};

namespace {
// the pool, the ring's rows, the staging window's, then the add's work buffers
int frame_rows(srl_frame_replay* R, WsRow* t) {
  const int64_t M = R->memory_size, E = R->num_envs, W = (int64_t)R->n_step * E;
  int n = 0;
  t[n++] = ws_row("pool", R->frame_capacity * FRAME_VEC, &R->pool);
  t[n++] = ws_row("handles", M * HANDLES, &R->ring.h);
  t[n++] = ws_row("oldest", M, &R->ring.oldest);
  t[n++] = ws_row("action", M, &R->ring.action);
  t[n++] = ws_row("reward", M, &R->ring.reward);
  t[n++] = ws_row("done", M, &R->ring.done);
  t[n++] = ws_row("retired", M, &R->retired);
  t[n++] = ws_row("retire_list", M, &R->retire_list);
  t[n++] = ws_row("window.handles", W * HANDLES, &R->win.h);
  t[n++] = ws_row("window.action", W, &R->win.action);
  t[n++] = ws_row("window.reward", W, &R->win.reward);
  t[n++] = ws_row("window.done", W, &R->win.done);
  t[n++] = ws_row("stage.state", E * OBS_VEC, &R->stage_s);
  t[n++] = ws_row("stage.next_state", E * OBS_VEC, &R->stage_ns);
  t[n++] = ws_row("scratch", R->n_step > 1 ? E * OBS_VEC : 0, &R->scratch);     // the oldest step's states (prioritized add)
  t[n++] = ws_row("ref", E * HANDLES, &R->ref);
  t[n++] = ws_row("count", E, &R->count);
  t[n++] = ws_row("state", 1, &R->st);
  return n;
}
constexpr int FRAME_ROWS = 18;

// the gather's outputs, as srl_replay_gather's
int check_outputs(const char* what, int64_t n, const int64_t* idxs, bool idxs_out, const uint8_t* state, const int64_t* action, const float* reward,
                  const uint8_t* next_state, const uint8_t* done, const float* weights) {
  REQ(state && action && reward && next_state && done, "%s: NULL output", what);
  REQ(!misaligned(state, 16) && !misaligned(next_state, 16), "%s: state / next_state must be 16-byte aligned", what);
  const Span s[] = {{idxs, n * 8, idxs_out, "idxs"}, {state, n * OBS_BYTES, true, "state"}, {action, n * 8, true, "action"},
                    {reward, n * 4, true, "reward"}, {next_state, n * OBS_BYTES, true, "next_state"}, {done, n, true, "done"},
                    {weights, n * 4, true, "weights"}};
  return check_spans(s, 7, what);
}
cudaError_t launch_gather(srl_frame_replay* R, const int64_t* idxs, int64_t n, uint8_t* state, int64_t* action, float* reward,
                          uint8_t* next_state, uint8_t* done, cudaStream_t st) {
  frame_gather_kernel<<<dim3((unsigned)n, FG_CHUNKS), FG_THREADS, 0, st>>>(R->pool, R->frame_capacity, R->ring.h, R->ring.action, R->ring.reward,
                                                                           R->ring.done, R->retired, R->memory_size, idxs,
                                                                           reinterpret_cast<uint4*>(state), reinterpret_cast<uint4*>(next_state),
                                                                           action, reward, done);
  return cudaGetLastError();
}
}  // namespace

extern "C" int srl_frame_replay_create(int64_t memory_size, int num_envs, int n_step, double gamma, double alpha, int64_t frame_capacity,
                                       srl_frame_replay_t** out) {
  REQ(out, "frame_replay_create: out is NULL");
  REQ(memory_size >= 2 && memory_size <= (int64_t(1) << 30), "frame_replay_create: memory_size must be in [2, 2^30], got %lld",
      (long long)memory_size);
  REQ(num_envs >= 1 && num_envs <= MAX_FRAMES && num_envs <= memory_size, "frame_replay_create: num_envs must be in [1, min(%d, memory_size)], got %d",
      MAX_FRAMES, num_envs);
  REQ(n_step >= 1 && n_step <= REPLAY_MAX_NSTEP, "frame_replay_create: n_step must be in [1, %d], got %d", REPLAY_MAX_NSTEP, n_step);
  REQ(isfinite(gamma), "frame_replay_create: gamma must be finite");
  const int64_t min_frames = (int64_t)HANDLES * num_envs * (n_step + 1);
  REQ(frame_capacity >= min_frames && frame_capacity <= (int64_t(1) << 32),
      "frame_replay_create: frame_capacity must be in [8 num_envs (n_step + 1) = %lld, 2^32], got %lld", (long long)min_frames,
      (long long)frame_capacity);
  srl_frame_replay* R = new (std::nothrow) srl_frame_replay();
  REQ(R, "out of memory");
  R->memory_size = memory_size; R->frame_capacity = frame_capacity; R->num_envs = num_envs; R->n_step = n_step; R->steps = 0;
  for (int k = 0; k < REPLAY_MAX_NSTEP; ++k) R->gp.g[k] = (float)pow(gamma, (double)k);    // numpy's float32(gamma ** k)
  R->gamma_n = (float)pow(gamma, (double)n_step);
  WsRow t[FRAME_ROWS];
  const int nrows = frame_rows(R, t);
  const int64_t bytes = rows_bytes(t, nrows, false);
  cudaError_t e = cudaMalloc(&R->arena, bytes);
  if (e != cudaSuccess) {
    cudaGetLastError();
    delete R;
    return fail((int)e, "frame_replay_create: cudaMalloc of %lld bytes (%lld frames of %lld B, %lld slots, %d x %d staged) failed: %s",
                (long long)bytes, (long long)frame_capacity, (long long)FRAME_BYTES, (long long)memory_size, n_step, num_envs, cudaGetErrorString(e));
  }
  carve_rows(t, nrows, false, static_cast<char*>(R->arena));
  frame_init_kernel<<<(unsigned)((memory_size + 255) / 256 < 4096 ? (memory_size + 255) / 256 : 4096), 256>>>(R->ring.h, R->ring.oldest, R->retired, memory_size,
                                                                                                             R->st, frame_capacity);
  e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { cudaFree(R->arena); delete R; return cuda_fail(e, "frame_replay_create: init"); }
  const int rc = srl_per_create(memory_size, alpha, &R->per);
  if (rc) { cudaFree(R->arena); delete R; return rc; }
  per_attach_retired(R->per, R->retired);
  *out = R;
  return 0;
}

extern "C" int srl_frame_replay_destroy(srl_frame_replay_t* R) {
  if (R) { srl_per_destroy(R->per); cudaFree(R->arena); delete R; }
  return 0;
}
extern "C" int64_t srl_frame_replay_size(const srl_frame_replay_t* R) { return R ? srl_per_size(R->per) : 0; }
extern "C" srl_per_t* srl_frame_replay_per(srl_frame_replay_t* R) { return R ? R->per : nullptr; }

namespace {
// one vector step: its stacks into the staging buffers and its fields into the window, the frames deduplicated, numbered and placed
// (retiring the slots whose frames they overwrite), and, once the window is full, the fold into ring slots (ptr + e) mod M.  *oldest:
// the window slot the fold took state and action from, -1 while the window is filling
int frame_stage_and_fold(srl_frame_replay* R, const uint8_t* state, const int64_t* action, const float* reward, const uint8_t* next_state,
                         const uint8_t* done, cudaStream_t st, int* oldest) {
  const int E = R->num_envs, n = R->n_step;
  const int64_t w = (R->steps % n) * E;                       // this vector step's window slot
  const int64_t F = R->frame_capacity;
  CU(cudaMemcpyAsync(R->stage_s, state, E * OBS_BYTES, cudaMemcpyDefault, st), "frame_replay_add: copy state");
  CU(cudaMemcpyAsync(R->stage_ns, next_state, E * OBS_BYTES, cudaMemcpyDefault, st), "frame_replay_add: copy next_state");
  CU(cudaMemcpyAsync(R->win.action + w, action, E * sizeof(int64_t), cudaMemcpyDefault, st), "frame_replay_add: copy action");
  CU(cudaMemcpyAsync(R->win.reward + w, reward, E * sizeof(float), cudaMemcpyDefault, st), "frame_replay_add: copy reward");
  CU(cudaMemcpyAsync(R->win.done + w, done, E, cudaMemcpyDefault, st), "frame_replay_add: copy done");
  const int64_t* prev_h = R->steps > 0 ? R->win.h + ((R->steps - 1) % n) * E * HANDLES : nullptr;
  frame_dedup_kernel<<<E, DEDUP_THREADS, 0, st>>>(R->stage_s, R->stage_ns, R->pool, F, prev_h, R->st, E, n, R->ref, R->count);
  CU(cudaGetLastError(), "frame_replay_add: dedup");
  frame_assign_kernel<<<1, 1024, 0, st>>>(R->ref, R->count, E, F, R->st, R->win.h + w * HANDLES);
  CU(cudaGetLastError(), "frame_replay_add: assign");
  const int64_t rb = (R->memory_size + RETIRE_THREADS - 1) / RETIRE_THREADS;
  frame_retire_scan_kernel<<<(unsigned)(rb < RETIRE_BLOCKS ? rb : RETIRE_BLOCKS), RETIRE_THREADS, 0, st>>>(R->ring.oldest, R->retired, R->memory_size,
                                                                                                         R->st, R->retire_list);
  CU(cudaGetLastError(), "frame_replay_add: retire scan");
  int rc = per_retire(R->per, R->retire_list, &R->st->n_retire, st);
  if (rc) return rc;
  frame_place_kernel<<<dim3(E, HANDLES), PLACE_THREADS, 0, st>>>(R->stage_s, R->stage_ns, R->ref, R->win.h + w * HANDLES, F, R->pool);
  CU(cudaGetLastError(), "frame_replay_add: place");
  R->steps++;
  *oldest = -1;
  if (R->steps < n) return 0;
  *oldest = (int)(R->steps % n);
  frame_fold_kernel<<<(E + FOLD_THREADS_F - 1) / FOLD_THREADS_F, FOLD_THREADS_F, 0, st>>>(R->win, R->ring, E, n, *oldest, R->gp,
                                                                                         per_tree_ptr(R->per), R->memory_size);
  CU(cudaGetLastError(), "frame_replay_add: fold");
  return 0;
}
}  // namespace

extern "C" int srl_frame_replay_add(srl_frame_replay_t* R, const uint8_t* state, const int64_t* action, const float* reward,
                                    const uint8_t* next_state, const uint8_t* done, void* stream) {
  REQ(R && state && action && reward && next_state && done, "frame_replay_add: NULL pointer");
  int oldest;
  const int rc = frame_stage_and_fold(R, state, action, reward, next_state, done, (cudaStream_t)stream, &oldest);
  if (rc || oldest < 0) return rc;
  return srl_per_add(R->per, R->num_envs, stream);
}

extern "C" int srl_frame_replay_add_prioritized(srl_frame_replay_t* R, srl_apex_actor_t* actor, const uint8_t* state, const int64_t* action,
                                                const float* reward, const uint8_t* next_state, const uint8_t* done, float priority_eps,
                                                void* stream) {
  REQ(R && actor && state && action && reward && next_state && done, "frame_replay_add_prioritized: NULL pointer");
  REQ(isfinite(priority_eps) && priority_eps > 0.f, "frame_replay_add_prioritized: priority_eps=%g must be finite and > 0", (double)priority_eps);
  REQ(apex_actor_num_envs(actor) == R->num_envs, "frame_replay_add_prioritized: the actor has num_envs=%d, the memory %d",
      apex_actor_num_envs(actor), R->num_envs);
  const cudaStream_t st = (cudaStream_t)stream;
  const int E = R->num_envs;
  const int64_t ptr = per_tree_ptr(R->per);
  int oldest;
  int rc = frame_stage_and_fold(R, state, action, reward, next_state, done, st, &oldest);
  if (rc || oldest < 0) return rc;
  // s: the oldest step's states (this step's own with n_step = 1, else rebuilt from the window's handles); s': this step's next_states
  const uint4* s = R->stage_s;
  if (R->n_step > 1) {
    frame_stacks_kernel<<<dim3(E, (OBS_VEC + FG_THREADS - 1) / FG_THREADS), FG_THREADS, 0, st>>>(R->pool, R->frame_capacity,
                                                                                                 R->win.h + (int64_t)oldest * E * HANDLES, R->scratch);
    CU(cudaGetLastError(), "frame_replay_add_prioritized: rebuild states");
    s = R->scratch;
  }
  const double* prio = nullptr;
  rc = apex_actor_priorities(actor, reinterpret_cast<const uint8_t*>(s), reinterpret_cast<const uint8_t*>(R->stage_ns), R->ring.action,
                             R->ring.reward, R->ring.done, ptr, R->memory_size, R->gamma_n, priority_eps, &prio, st);
  if (rc) return rc;
  return per_add_prioritized(R->per, prio, E, st);
}

extern "C" int srl_frame_replay_sample(srl_frame_replay_t* R, const double* uniforms, int batch, const double* beta_dev, uint8_t* state,
                                       int64_t* action, float* reward, uint8_t* next_state, uint8_t* done, int64_t* idxs, float* weights,
                                       void* stream) {
  REQ(R && uniforms && beta_dev && idxs, "frame_replay_sample: NULL pointer");
  REQ(batch >= 1 && batch <= MAX_FRAMES, "frame_replay_sample: batch must be in [1, %d], got %d", MAX_FRAMES, batch);
  int rc = check_outputs("frame_replay_sample", batch, idxs, true, state, action, reward, next_state, done, weights);
  if (rc) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  rc = per_sample(R->per, uniforms, batch, 0.0, beta_dev, idxs, nullptr, weights, st);
  if (rc) return rc;
  CU(launch_gather(R, idxs, batch, state, action, reward, next_state, done, st), "frame_replay_sample: gather");
  return 0;
}

extern "C" int srl_frame_replay_gather(srl_frame_replay_t* R, const int64_t* idxs, int64_t n, uint8_t* state, int64_t* action, float* reward,
                                       uint8_t* next_state, uint8_t* done, void* stream) {
  REQ(R && idxs, "frame_replay_gather: NULL pointer");
  REQ(n >= 0 && n <= (int64_t(1) << 31) - 1, "frame_replay_gather: n must be in [0, 2^31), got %lld", (long long)n);
  if (n == 0) return 0;
  const int rc = check_outputs("frame_replay_gather", n, idxs, false, state, action, reward, next_state, done, nullptr);
  if (rc) return rc;
  CU(launch_gather(R, idxs, n, state, action, reward, next_state, done, (cudaStream_t)stream), "frame_replay_gather");
  return 0;
}

namespace {
int64_t read_counter(srl_frame_replay* R, const void* src, void* stream) {
  if (!R) return -1;
  int64_t v = 0;
  if (cudaMemcpyAsync(&v, src, 8, cudaMemcpyDeviceToHost, (cudaStream_t)stream) != cudaSuccess) return -1;
  if (cudaStreamSynchronize((cudaStream_t)stream) != cudaSuccess) return -1;
  return v;
}
}  // namespace

extern "C" int64_t srl_frame_replay_frames_allocated(srl_frame_replay_t* R, void* stream) { return read_counter(R, R ? &R->st->head : nullptr, stream); }
extern "C" int64_t srl_frame_replay_retired(srl_frame_replay_t* R, void* stream) { return read_counter(R, R ? &R->st->retired : nullptr, stream); }
