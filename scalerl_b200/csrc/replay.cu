// GPU prioritized replay memory (Ape-X path): n-step transitions stored on the device in a ring whose slot i is leaf i of the
// memory's own sampler trees (srl_per, per.cu).  Restates the reference's
//   scalerl/data/replay_buffer.py:197-218 (MultiStepReplayBuffer.save_to_memory_vect_envs: an n-deep window per env),
//   :230-273 (_get_n_step_info: the fold), :319-323 (PrioritizedReplayBuffer._add: ring slot = tree_ptr), :325-344 (sample)
// with each field kept in its stored dtype.  The fold and the gather are HBM-bound byte copies (16-byte vectors), no tensor cores.
#include <math.h>
#include <new>
#include "common.cuh"
#include "errors.h"
#include "kernels.h"
#include "replay.cuh"
#include "../../include/scalerl_b200.h"

namespace srl {

constexpr int FOLD_THREADS = 256;
constexpr int GATHER_THREADS = 256, GATHER_VPT = 2;        // 16-byte vectors per thread, all loaded before any is stored
constexpr int GATHER_CHUNKS = (ROW_PAIR_VEC + GATHER_THREADS * GATHER_VPT - 1) / (GATHER_THREADS * GATHER_VPT);   // CTAs per transition

// The transition fields: the ring ([M] rows) and the staging window ([n_step][E] rows; vector step t sits in window slot t mod n_step).
struct ReplayRows {
  uint4 *state, *next_state;
  int64_t* action;
  float* reward;
  uint8_t* done;
};

// One n-step transition per env (blockIdx.x), written at ring slot (ptr + e) mod M; blockIdx.y splits the two 28,224-byte rows.
// The fold is _get_n_step_info's: state and action of the oldest step; reward r0 + r1*g^1 + r2*g^2 ... in fp32 with every product and
// sum rounded on its own (numpy's float32 arithmetic); stop after the first done, whose step gives next_state and done.
__global__ void __launch_bounds__(FOLD_THREADS) replay_fold_kernel(ReplayRows win, ReplayRows ring, int E, int n_step, int oldest,
                                                                   GammaPowers gp, int64_t ptr, int64_t M) {
  const int e = blockIdx.x;
  float r;
  uint8_t d;
  const int stop = fold_reward_done(win.reward, win.done, E, e, n_step, oldest, gp, &r, &d);
  const int64_t slot = (ptr + e) % M;
  const int i = blockIdx.y * FOLD_THREADS + threadIdx.x;
  if (i < OBS_VEC) ring.state[slot * OBS_VEC + i] = win.state[((int64_t)oldest * E + e) * OBS_VEC + i];
  else if (i < ROW_PAIR_VEC) ring.next_state[slot * OBS_VEC + i - OBS_VEC] = win.next_state[((int64_t)stop * E + e) * OBS_VEC + i - OBS_VEC];
  if (blockIdx.y == 0 && threadIdx.x == 0) {
    ring.action[slot] = win.action[(int64_t)oldest * E + e];
    ring.reward[slot] = r;
    ring.done[slot] = d;
  }
}

// out row b = ring slot idxs[b] (blockIdx.x = b); blockIdx.y splits the row pair.  A slot outside [0, M) leaves its output row as it was.
__global__ void __launch_bounds__(GATHER_THREADS) replay_gather_kernel(ReplayRows ring, int64_t M, const int64_t* __restrict__ idxs, ReplayRows out) {
  const int b = blockIdx.x;
  const int64_t slot = idxs[b];
  if (slot < 0 || slot >= M) return;
  const int i0 = blockIdx.y * GATHER_THREADS * GATHER_VPT + threadIdx.x;
  uint4 v[GATHER_VPT];
#pragma unroll
  for (int k = 0; k < GATHER_VPT; ++k) {
    const int i = i0 + k * GATHER_THREADS;
    if (i < OBS_VEC) v[k] = ring.state[slot * OBS_VEC + i];
    else if (i < ROW_PAIR_VEC) v[k] = ring.next_state[slot * OBS_VEC + i - OBS_VEC];
  }
#pragma unroll
  for (int k = 0; k < GATHER_VPT; ++k) {
    const int i = i0 + k * GATHER_THREADS;
    if (i < OBS_VEC) out.state[(int64_t)b * OBS_VEC + i] = v[k];
    else if (i < ROW_PAIR_VEC) out.next_state[(int64_t)b * OBS_VEC + i - OBS_VEC] = v[k];
  }
  if (blockIdx.y == 0 && threadIdx.x == 0) {
    out.action[b] = ring.action[slot];
    out.reward[b] = ring.reward[slot];
    out.done[b] = ring.done[slot];
  }
}

}  // namespace srl
using namespace srl;

struct srl_replay {
  srl_per_t* per;
  int64_t memory_size;
  int num_envs, n_step;
  GammaPowers gp;
  float gamma_n;                   // fp32(gamma^n_step): the bootstrap discount of an n-step transition (srl_replay_add_prioritized)
  int64_t steps;                   // vector steps added so far (host-known: adds are host calls)
  void* arena;
  ReplayRows ring, win;
};

namespace {
// the ring's rows, then the staging window's
int replay_rows(srl_replay* R, WsRow* t) {
  const int64_t M = R->memory_size, W = (int64_t)R->n_step * R->num_envs;
  int n = 0;
  t[n++] = ws_row("state", M * OBS_VEC, &R->ring.state);
  t[n++] = ws_row("next_state", M * OBS_VEC, &R->ring.next_state);
  t[n++] = ws_row("action", M, &R->ring.action);
  t[n++] = ws_row("reward", M, &R->ring.reward);
  t[n++] = ws_row("done", M, &R->ring.done);
  t[n++] = ws_row("window.state", W * OBS_VEC, &R->win.state);
  t[n++] = ws_row("window.next_state", W * OBS_VEC, &R->win.next_state);
  t[n++] = ws_row("window.action", W, &R->win.action);
  t[n++] = ws_row("window.reward", W, &R->win.reward);
  t[n++] = ws_row("window.done", W, &R->win.done);
  return n;
}
// the gather's outputs: state / next_state u8 [n,4,84,84] (16-byte aligned), action i64, reward f32, done u8 [n]
int check_outputs(const char* what, int64_t n, const int64_t* idxs, bool idxs_out, const uint8_t* state, const int64_t* action, const float* reward,
                  const uint8_t* next_state, const uint8_t* done, const float* weights) {
  REQ(state && action && reward && next_state && done, "%s: NULL output", what);
  REQ(!misaligned(state, 16) && !misaligned(next_state, 16), "%s: state / next_state must be 16-byte aligned", what);
  const Span s[] = {{idxs, n * 8, idxs_out, "idxs"}, {state, n * OBS_BYTES, true, "state"}, {action, n * 8, true, "action"},
                    {reward, n * 4, true, "reward"}, {next_state, n * OBS_BYTES, true, "next_state"}, {done, n, true, "done"},
                    {weights, n * 4, true, "weights"}};
  return check_spans(s, 7, what);
}
cudaError_t launch_gather(srl_replay* R, const int64_t* idxs, int64_t n, uint8_t* state, int64_t* action, float* reward, uint8_t* next_state,
                          uint8_t* done, cudaStream_t st) {
  const ReplayRows out = {reinterpret_cast<uint4*>(state), reinterpret_cast<uint4*>(next_state), action, reward, done};
  replay_gather_kernel<<<dim3((unsigned)n, GATHER_CHUNKS), GATHER_THREADS, 0, st>>>(R->ring, R->memory_size, idxs, out);
  return cudaGetLastError();
}
}  // namespace

extern "C" int srl_replay_create(int64_t memory_size, int num_envs, int n_step, double gamma, double alpha, srl_replay_t** out) {
  REQ(out, "replay_create: out is NULL");
  REQ(memory_size >= 2 && memory_size <= (int64_t(1) << 30), "replay_create: memory_size must be in [2, 2^30], got %lld", (long long)memory_size);
  REQ(num_envs >= 1 && num_envs <= MAX_FRAMES && num_envs <= memory_size, "replay_create: num_envs must be in [1, min(%d, memory_size)], got %d",
      MAX_FRAMES, num_envs);
  REQ(n_step >= 1 && n_step <= REPLAY_MAX_NSTEP, "replay_create: n_step must be in [1, %d], got %d", REPLAY_MAX_NSTEP, n_step);
  REQ(isfinite(gamma), "replay_create: gamma must be finite");
  srl_replay* R = new (std::nothrow) srl_replay();
  REQ(R, "out of memory");
  R->memory_size = memory_size; R->num_envs = num_envs; R->n_step = n_step; R->steps = 0;
  for (int k = 0; k < REPLAY_MAX_NSTEP; ++k) R->gp.g[k] = (float)pow(gamma, (double)k);    // numpy's float32(gamma ** k)
  R->gamma_n = (float)pow(gamma, (double)n_step);
  WsRow t[10];
  const int nrows = replay_rows(R, t);
  const int64_t bytes = rows_bytes(t, nrows, false);
  const cudaError_t e = cudaMalloc(&R->arena, bytes);
  if (e != cudaSuccess) {
    cudaGetLastError();
    delete R;
    return fail((int)e, "replay_create: cudaMalloc of %lld bytes (%lld transitions of %lld B, %d x %d staged) failed: %s", (long long)bytes,
                (long long)memory_size, (long long)(2 * OBS_BYTES + 13), n_step, num_envs, cudaGetErrorString(e));
  }
  carve_rows(t, nrows, false, static_cast<char*>(R->arena));
  const int rc = srl_per_create(memory_size, alpha, &R->per);
  if (rc) { cudaFree(R->arena); delete R; return rc; }
  *out = R;
  return 0;
}

extern "C" int srl_replay_destroy(srl_replay_t* R) {
  if (R) { srl_per_destroy(R->per); cudaFree(R->arena); delete R; }
  return 0;
}
extern "C" int64_t srl_replay_size(const srl_replay_t* R) { return R ? srl_per_size(R->per) : 0; }
extern "C" srl_per_t* srl_replay_per(srl_replay_t* R) { return R ? R->per : nullptr; }

namespace {
// one vector step into the window and, once the window is full, its fold into ring slots (ptr + e) mod M.  *oldest: the window slot
// of the step the fold took state and action from, -1 while the window is filling (replay_buffer.py:208-210: no transition yet)
int stage_and_fold(srl_replay* R, const uint8_t* state, const int64_t* action, const float* reward, const uint8_t* next_state,
                   const uint8_t* done, cudaStream_t st, int* oldest) {
  const int E = R->num_envs, n = R->n_step;
  const int64_t w = (R->steps % n) * E;                       // this vector step's window slot
  CU(cudaMemcpyAsync(R->win.state + w * OBS_VEC, state, E * OBS_BYTES, cudaMemcpyDefault, st), "replay_add: copy state");
  CU(cudaMemcpyAsync(R->win.next_state + w * OBS_VEC, next_state, E * OBS_BYTES, cudaMemcpyDefault, st), "replay_add: copy next_state");
  CU(cudaMemcpyAsync(R->win.action + w, action, E * sizeof(int64_t), cudaMemcpyDefault, st), "replay_add: copy action");
  CU(cudaMemcpyAsync(R->win.reward + w, reward, E * sizeof(float), cudaMemcpyDefault, st), "replay_add: copy reward");
  CU(cudaMemcpyAsync(R->win.done + w, done, E, cudaMemcpyDefault, st), "replay_add: copy done");
  R->steps++;
  *oldest = -1;
  if (R->steps < n) return 0;
  *oldest = (int)(R->steps % n);
  replay_fold_kernel<<<dim3(E, (ROW_PAIR_VEC + FOLD_THREADS - 1) / FOLD_THREADS), FOLD_THREADS, 0, st>>>(R->win, R->ring, E, n, *oldest, R->gp,
                                                                                                       per_tree_ptr(R->per), R->memory_size);
  CU(cudaGetLastError(), "replay_add: fold");
  return 0;
}
}  // namespace

extern "C" int srl_replay_add(srl_replay_t* R, const uint8_t* state, const int64_t* action, const float* reward, const uint8_t* next_state,
                              const uint8_t* done, void* stream) {
  REQ(R && state && action && reward && next_state && done, "replay_add: NULL pointer");
  int oldest;
  const int rc = stage_and_fold(R, state, action, reward, next_state, done, (cudaStream_t)stream, &oldest);
  if (rc || oldest < 0) return rc;
  return srl_per_add(R->per, R->num_envs, stream);            // the trees' _add of E leaves, env order (replay_buffer.py:319-323)
}

extern "C" int srl_replay_add_prioritized(srl_replay_t* R, srl_apex_actor_t* actor, const uint8_t* state, const int64_t* action, const float* reward,
                                          const uint8_t* next_state, const uint8_t* done, float priority_eps, void* stream) {
  REQ(R && actor && state && action && reward && next_state && done, "replay_add_prioritized: NULL pointer");
  REQ(isfinite(priority_eps) && priority_eps > 0.f, "replay_add_prioritized: priority_eps=%g must be finite and > 0", (double)priority_eps);
  REQ(apex_actor_num_envs(actor) == R->num_envs, "replay_add_prioritized: the actor has num_envs=%d, the memory %d", apex_actor_num_envs(actor),
      R->num_envs);
  const cudaStream_t st = (cudaStream_t)stream;
  const int E = R->num_envs;
  const int64_t ptr = per_tree_ptr(R->per);                   // the fold's first ring slot
  int oldest;
  int rc = stage_and_fold(R, state, action, reward, next_state, done, st, &oldest);
  if (rc || oldest < 0) return rc;
  // s: the oldest step's state rows; s': the newest step's next_state rows, the s' of every transition without a done in its window
  // (one with a done has d = 1, which zeroes its bootstrap term)
  const int newest = (int)((R->steps - 1) % R->n_step);
  const double* prio = nullptr;
  rc = apex_actor_priorities(actor, reinterpret_cast<const uint8_t*>(R->win.state + (int64_t)oldest * E * OBS_VEC),
                             reinterpret_cast<const uint8_t*>(R->win.next_state + (int64_t)newest * E * OBS_VEC), R->ring.action, R->ring.reward,
                             R->ring.done, ptr, R->memory_size, R->gamma_n, priority_eps, &prio, st);
  if (rc) return rc;
  return per_add_prioritized(R->per, prio, E, st);           // leaves ptr .. ptr + E - 1 in env order
}

extern "C" int srl_replay_sample(srl_replay_t* R, const double* uniforms, int batch, const double* beta_dev, uint8_t* state, int64_t* action,
                                 float* reward, uint8_t* next_state, uint8_t* done, int64_t* idxs, float* weights, void* stream) {
  REQ(R && uniforms && beta_dev && idxs, "replay_sample: NULL pointer");
  REQ(batch >= 1 && batch <= MAX_FRAMES, "replay_sample: batch must be in [1, %d], got %d", MAX_FRAMES, batch);
  int rc = check_outputs("replay_sample", batch, idxs, true, state, action, reward, next_state, done, weights);
  if (rc) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  rc = per_sample(R->per, uniforms, batch, 0.0, beta_dev, idxs, nullptr, weights, st);
  if (rc) return rc;
  CU(launch_gather(R, idxs, batch, state, action, reward, next_state, done, st), "replay_sample: gather");
  return 0;
}

extern "C" int srl_replay_gather(srl_replay_t* R, const int64_t* idxs, int64_t n, uint8_t* state, int64_t* action, float* reward,
                                 uint8_t* next_state, uint8_t* done, void* stream) {
  REQ(R && idxs, "replay_gather: NULL pointer");
  REQ(n >= 0 && n <= (int64_t(1) << 31) - 1, "replay_gather: n must be in [0, 2^31), got %lld", (long long)n);
  if (n == 0) return 0;
  const int rc = check_outputs("replay_gather", n, idxs, false, state, action, reward, next_state, done, nullptr);
  if (rc) return rc;
  CU(launch_gather(R, idxs, n, state, action, reward, next_state, done, (cudaStream_t)stream), "replay_gather");
  return 0;
}
