// What the two GPU replay memories share (replay.cu: transitions stored as frame stacks; frame_replay.cu: each frame stored once):
// the stack geometry, the n-step window's depth and the fold's reward and done arithmetic.
#pragma once
#include <stdint.h>

namespace srl {

constexpr int64_t OBS_BYTES = 4 * 84 * 84;                 // one u8 frame stack: 28,224 B
constexpr int OBS_VEC = (int)(OBS_BYTES / 16);             // 1,764 16-byte vectors
constexpr int ROW_PAIR_VEC = 2 * OBS_VEC;                  // state + next_state of one transition
constexpr int REPLAY_MAX_NSTEP = 32;

struct GammaPowers { float g[REPLAY_MAX_NSTEP]; };         // g[k] = fp32(double(gamma) ** k)

// _get_n_step_info's reward and done for env e of a window of n_step vector steps ([n_step][E] rows, `oldest` the window slot of the
// oldest step): r0 + r1*g^1 + r2*g^2 ... in fp32 with every product and sum rounded on its own (numpy's float32 arithmetic), stopping
// after the first done.  Returns the window slot of the step that gives next_state (the first done's, else the newest).
__device__ __forceinline__ int fold_reward_done(const float* reward, const uint8_t* done, int E, int e, int n_step, int oldest,
                                                const GammaPowers& gp, float* r_out, uint8_t* d_out) {
  int stop = oldest;
  uint8_t d = done[(int64_t)oldest * E + e];
  float r = reward[(int64_t)oldest * E + e];
  for (int k = 1; k < n_step && !d; ++k) {
    const int s = (oldest + k) % n_step;
    r = __fadd_rn(r, __fmul_rn(reward[(int64_t)s * E + e], gp.g[k]));
    d = done[(int64_t)s * E + e];
    stop = s;
  }
  *r_out = r;
  *d_out = d;
  return stop;
}

}  // namespace srl
