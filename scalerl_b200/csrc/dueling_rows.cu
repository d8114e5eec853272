// The distributional dueling head of the Ape-X learner and actors (Rainbow: Wang et al. 2016's dueling architecture on C51's atoms
// or QR-DQN's quantiles, Hessel et al. 2018).  With W rows per action (K atoms or N quantiles), value = Linear(512, W) and
// advantage = Linear(512, A W):
//   rows[a W + k] = (v[k] + adv[a W + k]) - (1/A) sum_a' adv[a' W + k]
// The combination is linear in h, so the head is the plain distributional head on composed weights, and every C51 / QR kernel runs
// unchanged on them:
//   dist_dueling_compose_kernel  W_eff [A W][512] and b_eff [A W] from the value and advantage layers (of one or two networks)
//   dist_dueling_grad_kernel     g_v[k] = sum_a gW_eff[a W + k] and g_adv[a W + k] = gW_eff[a W + k] - (1/A) sum_a' gW_eff[a' W + k]
// Each column's sum runs over a = 0 .. A-1 in that order from 0, then one IEEE division by A; every add, subtraction and division is
// rounded once in dueling_q's order (dqn_head.cuh), nothing is contracted and nothing is atomic: the bits are the same on every run.
#include "common.cuh"
#include "kernels.h"

namespace srl {

namespace {

constexpr int DD_THREADS = 128;
constexpr int DD_COLS = 513;              // the 512 weight columns and the bias

struct DistDuelingCompose {
  const float *wv[2], *bv[2], *wa[2], *ba[2];     // value.weight [W][512], value.bias [W], advantage.weight [A W][512], advantage.bias [A W]
  float *W[2], *b[2];                             // W_eff [A W][512], b_eff [A W]
  int A, V;
};
// grid (V, columns / 128, networks): thread = one column j of row k (j == 512: the bias) of every action
__global__ void __launch_bounds__(DD_THREADS) dist_dueling_compose_kernel(const __grid_constant__ DistDuelingCompose p) {
  const int k = blockIdx.x, j = blockIdx.y * DD_THREADS + threadIdx.x, net = blockIdx.z;
  if (j >= DD_COLS) return;
  const bool bias = j == 512;
  const int A = p.A, V = p.V;
  // element (row r, column j) of the value or advantage layer
  const float* wa = bias ? p.ba[net] : p.wa[net] + j;
  const int64_t stride = bias ? 1 : 512;
  float s = 0.f;
  for (int a = 0; a < A; ++a) s = __fadd_rn(s, __ldg(wa + (int64_t)(a * V + k) * stride));
  const float mean = __fdiv_rn(s, (float)A);
  const float v = bias ? __ldg(p.bv[net] + k) : __ldg(p.wv[net] + (int64_t)k * 512 + j);
  float* out = bias ? p.b[net] : p.W[net] + j;
  for (int a = 0; a < A; ++a) {
    const int64_t r = a * V + k;
    out[r * stride] = __fsub_rn(__fadd_rn(v, __ldg(wa + r * stride)), mean);
  }
}

struct DistDuelingGrad {
  const float *gW, *gb;                   // gW_eff [A W][512], gb_eff [A W]
  float *gwv, *gbv, *gba;                 // value.weight's and advantage.weight's gradient rows (one [(W + A W)][512] block), the biases'
  int A, V;
};
// grid (V, columns / 128): thread = one column j of row k (j == 512: the bias) of every action
__global__ void __launch_bounds__(DD_THREADS) dist_dueling_grad_kernel(const __grid_constant__ DistDuelingGrad p) {
  const int k = blockIdx.x, j = blockIdx.y * DD_THREADS + threadIdx.x;
  if (j >= DD_COLS) return;
  const bool bias = j == 512;
  const int A = p.A, V = p.V;
  const float* g = bias ? p.gb : p.gW + j;
  const int64_t stride = bias ? 1 : 512;
  float s = 0.f;
  for (int a = 0; a < A; ++a) s = __fadd_rn(s, __ldg(g + (int64_t)(a * V + k) * stride));
  const float mean = __fdiv_rn(s, (float)A);
  if (bias) p.gbv[k] = s; else p.gwv[(int64_t)k * 512 + j] = s;
  float* ga = bias ? p.gba : p.gwv + (int64_t)V * 512 + j;        // the advantage rows follow the value rows
  for (int a = 0; a < A; ++a) {
    const int64_t r = a * V + k;
    ga[r * stride] = __fsub_rn(__ldg(g + r * stride), mean);
  }
}

}  // namespace

cudaError_t launch_dist_dueling_compose(const QHead* p, const HeadRows* rows, int nets, int V, cudaStream_t st) {
  DistDuelingCompose a = {};
  for (int i = 0; i < nets; ++i) {
    a.wv[i] = p[i].W; a.bv[i] = p[i].b; a.wa[i] = p[i].W + (size_t)V * 512; a.ba[i] = p[i].ba;
    a.W[i] = rows[i].W; a.b[i] = rows[i].b;
  }
  a.A = p[0].A;
  a.V = V;
  dist_dueling_compose_kernel<<<dim3(V, (DD_COLS + DD_THREADS - 1) / DD_THREADS, nets), DD_THREADS, 0, st>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_dist_dueling_grad(const HeadRows& g, const QHeadGrad& out, int A, int V, cudaStream_t st) {
  const DistDuelingGrad a = {g.W, g.b, out.gW, out.gb, out.gba, A, V};
  dist_dueling_grad_kernel<<<dim3(V, (DD_COLS + DD_THREADS - 1) / DD_THREADS), DD_THREADS, 0, st>>>(a);
  return cudaGetLastError();
}

}  // namespace srl
