// Noisy networks for the Ape-X learner and actors (Fortunato et al. 2018, factorised Gaussian noise) on the fc layer and the Q head:
//   y = (mu_w + sigma_w (.) eps_w) x + (mu_b + sigma_b (.) eps_b),  eps_w = f(eps_out) f(eps_in)^T,  eps_b = f(eps_out),  f(x) = sgn(x) sqrt|x|
// The existing encoder and head kernels run unchanged on composed weights:
//   noisy_draw_kernel        the standard normals of one or two networks (Philox4x32-10 + Box-Muller) and f of them
//   noisy_compose_kernel     the effective fc and head weights and biases, in the layouts the encoder and QHead read
//   noisy_sigma_grad_kernel  dL/dsigma = dL/dW (.) eps from the gradients of the composed weights (= the mu gradients)
// Every product and sum is rounded once, in torch's order: eps = fl(fo fi), W = fl(mu + fl(sigma eps)), dsigma = fl(dW eps).  No
// contraction (__fmul_rn / __fadd_rn), no atomics: the bits equal torch's for the same noise vectors.
#include "common.cuh"
#include "kernels.h"

namespace srl {

namespace {

constexpr uint32_t NOISE_TAG = 0x6E6F6973u;        // 'nois': keeps the noise counters apart from the actor's epsilon-greedy ones

// row r of one network's noisy layers: fc rows 0 .. 511, then the head's parameter rows (V value rows first, when V > 0)
struct NoisyRow {
  const float* fi;          // f(eps_in) of the row's layer
  float fo;                 // f(eps_out) of the row
  int n4;                   // float4s per row
  int64_t w;                // the row's first element in its weight tensor
  int bias;                 // 0: fc bias, 1: head b, 2: head ba (the advantage biases)
  int b;                    // the row's index in that bias
};
SRL_DEVINL NoisyRow noisy_row(int r, int V, const float* nz) {
  NoisyRow q;
  if (r < NOISE_FC_OUT) {
    q.fi = nz; q.fo = nz[NOISE_FC_IN + r]; q.n4 = NOISE_FC_IN / 4; q.w = (int64_t)r * NOISE_FC_IN; q.bias = 0; q.b = r;
  } else {
    const int h = r - NOISE_FC_OUT, two = V > 0, adv = two && h >= V;
    q.fi = nz + NOISE_HEAD_IN_OFF + NOISE_HEAD_IN * adv;
    q.fo = nz[NOISE_HEAD_IN_OFF + NOISE_HEAD_IN * (1 + two) + h];
    q.n4 = NOISE_HEAD_IN / 4; q.w = (int64_t)h * NOISE_HEAD_IN; q.bias = adv ? 2 : 1; q.b = adv ? h - V : h;
  }
  return q;
}
SRL_DEVINL float* noisy_w(const NoisyTensors& t, int which, bool fc) { return fc ? t.fc_w[which] : t.h_w[which]; }
SRL_DEVINL float* noisy_b(const NoisyTensors& t, int which, int bias) {
  return bias == 0 ? t.fc_b[which] : (bias == 1 ? t.h_b[which] : t.h_ba[which]);
}
// the torch product order: fl(fl(fo fi) x)
SRL_DEVINL float eps_mul(float fo, float fi, float x) { return __fmul_rn(x, __fmul_rn(fo, fi)); }

// two standard normals from two 32-bit words: u1 in (0, 1] and u2 in [0, 1) from their top 24 bits
SRL_DEVINL void box_muller(uint32_t w1, uint32_t w2, float* z0, float* z1) {
  const float u1 = (float)((w1 >> 8) + 1u) * 0x1p-24f, u2 = (float)(w2 >> 8) * 0x1p-24f;
  const float rad = sqrtf(-2.f * logf(u1));
  float s, c;
  sincospif(2.f * u2, &s, &c);
  *z0 = rad * c;
  *z1 = rad * s;
}

struct NoisyDraw {
  uint2 key;
  const int* step;                   // learner: the Adam step count (not advanced here)
  unsigned long long* draws;         // actor: the noise draw counter, advanced by one after the draw (nets = 1)
  int nn;
  float *normals[2], *noise[2];
};
// one block per network; thread t draws the normals 4g .. 4g + 3, g = t, t + 256, ...: Philox4x32-10 of counter (g, NOISE_TAG, c,
// c >> 32 | net << 31), two Box-Muller pairs from u1 in (0, 1] and u2 in [0, 1)
__global__ void __launch_bounds__(256) noisy_draw_kernel(const NoisyDraw a) {
  const int net = blockIdx.x;
  const unsigned long long c = a.draws ? *a.draws : (unsigned long long)(unsigned)*a.step;
  float* __restrict__ normals = net ? a.normals[1] : a.normals[0];
  float* __restrict__ noise = net ? a.noise[1] : a.noise[0];
  for (int g = threadIdx.x; 4 * g < a.nn; g += blockDim.x) {
    const uint4 r = philox4x32_10(make_uint4((uint32_t)g, NOISE_TAG, (uint32_t)c, (uint32_t)(c >> 32) | ((uint32_t)net << 31)), a.key);
    float z[4];
    box_muller(r.x, r.y, &z[0], &z[1]);
    box_muller(r.z, r.w, &z[2], &z[3]);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int i = 4 * g + k;
      if (i < a.nn) {
        normals[i] = z[k];
        noise[i] = copysignf(sqrtf(fabsf(z[k])), z[k]);
      }
    }
  }
  if (a.draws) {
    __syncthreads();                 // every thread has read the counter
    if (threadIdx.x == 0) *a.draws = c + 1;
  }
}

struct NoisyCompose {
  NoisyTensors p[2];
  NoisyWeights w[2];
  const float* noise[2];
  int V;
};
// one block per (row, network): W row = mu + sigma eps over float4s, and the row's bias
__global__ void __launch_bounds__(256) noisy_compose_kernel(const __grid_constant__ NoisyCompose a) {
  const int net = blockIdx.y;
  const NoisyTensors& p = a.p[net];
  const NoisyRow q = noisy_row(blockIdx.x, a.V, a.noise[net]);
  const bool fc = q.bias == 0;
  const float4* __restrict__ mu = reinterpret_cast<const float4*>(noisy_w(p, 0, fc) + q.w);
  const float4* __restrict__ sg = reinterpret_cast<const float4*>(noisy_w(p, 1, fc) + q.w);
  const float4* __restrict__ fi = reinterpret_cast<const float4*>(q.fi);
  float4* __restrict__ out = reinterpret_cast<float4*>((fc ? a.w[net].fc_w : a.w[net].h_w) + q.w);
  for (int j = threadIdx.x; j < q.n4; j += blockDim.x) {
    const float4 m = mu[j], s = sg[j], f = fi[j];
    out[j] = make_float4(__fadd_rn(m.x, eps_mul(q.fo, f.x, s.x)), __fadd_rn(m.y, eps_mul(q.fo, f.y, s.y)),
                         __fadd_rn(m.z, eps_mul(q.fo, f.z, s.z)), __fadd_rn(m.w, eps_mul(q.fo, f.w, s.w)));
  }
  if (threadIdx.x == 0) {
    float* ob = q.bias == 0 ? a.w[net].fc_b : (q.bias == 1 ? a.w[net].h_b : a.w[net].h_ba);
    ob[q.b] = __fadd_rn(noisy_b(p, 0, q.bias)[q.b], __fmul_rn(noisy_b(p, 1, q.bias)[q.b], q.fo));
  }
}

struct NoisySigmaGrad {
  NoisyTensors g;
  const float* noise;
  int V;
};
// one block per row of the online network: dsigma = dmu (.) eps for the row's weights and its bias
__global__ void __launch_bounds__(256) noisy_sigma_grad_kernel(const __grid_constant__ NoisySigmaGrad a) {
  const NoisyRow q = noisy_row(blockIdx.x, a.V, a.noise);
  const bool fc = q.bias == 0;
  const float4* __restrict__ gm = reinterpret_cast<const float4*>(noisy_w(a.g, 0, fc) + q.w);
  const float4* __restrict__ fi = reinterpret_cast<const float4*>(q.fi);
  float4* __restrict__ gs = reinterpret_cast<float4*>(noisy_w(a.g, 1, fc) + q.w);
  for (int j = threadIdx.x; j < q.n4; j += blockDim.x) {
    const float4 d = gm[j], f = fi[j];
    gs[j] = make_float4(eps_mul(q.fo, f.x, d.x), eps_mul(q.fo, f.y, d.y), eps_mul(q.fo, f.z, d.z), eps_mul(q.fo, f.w, d.w));
  }
  if (threadIdx.x == 0) noisy_b(a.g, 1, q.bias)[q.b] = __fmul_rn(noisy_b(a.g, 0, q.bias)[q.b], q.fo);
}

}  // namespace

cudaError_t launch_noisy_draw(uint2 key, const int* step, unsigned long long* draws, int nets, int nn, float* const* normals,
                              float* const* noise, cudaStream_t st) {
  NoisyDraw a = {key, step, draws, nn, {normals[0], nets > 1 ? normals[1] : nullptr}, {noise[0], nets > 1 ? noise[1] : nullptr}};
  noisy_draw_kernel<<<nets, 256, 0, st>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_noisy_compose(const NoisyTensors* p, const NoisyWeights* w, const float* const* noise, int nets, const ApexNetDesc& d,
                                 cudaStream_t st) {
  NoisyCompose a = {};
  for (int i = 0; i < nets; ++i) { a.p[i] = p[i]; a.w[i] = w[i]; a.noise[i] = noise[i]; }
  a.V = d.vrows;
  noisy_compose_kernel<<<dim3(NOISE_FC_OUT + param_rows(d), nets), 256, 0, st>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_noisy_sigma_grad(const NoisyTensors& g, const float* noise, const ApexNetDesc& d, cudaStream_t st) {
  const NoisySigmaGrad a = {g, noise, d.vrows};
  noisy_sigma_grad_kernel<<<NOISE_FC_OUT + param_rows(d), 256, 0, st>>>(a);
  return cudaGetLastError();
}

}  // namespace srl
