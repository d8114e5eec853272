// GPU prioritized-replay sampler (Ape-X / DQN path, BASELINE.json configs[3]; SURVEY.md §8f rank 3).
// Device-resident float64 sum / min segment trees with the arithmetic of the reference's
//   scalerl/data/segment_tree.py:95-109 (__setitem__), :43-93 (operate), :139-163 (find_prefixsum_idx)
//   scalerl/data/replay_buffer.py:318-322 (_add), :346-351 (update_priorities), :353-381 (_sample_proprtional, _calculate_weight)
// float64 so that sampled INDICES are identical to the reference's Python-float trees; HBM/latency-bound integer+fp64 work,
// no tensor cores.  `retrieve` (missing upstream) = find_prefixsum_idx; p_total excludes the last stored item as upstream does.
#include <new>
#include "common.cuh"
#include "errors.h"
#include "kernels.h"
#include "../../include/scalerl_b200.h"

namespace srl {

// scal: [0] max_priority, [1] invalid-update counter (u64 bits), [2] stored transitions (i64 bits).  The count lives on the device so
// that a captured sample or priority update reads the size as it is when the graph replays, not as it was at capture.
__device__ __forceinline__ int64_t* per_count_slot(double* scal) { return reinterpret_cast<int64_t*>(scal + 2); }

// Batched tree update by ONE block (n <= 1024 leaves per launch): write the leaves (duplicates: the LAST occurrence wins, as a
// sequential loop would), then recompute every touched ancestor level by level.
//   mode 0: idxs/priorities given, leaf = priority^alpha, max_priority updated; idxs at or above the stored count are skipped.
//   mode 1: leaves ptr.. (mod memory_size) = max_priority^alpha, stored count = min(count + n, memory_size)
//   mode 2: leaves ptr.. (mod memory_size) = priority^alpha from prios, max_priority updated, the count as mode 1.  A non-finite priority
//           is counted in scal[1] and stored as mode 1 would store it (max_priority^alpha as the launch found it)
// retired (optional, [memory_size]): the leaves per_retire_kernel took out of sampling.  Mode 0 skips a retired leaf without counting it
// (its priority may be written after it retired); modes 1 and 2 make the leaves they write live again.
__global__ void __launch_bounds__(1024) per_update_kernel(double* __restrict__ sum, double* __restrict__ mn, int64_t cap, int levels,
                                                          const int64_t* __restrict__ idxs, const double* __restrict__ prios, int n,
                                                          double alpha, double* __restrict__ scal, int mode, int64_t ptr, int64_t memory_size,
                                                          uint8_t* __restrict__ retired) {
  __shared__ int64_t sidx[1024];
  __shared__ double smax[32];
  const int t = threadIdx.x;
  int64_t leaf = -1;
  double v = 0.0, pr = 0.0;
  bool valid = t < n;
  if (t < n) {
    if (mode == 0) {
      const int64_t count = *per_count_slot(scal);
      leaf = idxs[t]; pr = prios[t];
      // the reference asserts priority > 0 and 0 <= idx < len(self) (replay_buffer.py:346-351): an invalid entry is
      // skipped here (never an out-of-bounds write) and counted in scal[1]; the Python wrapper raises on it
      if (!(leaf >= 0 && leaf < count) || !(pr > 0.0)) { valid = false; leaf = -1; atomicAdd(reinterpret_cast<unsigned long long*>(scal + 1), 1ull); }
      else if (retired && retired[leaf]) { valid = false; leaf = -1; }
    } else {
      leaf = (ptr + t) % memory_size;
      if (mode == 2) pr = prios[t];
      if (mode == 1 || !isfinite(pr)) {
        if (mode == 2) atomicAdd(reinterpret_cast<unsigned long long*>(scal + 1), 1ull);
        pr = scal[0];                  // read before the barrier that precedes thread 0's max_priority store: max(max, max) = max
      }
    }
    v = pow(pr, alpha);
  }
  sidx[t] = leaf;
  __syncthreads();
  if (mode != 0 && t == 0) { int64_t* c = per_count_slot(scal); *c = *c + n < memory_size ? *c + n : memory_size; }
  bool winner = valid;
  if (winner && mode == 0)
    for (int u = t + 1; u < n; ++u)
      if (sidx[u] == leaf) { winner = false; break; }
  if (winner) {
    sum[cap + leaf] = v; mn[cap + leaf] = v;
    if (retired && mode != 0) retired[leaf] = 0;
  }
  if (mode != 1) {       // max_priority = max(max_priority, priorities...)
    double m = valid ? pr : 0.0;
    for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((t & 31) == 0) smax[t >> 5] = m;
    __syncthreads();
    if (t == 0) { double mm = scal[0]; for (int w = 0; w < 32; ++w) mm = fmax(mm, smax[w]); scal[0] = mm; }
  }
  __syncthreads();
  for (int d = 1; d <= levels; ++d) {
    if (valid) {
      const int64_t node = (cap + leaf) >> d;
      sum[node] = sum[2 * node] + sum[2 * node + 1];
      mn[node] = fmin(mn[2 * node], mn[2 * node + 1]);
    }
    __syncthreads();
  }
}

// sum over leaves [0, end] with the reference's recursive split order: L1 + (L2 + (L3 + ...))  (segment_tree.py:43-73 with start = 0)
__device__ double prefix_sum_ref_order(const double* __restrict__ sum, int64_t cap, int64_t end) {
  double parts[64];
  int np = 0;
  int64_t node = 1, ns = 0, ne = cap - 1;
  while (true) {
    if (ns == 0 && false) {}
    if (end == ne) { parts[np++] = sum[node]; break; }           // exact match of [ns, ne]
    const int64_t mid = (ns + ne) / 2;
    if (end <= mid) { node = 2 * node; ne = mid; }               // whole query inside the left child
    else { parts[np++] = sum[2 * node]; node = 2 * node + 1; ns = mid + 1; }   // left child fully inside + recurse right
  }
  double r = parts[np - 1];
  for (int i = np - 2; i >= 0; --i) r = parts[i] + r;
  return r;
}

// beta_dev (optional): beta read from the device when the kernel runs, so a replayed graph sees every change; else `beta`.
// skip_empty (trees with retired leaves): the descent never enters a subtree of sum 0, so it ends on a leaf of positive priority even
// where rounding puts the prefix at or past the mass it came from (a retired leaf, 0, would otherwise be the rightmost choice).
__global__ void per_sample_kernel(const double* __restrict__ sum, const double* __restrict__ mn, int64_t cap, const double* __restrict__ u,
                                  int batch, const double* __restrict__ scal, double beta, const double* __restrict__ beta_dev,
                                  int64_t* __restrict__ idxs, double* __restrict__ w64, float* __restrict__ w32, bool skip_empty) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= batch) return;
  const int64_t n = *reinterpret_cast<const int64_t*>(scal + 2);
  if (beta_dev) beta = *beta_dev;
  const double p_total = prefix_sum_ref_order(sum, cap, n - 2);  // sum_tree.sum(0, len - 1)  (replay_buffer.py:359)
  const double segment = p_total / batch;
  const double a = segment * i, b = segment * (i + 1);
  double prefix = a + (b - a) * u[i];                            // random.uniform(a, b)
  int64_t idx = 1;
  while (idx < cap) {                                            // find_prefixsum_idx
    const int64_t left = 2 * idx;
    const double lv = sum[left];
    if (lv > prefix || (skip_empty && sum[left + 1] == 0.0)) idx = left;
    else { prefix -= lv; idx = left + 1; }
  }
  idx -= cap;
  idxs[i] = idx;
  const double total = sum[1];
  const double p_min = mn[1] / total;
  const double max_weight = pow(p_min * (double)n, -beta);
  const double wt = pow((sum[cap + idx] / total) * (double)n, -beta) / max_weight;
  if (w64) w64[i] = wt;
  if (w32) w32[i] = (float)wt;
}

// leaves[0 .. *n_dev) leave sampling: sum 0, min +inf (so they enter neither p_total nor p_min), marked in `retired`; their
// ancestors are recomputed level by level, 1024 leaves at a time, as per_update_kernel does.  One block.
__global__ void __launch_bounds__(1024) per_retire_kernel(double* __restrict__ sum, double* __restrict__ mn, int64_t cap, int levels,
                                                          const int64_t* __restrict__ leaves, const unsigned long long* __restrict__ n_dev,
                                                          uint8_t* __restrict__ retired) {
  const int64_t n = (int64_t)*n_dev;
  for (int64_t o = 0; o < n; o += 1024) {
    const bool valid = o + threadIdx.x < n;
    const int64_t leaf = valid ? leaves[o + threadIdx.x] : 0;
    if (valid) { sum[cap + leaf] = 0.0; mn[cap + leaf] = INFINITY; retired[leaf] = 1; }
    __syncthreads();
    for (int d = 1; d <= levels; ++d) {
      if (valid) {
        const int64_t node = (cap + leaf) >> d;
        sum[node] = sum[2 * node] + sum[2 * node + 1];
        mn[node] = fmin(mn[2 * node], mn[2 * node + 1]);
      }
      __syncthreads();
    }
  }
}

__global__ void per_fill_kernel(double* __restrict__ sum, double* __restrict__ mn, int64_t n2, double* scal) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n2) { sum[i] = 0.0; mn[i] = INFINITY; }
  if (i == 0) { scal[0] = 1.0; scal[1] = 0.0; *per_count_slot(scal) = 0; }   // max_priority (replay_buffer.py:308), counter, count
}

}  // namespace srl
using namespace srl;

struct srl_per {
  int64_t memory_size, capacity, tree_ptr, size;
  int levels;
  double alpha;
  double *sum, *mn, *scal;
  uint8_t* retired;                // per-leaf retired mask (per_attach_retired), NULL for a plain sampler
};
extern "C" const char* srl_per_last_error(void) { return srl_last_error(); }

extern "C" int srl_per_create(int64_t memory_size, double alpha, srl_per_t** out) {
  REQ(memory_size >= 2 && memory_size <= (int64_t(1) << 30) && out, "per_create: memory_size must be in [2, 2^30]");
  srl_per* P = new (std::nothrow) srl_per();
  REQ(P, "out of memory");
  P->memory_size = memory_size; P->alpha = alpha; P->tree_ptr = 0; P->size = 0;
  P->capacity = 1; P->levels = 0;
  while (P->capacity < memory_size) { P->capacity *= 2; P->levels++; }
  const int64_t n2 = 2 * P->capacity;
  if (cudaMalloc(&P->sum, n2 * 8) != cudaSuccess || cudaMalloc(&P->mn, n2 * 8) != cudaSuccess || cudaMalloc(&P->scal, 64) != cudaSuccess) {
    delete P; return fail(SRL_EINVAL, "per_create: cudaMalloc failed");
  }
  per_fill_kernel<<<(int)((n2 + 255) / 256), 256>>>(P->sum, P->mn, n2, P->scal);
  CU(cudaDeviceSynchronize(), "per_create");
  *out = P;
  return 0;
}
extern "C" int srl_per_destroy(srl_per_t* P) { if (P) { cudaFree(P->sum); cudaFree(P->mn); cudaFree(P->scal); delete P; } return 0; }
extern "C" int64_t srl_per_size(const srl_per_t* P) { return P ? P->size : 0; }
extern "C" int64_t srl_per_capacity(const srl_per_t* P) { return P ? P->capacity : 0; }

namespace {
// n new leaves at tree_ptr.., in launches of at most 1024 (and at most memory_size: never two writes to one leaf inside a launch):
// max_priority^alpha (prios NULL, mode 1), or prios[i]^alpha (mode 2)
cudaError_t per_insert(srl_per* P, const double* prios, int64_t n, cudaStream_t st) {
  for (int64_t o = 0; o < n;) {
    const int64_t c = n - o < 1024 ? n - o : 1024;
    const int cc = (int)(c < P->memory_size ? c : P->memory_size);
    per_update_kernel<<<1, 1024, 0, st>>>(P->sum, P->mn, P->capacity, P->levels, nullptr, prios ? prios + o : nullptr, cc, P->alpha, P->scal,
                                          prios ? 2 : 1, P->tree_ptr, P->memory_size, P->retired);
    P->tree_ptr = (P->tree_ptr + cc) % P->memory_size;
    P->size = P->size + cc < P->memory_size ? P->size + cc : P->memory_size;
    o += cc;
  }
  return cudaGetLastError();
}
}  // namespace

// n new transitions written at tree_ptr.. with priority max_priority^alpha (_add, replay_buffer.py:318-322)
extern "C" int srl_per_add(srl_per_t* P, int64_t n, void* stream) {
  REQ(P && n >= 0, "per_add: bad argument");
  CU(per_insert(P, nullptr, n, (cudaStream_t)stream), "per_add");
  return 0;
}
// idxs i64 [n], priorities f64 [n] (device): leaf = priority^alpha, max_priority updated (update_priorities, replay_buffer.py:346-351)
extern "C" int srl_per_update_priorities(srl_per_t* P, const int64_t* idxs, const double* priorities, int64_t n, void* stream) {
  REQ(P && idxs && priorities && n >= 0, "per_update_priorities: bad argument");
  for (int64_t o = 0; o < n; o += 1024) {
    const int c = (int)(n - o < 1024 ? n - o : 1024);
    per_update_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(P->sum, P->mn, P->capacity, P->levels, idxs + o, priorities + o, c, P->alpha, P->scal, 0,
                                                            0, P->memory_size, P->retired);  // mode 0 bounds idx by the device count (idx < len(self))
  }
  CU(cudaGetLastError(), "per_update_priorities");
  return 0;
}
// number of (idx, priority) pairs skipped so far because idx was outside [0, size) or priority <= 0 (the reference asserts,
// replay_buffer.py:346-351); synchronises `stream`
extern "C" int64_t srl_per_invalid_updates(srl_per_t* P, void* stream) {
  if (!P) return -1;
  unsigned long long c = 0;
  if (cudaMemcpyAsync(&c, P->scal + 1, 8, cudaMemcpyDeviceToHost, (cudaStream_t)stream) != cudaSuccess) return -1;
  if (cudaStreamSynchronize((cudaStream_t)stream) != cudaSuccess) return -1;
  return (int64_t)c;
}
namespace srl {
int64_t per_tree_ptr(const srl_per* P) { return P->tree_ptr; }
void per_attach_retired(srl_per* P, uint8_t* retired) { P->retired = retired; }
int per_retire(srl_per* P, const int64_t* leaves, const unsigned long long* n_dev, cudaStream_t st) {
  per_retire_kernel<<<1, 1024, 0, st>>>(P->sum, P->mn, P->capacity, P->levels, leaves, n_dev, P->retired);
  CU(cudaGetLastError(), "per_retire");
  return 0;
}
int per_add_prioritized(srl_per* P, const double* priorities, int64_t n, cudaStream_t st) {
  CU(per_insert(P, priorities, n, st), "per_add_prioritized");
  return 0;
}
int per_sample(srl_per* P, const double* uniforms, int batch, double beta, const double* beta_dev, int64_t* idxs, double* weights64,
               float* weights32, cudaStream_t st) {
  REQ(P && uniforms && idxs && batch >= 1, "per_sample: bad argument");
  REQ(P->size >= 2, "per_sample: need at least 2 stored transitions");
  per_sample_kernel<<<(batch + 127) / 128, 128, 0, st>>>(P->sum, P->mn, P->capacity, uniforms, batch, P->scal, beta, beta_dev, idxs, weights64,
                                                         weights32, P->retired != nullptr);
  CU(cudaGetLastError(), "per_sample");
  return 0;
}
}  // namespace srl
// uniforms f64 [batch] in [0,1) (device) -> idxs i64 [batch], IS weights (f64 and/or f32, either may be NULL)
extern "C" int srl_per_sample(srl_per_t* P, const double* uniforms, int batch, double beta, int64_t* idxs, double* weights64, float* weights32,
                              void* stream) {
  return per_sample(P, uniforms, batch, beta, nullptr, idxs, weights64, weights32, (cudaStream_t)stream);
}
// copies the trees (2*capacity doubles each, root at [1], leaves at [capacity..)) and max_priority to device buffers
extern "C" int srl_per_debug_trees(srl_per_t* P, double* sum_out, double* min_out, double* max_priority_out, void* stream) {
  REQ(P, "per_debug_trees: NULL");
  cudaStream_t st = (cudaStream_t)stream;
  if (sum_out) CU(cudaMemcpyAsync(sum_out, P->sum, 2 * P->capacity * 8, cudaMemcpyDeviceToDevice, st), "copy sum");
  if (min_out) CU(cudaMemcpyAsync(min_out, P->mn, 2 * P->capacity * 8, cudaMemcpyDeviceToDevice, st), "copy min");
  if (max_priority_out) CU(cudaMemcpyAsync(max_priority_out, P->scal, 8, cudaMemcpyDeviceToDevice, st), "copy max");
  return 0;
}
