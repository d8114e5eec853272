// Encoder forward / backward drivers: weight packing + the sequence of wgmma implicit-GEMM launches.
#include "encoder_problems.cuh"
#include "tma_problems.cuh"
#include "res_problems.cuh"
#include "enc_fused.cuh"
#include "kernels.h"
#include <stdio.h>
#include <stdlib.h>

namespace srl {

// fp32 master parameters (PyTorch layouts) -> bf16 operand copies in the layouts the GEMMs consume.
// One launch, three block roles (fc.weight is 96 % of the elements and is written twice -- K-major for the forward GEMM, transposed
// for dgrad -- so both copies go through a shared-memory tile: coalesced fp32 reads, >= 128-byte contiguous bf16 writes):
//   blocks [0, 256)    wfk[j][hw*64 + c] = Wfc[j][c*49 + hw]        two rows j per block
//   blocks [256, 512)  wfd[hw*64 + c][j] = Wfc[j][c*49 + hw]        tile = 64 j x 2 c (98 consecutive source columns)
//   blocks [512, 800)  the conv weight copies (147,456 elements), two elements per thread
constexpr int PACK_BLOCKS_FK = 256, PACK_BLOCKS_FD = 256, PACK_BLOCKS_CONV = 288;
SRL_DEVINL void pack_store(bf16* __restrict__ out, bf16* __restrict__ out_lo, int64_t i, float v) {
  const bf16 hi = __float2bfloat16_rn(v);
  out[i] = hi;
  if (out_lo) out_lo[i] = __float2bfloat16_rn(v - __bfloat162float(hi));     // fp32-accurate mode: w = hi + lo to 16 significant bits
}
SRL_DEVINL void pack_store2(bf16* __restrict__ out, bf16* __restrict__ out_lo, int64_t i, float v0, float v1) {      // i even
  const bf16 h0 = __float2bfloat16_rn(v0), h1 = __float2bfloat16_rn(v1);
  *reinterpret_cast<uint32_t*>(out + i) = pack_bf16x2(v0, v1);
  if (out_lo) *reinterpret_cast<uint32_t*>(out_lo + i) = pack_bf16x2(v0 - __bfloat162float(h0), v1 - __bfloat162float(h1));
}
__global__ void __launch_bounds__(256) pack_weights_kernel(ParamPtrs p, bf16* __restrict__ out, bf16* __restrict__ out_lo, int skip_w1k) {
  pdl_wait(2);     // (not launched with the attribute: returns at once; names the kernel in the diagnostics timeline)
  __shared__ __align__(16) float tile[64 * 99];                 // role 1: two fc rows (2 x 3136); role 2: [64 j][99]
  const int t = threadIdx.x, b = blockIdx.x;
  if (b < PACK_BLOCKS_FK) {
    const float4* src = reinterpret_cast<const float4*>(p.wf + (size_t)(2 * b) * 3136);       // rows 2b, 2b+1: 1568 float4, all loads in flight
    float4 v[7];
#pragma unroll
    for (int u = 0; u < 7; ++u) { const int q = t + 256 * u; if (q < 1568) v[u] = __ldg(src + q); }
#pragma unroll
    for (int u = 0; u < 7; ++u) { const int q = t + 256 * u; if (q < 1568) *reinterpret_cast<float4*>(tile + 4 * q) = v[u]; }
    __syncthreads();
#pragma unroll 4
    for (int pp = t; pp < 2 * 1568; pp += 256) {   // output pair: row r, k = 2 pp' = hw*64 + c
      const int r = pp >= 1568, k = 2 * (pp - r * 1568), hw = k >> 6, c = k & 63;
      const float* row = tile + r * 3136;
      pack_store2(out, out_lo, WPack::WFK + (int64_t)(2 * b + r) * 3136 + k, row[c * 49 + hw], row[(c + 1) * 49 + hw]);
    }
  } else if (b < PACK_BLOCKS_FK + PACK_BLOCKS_FD) {
    const int bb = b - PACK_BLOCKS_FK, j0 = (bb & 7) * 64, c0 = (bb >> 3) * 2;
    // 64 rows x 49 float2 (98 consecutive source columns c0*49 .. c0*49+97), all 13 loads of a thread in flight together
    float2 v[13];
#pragma unroll
    for (int u = 0; u < 13; ++u) {
      const int q = t + 256 * u, jj = q / 49, e = q - jj * 49;
      if (q < 64 * 49) v[u] = __ldg(reinterpret_cast<const float2*>(p.wf + (size_t)(j0 + jj) * 3136 + c0 * 49 + 2 * e));
    }
#pragma unroll
    for (int u = 0; u < 13; ++u) {
      const int q = t + 256 * u, jj = q / 49, e = q - jj * 49;
      if (q < 64 * 49) { tile[jj * 99 + 2 * e] = v[u].x; tile[jj * 99 + 2 * e + 1] = v[u].y; }
    }
    __syncthreads();
    const int lane = t & 31, warp = t >> 5;
    for (int kk = warp; kk < 98; kk += 8) {      // source column kk = cc*49 + hw -> destination row hw*64 + c0 + cc
      const int cc = kk >= 49, hw = kk - cc * 49;
      pack_store2(out, out_lo, WPack::WFD + (int64_t)(hw * 64 + c0 + cc) * 512 + j0 + 2 * lane, tile[(2 * lane) * 99 + kk], tile[(2 * lane + 1) * 99 + kk]);
    }
  } else {
    const int bb = b - PACK_BLOCKS_FK - PACK_BLOCKS_FD;
    constexpr int64_t NCONV = WPack::WFK + (WPack::TOTAL - WPack::W3D);       // the copies before and after the two fc blocks
    for (int64_t n = (int64_t)bb * 256 + t; n < NCONV; n += (int64_t)PACK_BLOCKS_CONV * 256) {
      const int64_t i = n < WPack::WFK ? n : n - WPack::WFK + WPack::W3D;
      float v;
      if (i < WPack::W2K) {                       // w1k[co][(kh2*2+kw2)*64 + c*16 + dy*4 + dx] = W1[co][c][4kh2+dy][4kw2+dx]
        if (skip_w1k) continue;                   // written by obs_s2d_kernel's extra blocks inside a step
        const int e = (int)(i - WPack::W1K), co = e >> 8, k = e & 255, tap = k >> 6, q = k & 63;
        const int c = q >> 4, dy = (q >> 2) & 3, dx = q & 3, kh = 4 * (tap >> 1) + dy, kw = 4 * (tap & 1) + dx;
        v = p.w1[co * 256 + c * 64 + kh * 8 + kw];
      } else if (i < WPack::W3K) {                // w2k[co][(kh*4+kw)*32 + c]
        const int e = (int)(i - WPack::W2K), co = e >> 9, k = e & 511, tap = k >> 5, c = k & 31;
        v = p.w2[((co * 32 + c) << 4) + tap];
      } else if (i < WPack::WFK) {                // w3k[co][(kh*3+kw)*64 + c]
        const int e = (int)(i - WPack::W3K), co = e / 576, k = e - co * 576, tap = k >> 6, c = k & 63;
        v = p.w3[(co * 64 + c) * 9 + tap];
      } else if (i < WPack::W2D) {                // w3d[c][(kh*3+kw)*64 + co]
        const int e = (int)(i - WPack::W3D), c = e / 576, k = e - c * 576, tap = k >> 6, co = k & 63;
        v = p.w3[(co * 64 + c) * 9 + tap];
      } else {                                    // w2d[cls][c][(kh'*2+kw')*64 + co], kh = ph + 2kh', kw = pw + 2kw'
        const int e = (int)(i - WPack::W2D), cls = e >> 13, r = e & 8191, c = r >> 8, k = r & 255, tt = k >> 6, co = k & 63;
        const int kh = (cls >> 1) + 2 * (tt >> 1), kw = (cls & 1) + 2 * (tt & 1);
        v = p.w2[((co * 32 + c) << 4) + kh * 4 + kw];
      }
      pack_store(out, out_lo, i, v);
    }
  }
}

// u8 NCHW frames -> space-to-depth bf16 NHWC: xs[n][Y][X][c*16+dy*4+dx] = obs[n][c][4Y+dy][4X+dx]  (exact: u8 fits bf16).
// One block per frame: the 16 x 21 source rows (c,dy) are read coalesced (21 u32 each, 84 B of loads in flight per thread) into
// shared memory, then each thread converts u32 (4 x dx) -> 4 bf16 and the block writes 21 x 21 x 128 B contiguously.
__global__ void __launch_bounds__(352) obs_s2d_kernel(const uint8_t* __restrict__ obs, bf16* __restrict__ xs, int frame_blocks,
                                                      const float* __restrict__ w1, bf16* __restrict__ w1k, bf16* __restrict__ w1k_lo) {
  pdl_wait(1);     // launched with programmatic stream serialization: see common.cuh
  pdl_launch();
  if ((int)blockIdx.x >= frame_blocks) {
    // extra blocks: conv1's K-major weight copy w1k[co][(kh2*2+kw2)*64 + c*16 + dy*4 + dx] = W1[co][c][4kh2+dy][4kw2+dx] -- conv1 is the next kernel
    // of the stream, so it never has to wait for pack_weights_kernel (which skips this copy when the step launches it)
    const int e = ((int)blockIdx.x - frame_blocks) * 352 + (int)threadIdx.x;
    if (e < 32 * 256 && w1k) {
      const int co = e >> 8, k = e & 255, tap = k >> 6, q = k & 63;
      const int c = q >> 4, dy = (q >> 2) & 3, dx = q & 3, kh = 4 * (tap >> 1) + dy, kw = 4 * (tap & 1) + dx;
      pack_store(w1k, w1k_lo, e, __ldg(w1 + co * 256 + c * 64 + kh * 8 + kw));
    }
    return;
  }
  __shared__ uint32_t tile[21][16][21];
  const int n = blockIdx.x;
  const int t = threadIdx.x;
  if (t < 336) {
    const int g = t / 21, X = t - g * 21;      // g = (c, dy)
    const uint8_t* src = obs + (size_t)n * 28224 + (g >> 2) * 7056 + (g & 3) * 84;
#pragma unroll
    for (int y = 0; y < 21; ++y) tile[y][g][X] = __ldg(reinterpret_cast<const uint32_t*>(src + y * 336) + X);
  }
  __syncthreads();
  if (t < 336) {
    const int X = t >> 4, g = t & 15;
#pragma unroll
    for (int y = 0; y < 21; ++y) {
      const uint32_t w = tile[y][g][X];
      const float f0 = __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7540)) - 8388608.f;
      const float f1 = __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7541)) - 8388608.f;
      const float f2 = __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7542)) - 8388608.f;
      const float f3 = __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7543)) - 8388608.f;
      *reinterpret_cast<uint2*>(xs + (((size_t)n * 21 + y) * 21 + X) * 64 + g * 4) = make_uint2(pack_bf16x2(f0, f1), pack_bf16x2(f2, f3));
    }
  }
}

// a3 [n][hw][c] (NHWC rows, what conv3 writes and fc forward / dgrad consume) -> a3t [n][c*49 + hw], fc.weight's own column order:
// with a3t as its B operand the fc weight-gradient GEMM produces 64 CONSECUTIVE columns of dW per row (16-byte stores) instead of 64
// stores 196 B apart.  One frame per block through shared memory, 16-byte reads, 4-byte writes; runs on the wgrad side stream.
__global__ void __launch_bounds__(256) a3_transpose_kernel(const bf16* __restrict__ a3, bf16* __restrict__ a3t) {
  pdl_wait(53);
  __shared__ __align__(16) uint16_t tile[49 * 66];        // row hw: 64 channels + 2 pad (132 B pitch: conflict-free column reads)
  const int n = blockIdx.x, t = threadIdx.x;
  const uint4* src = reinterpret_cast<const uint4*>(a3 + (size_t)n * 3136);
  for (int q = t; q < 392; q += 256) {                    // 392 x 16 B: row hw = q >> 3, channels 8 (q & 7) ..
    const uint4 v = __ldg(src + q);
    uint32_t* d = reinterpret_cast<uint32_t*>(tile + (q >> 3) * 66 + (q & 7) * 8);
    d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
  }
  __syncthreads();
  uint32_t* dst = reinterpret_cast<uint32_t*>(a3t + (size_t)n * 3136);
  for (int pp = t; pp < 1568; pp += 256) {                // output pair o = 2 pp = c*49 + hw
    const int o = 2 * pp, c0 = o / 49, h0 = o - c0 * 49, o1 = o + 1, c1 = o1 / 49, h1 = o1 - c1 * 49;
    dst[pp] = (uint32_t)tile[h0 * 66 + c0] | ((uint32_t)tile[h1 * 66 + c1] << 16);
  }
}
SRL_KSTAMP_SETTER(kstamp_set_encoder)

cudaError_t launch_a3_transpose(const bf16* a3, bf16* a3t, int frames, cudaStream_t st) {
  if (frames <= 0) return cudaSuccess;
  a3_transpose_kernel<<<frames, 256, 0, st>>>(a3, a3t);
  return cudaGetLastError();
}

cudaError_t launch_pack_weights(const ParamPtrs& p, bf16* wpack, cudaStream_t st, bf16* wpack_lo, bool skip_w1k) {
  pack_weights_kernel<<<PACK_BLOCKS_FK + PACK_BLOCKS_FD + PACK_BLOCKS_CONV, 256, 0, st>>>(p, wpack, wpack_lo, skip_w1k ? 1 : 0);
  return cudaGetLastError();
}

#define SRL_TRY(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return e_; } while (0)

static inline int cdiv(int a, int b) { return (a + b - 1) / b; }

// ------------------------------------------------------------------------------------------------
// tensor maps
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(f);
  }
  return fn;
}

// bf16 tensor, dims innermost-first, strides in ELEMENTS for dims 1..rank-1, SWIZZLE_128B, zero OOB fill
bool make_map(CUtensorMap* m, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_elems, const uint32_t* box,
              bool swizzle64) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return false;
  cuuint64_t gd[5], gs[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) { gd[i] = dims[i]; bx[i] = box[i]; es[i] = 1; }
  for (int i = 0; i + 1 < rank; ++i) gs[i] = strides_elems[i] * 2;
  return fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
            swizzle64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Every map is 2-D over dense rows of `inner` elements (box = box_inner x box_rows).  The first map that cannot be built is
// remembered by name (with "_lo" for the low operand set) and every later one is skipped.
struct MapBuilder {
  const char* failed = nullptr;
  bool lo = false, failed_lo = false;
  void operator()(CUtensorMap* m, const void* base, uint64_t inner, uint64_t rows, uint32_t box_inner, uint32_t box_rows, const char* name,
                  bool swizzle64 = false) {
    const uint64_t d[2] = {inner, rows}, s[1] = {inner};
    const uint32_t bx[2] = {box_inner, box_rows};
    if (!failed && !make_map(m, base, 2, d, s, bx, swizzle64)) { failed = name; failed_lo = lo; }
  }
};

static void build_operand_maps(MapBuilder& mk, const OperandTensors& b, uint64_t nf, uint64_t nb, OperandMaps* M) {
  mk(&M->a1p0_w, b.a1, 64, nf * 100, 64, RConv2Fwd::WROWS, "a1p0_w");
  mk(&M->a1p1_w, b.a1 + (size_t)nf * 100 * 64, 64, nf * 100, 64, RConv2Fwd::WROWS, "a1p1_w");
  mk(&M->a2_w, b.a2, 64, nf * 81, 64, RConv3Fwd::WROWS, "a2_w");
  mk(&M->da3g_w, b.da3, 64, nb * 81, 64, RConv3Dgrad::WROWS, "da3g_w");
  mk(&M->da3g_b, b.da3, 64, nb * 81, 64, 128, "da3g_b");
  mk(&M->da2g_w, b.da2, 64, nb * 100, 64, RConv2Dgrad::WROWS, "da2g_w");
  mk(&M->da2g_b, b.da2, 64, nb * 100, 64, 128, "da2g_b");
  mk(&M->da1g_b, b.da1, 32, nb * 441, 32, 128, "da1g_b", true);      // da1g: 32-channel rows (64 B), SWIZZLE_64B
  mk(&M->a3m128, b.a3, 3136, nf, 64, 128, "a3m128");
  mk(&M->a3m64, b.a3, 3136, nf, 64, 64, "a3m64");
  mk(&M->dhm128, b.dh, 512, nb, 64, 128, "dhm128");
  mk(&M->dhm64, b.dh, 512, nb, 64, 64, "dhm64");
  const bf16* w = b.wpack;
  mk(&M->w1k, w + WPack::W1K, 256, 32, 64, 32, "w1k");
  mk(&M->w2k, w + WPack::W2K, 512, 64, 64, 64, "w2k");
  mk(&M->w3k, w + WPack::W3K, 576, 64, 64, 64, "w3k");
  mk(&M->wfk, w + WPack::WFK, 3136, 512, 64, 64, "wfk");
  mk(&M->wfd, w + WPack::WFD, 512, 3136, 64, 64, "wfd");
  mk(&M->w3d, w + WPack::W3D, 576, 64, 64, 64, "w3d");
  mk(&M->w2d, w + WPack::W2D, 256, 128, 64, 128, "w2d");
}

cudaError_t build_tma_maps(const EncoderBuffers& b, int NF, int NB, TmaMaps* M, const char** why) {
  static_assert(RConv1Wgrad::WROWS == RConv1Fwd::WROWS && RConv2Wgrad::WROWS == RConv2Fwd::WROWS && RConv3Wgrad::WROWS == RConv3Fwd::WROWS,
                "forward and wgrad share the window maps");
  const uint64_t nf = NF, nb = NB;
  MapBuilder mk;
  mk(&M->xs_w, b.xs, 64, nf * 441, 64, RConv1Fwd::WROWS, "xs_w");
  mk(&M->a3tm64, b.a3t, 3136, nf, 64, 64, "a3tm64");
  build_operand_maps(mk, b.hi, nf, nb, &M->hi);
  mk.lo = true;
  if (b.lo.wpack) build_operand_maps(mk, b.lo, nf, nb, &M->lo);
  M->valid = !mk.failed;
  if (mk.failed && why) {
    static thread_local char name[32];
    snprintf(name, sizeof(name), "%s%s", mk.failed, mk.failed_lo ? "_lo" : "");
    *why = name;
  }
  return mk.failed ? cudaErrorInvalidValue : cudaSuccess;
}

// frames = 0: only the weight-copy blocks (conv1 converts the frames itself: RConv1Fwd::FromFrames)
static cudaError_t launch_s2d(const uint8_t* obs, int frames, bf16* xs, cudaStream_t st, const float* w1, bf16* w1k, bf16* w1k_lo) {
  constexpr int WB = (32 * 256 + 351) / 352;      // extra blocks that write conv1's weight copy
  SRL_TRY(launch_chain(obs_s2d_kernel, dim3(frames + WB), dim3(352), 0, st, obs, xs, frames, w1, w1k, w1k_lo));
  return cudaGetLastError();
}

static int sm_count() {
  static const int n = [] { int d = 0, v = 0; cudaGetDevice(&d); cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, d); return v > 0 ? v : 132; }();
  return n;
}
// persistent CTAs of the resident-window kernels: one per SM by default; data-parallel runs leave a few SMs to the NCCL
// all-reduce that overlaps the conv backward (SRL_PERSISTENT_CTAS, read once)
static int persistent_ctas() {
  static int v = 0;
  if (!v) {
    const char* e = getenv("SRL_PERSISTENT_CTAS");
    v = e ? atoi(e) : sm_count();
    if (v < 16 || v > sm_count()) v = sm_count();
  }
  return v;
}
#define kPersistentCtas persistent_ctas()
// persistent CTAs of the backward chain's resident-window kernels (conv3 / conv2 dgrad, conv1 wgrad): fewer than one per SM leaves SMs to the
// lower-priority side-stream wgrads while the chain runs.  SRL_BWD_CTAS overrides (diagnostics).
static int bwd_ctas() {
  static const int v = [] { const char* e = getenv("SRL_BWD_CTAS"); int x = e ? atoi(e) : 0; return x < 16 || x > sm_count() ? 0 : x; }();
  return v ? v : persistent_ctas() - persistent_ctas() / 9;      // about one SM in nine left to the side-stream wgrads
}
// CTAs of the conv3 / conv2 weight-gradient kernels (side streams).  SRL_WGRAD_CTAS overrides (diagnostics).
static int side_wgrad_ctas() {
  static const int v = [] { const char* e = getenv("SRL_WGRAD_CTAS"); int x = e ? atoi(e) : 64; return x < 8 || x > sm_count() ? 64 : x; }();
  return v;
}

// Per-CTA partial slices of one conv wgrad launch (res_problems.cuh) -> that layer's PyTorch-layout weight gradient, and its bias
// gradient added into the pre-zeroed g.b*.  A slice row is one K index of the wgrad GEMM (CO floats, one per output channel).
// A tile is NR slice rows x 8 output channels chosen so that its NR entries of each channel's PyTorch row are consecutive:
// dW[co0 + j][NR * rg + i] = sum over CTAs of slice[row(rg, i)][co0 + j].  The block copies the tile of every slice into shared
// memory (16-byte cp.async, 32-byte runs of the slice rows, all of them in flight at once), then thread e = 8 i + j adds its element
// over the slices in CTA order -- the same fp32 additions, in the same order, for every CTA count and stream placement -- and
// stores it.  The block after the last tile does the bias the same way.
// KID: diagnostics timeline id.  conv1's reduce, the one on the main chain, is stamped as `conv_wgrad_finalize` (the profile slot it
// keeps); the side-stream reduces are not stamped (0).
struct WgradReduce3 {   // dW3[co][c*9 + tap] = slice[tap*64 + c][co]          tile rg = 2 channels c x 9 taps
  static constexpr int KID = 0, CO = 64, BIAS = 64, PART = WSP_W3, NR = 18, ROW_GROUPS = 32;
  static constexpr bool FRAMES_U8 = false;
  SRL_DEVINL static int row(int rg, int i) { return (i % 9) * 64 + 2 * rg + i / 9; }
};
struct WgradReduce2 {   // dW2[co][c*16 + kh*4 + kw] = slice[kh*128 + kw*32 + c][co]       tile rg = channel c x 16 taps
  static constexpr int KID = 0, CO = 64, BIAS = 64, PART = WSP_W2, NR = 16, ROW_GROUPS = 32;
  static constexpr bool FRAMES_U8 = false;
  SRL_DEVINL static int row(int rg, int i) { return (i >> 2) * 128 + (i & 3) * 32 + rg; }
};
struct WgradReduce1 {   // dW1[co][c*64 + kh*8 + kw] = slice[(kh>>2)*128 + (kw>>2)*64 + c*16 + (kh&3)*4 + (kw&3)][co] / 255
  static constexpr int KID = 51, CO = 32, BIAS = 32, PART = WSP_W1, NR = 16, ROW_GROUPS = 16;
  static constexpr bool FRAMES_U8 = true;          // the frames entered the GEMM as u8 values: the 1/255 is applied to the sum
  // rg = (c, kh2, dy >> 1), i = ((dy & 1), kw): kh = 4 kh2 + dy
  SRL_DEVINL static int row(int rg, int i) {
    const int c = rg >> 2, kh2 = (rg >> 1) & 1, dy = 2 * (rg & 1) + (i >> 3), kw = i & 7;
    return kh2 * 128 + (kw >> 2) * 64 + c * 16 + dy * 4 + (kw & 3);
  }
};
template <class L>
__global__ void __launch_bounds__(L::NR * 8) conv_wgrad_reduce_kernel(const float* __restrict__ part, int n, float* __restrict__ g,
                                                                       float* __restrict__ db) {
  constexpr int CG = L::CO / 8, TILES = L::ROW_GROUPS * CG;
  static_assert(L::BIAS <= 8 * L::NR, "the bias block fits the tile's threads and shared memory");
  extern __shared__ __align__(16) float stage[];          // [n][NR][8] (tile) or [n][BIAS] (bias block)
  pdl_wait(L::KID);    // (not launched with the attribute: returns at once; names the kernel in the diagnostics timeline)
  pdl_launch();
  const int t = threadIdx.x, rg = blockIdx.x / CG, co0 = (blockIdx.x % CG) * 8;
  const bool bias = blockIdx.x == TILES;
  const int per = bias ? L::BIAS / 4 : 2 * L::NR;         // 16-byte pieces per slice
  for (int k = t; k < n * per; k += L::NR * 8) {
    const int c = k / per, q = k - c * per;
    const float* src = part + (size_t)c * L::PART + (bias ? L::PART - L::BIAS + 4 * q : L::row(rg, q >> 1) * L::CO + co0 + 4 * (q & 1));
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(stage + 4 * k)), "l"(src) : "memory");
  }
  asm volatile("cp.async.wait_all;" ::: "memory");
  __syncthreads();
  const int w = bias ? L::BIAS : 8 * L::NR;
  if (t >= w) return;
  float s = 0.f;
  for (int c = 0; c < n; ++c) s += stage[c * w + t];
  if (bias) db[t] += s;
  else g[(size_t)(co0 + (t & 7)) * (L::ROW_GROUPS * L::NR) + L::NR * rg + (t >> 3)] = L::FRAMES_U8 ? s * (1.0f / 255.0f) : s;
}

// The reduces gate the step's join and the optimizer, so they take the device's greatest stream priority: a side stream's reduce is
// not queued behind the other side streams' GEMM CTAs.  They are launched without programmatic stream serialization: the wgrad
// kernels release their dependents at once, and blocks parked in pdl_wait() for a whole wgrad would hold shared memory that the
// other streams' GEMM CTAs need (measured: LSTM at T=100, B=128 ran 0.8 % slower with it).
template <class L>
static cudaError_t launch_wgrad_reduce(const float* part, int n, float* g, float* db, cudaStream_t st) {
  static PerDeviceOnce once;
  SRL_TRY(ensure_max_dynamic_smem(once, conv_wgrad_reduce_kernel<L>, WG_PART_CTAS * L::NR * 32));
  static const int greatest = [] { int lo = 0, hi = 0; return cudaDeviceGetStreamPriorityRange(&lo, &hi) == cudaSuccess ? hi : 0; }();
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(L::ROW_GROUPS * (L::CO / 8) + 1); cfg.blockDim = dim3(L::NR * 8); cfg.dynamicSmemBytes = (size_t)n * L::NR * 32; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributePriority;
  attr[0].val.priority = greatest;
  cfg.attrs = attr; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, conv_wgrad_reduce_kernel<L>, part, n, g, db);
}

cudaError_t encoder_forward(const uint8_t* obs, int frames, const ParamPtrs& p, const EncoderBuffers& buf, const TmaMaps& maps, int mode,
                            const StepStreams& S, bool fused_front) {
  if (frames <= 0) return cudaSuccess;
  if ((mode != 0 && mode != 1) || !maps.valid) return cudaErrorInvalidValue;
  const int sp = mode;                                    // 1: fp32-accurate split operands
  if (sp && !buf.lo.wpack) return cudaErrorInvalidValue;  // bf16 mode: the kernels never touch the low tensors and maps
  const cudaStream_t st = S.main;
  // bf16 mode: frame conversion + conv1 + conv2 as ONE persistent kernel (enc_fused.cuh); SRL_FUSED_FWD=0 or the fp32-accurate
  // operand mode use the three separate kernels
  if (fused_front && !sp && (reinterpret_cast<uintptr_t>(obs) & 15) == 0) {
    EncFusedParams q{obs, p.w1, p.b1, p.w2, p.b2, buf.xs, buf.hi.a1, buf.hi.a2, frames, buf.NF};
    S.b(PS_ENC_FUSED); SRL_TRY(enc_fused_fwd_launch(q, kPersistentCtas, st)); S.e(PS_ENC_FUSED);
    SRL_TRY(S.join(LANE_PACK));      // conv3 / fc read the packed weights
  } else {
  // bf16 mode with 16-byte aligned frames (the bulk copies' alignment): conv1 converts its windows from the frames and writes xs itself,
  // and the frame-conversion kernel only writes conv1's weight copy.  The fp32-accurate mode and 4-byte aligned frames convert the
  // frames to xs first and feed conv1 from xs.
  const bool u8_feed = !sp && (reinterpret_cast<uintptr_t>(obs) & 15) == 0;
  S.b(PS_S2D);
  SRL_TRY(launch_s2d(obs, u8_feed ? 0 : frames, buf.xs, st, p.w1, buf.hi.wpack + WPack::W1K, sp ? buf.lo.wpack + WPack::W1K : nullptr));
  S.e(PS_S2D);
  { RConv1Fwd::Params q{maps.xs_w, maps.hi.w1k, maps.lo.w1k, p.b1, buf.hi.a1, buf.lo.a1, frames, buf.NF};
    S.b(PS_CONV1_FWD);
    if (u8_feed) SRL_TRY((res_fwd_launch_t<RConv1Fwd::FromFrames, 0>(RConv1Fwd::FromFrames::Params{q, obs, buf.xs}, cdiv(frames * 441, 128), kPersistentCtas, st)));
    else SRL_TRY(res_fwd_launch<RConv1Fwd>(q, cdiv(frames * 441, 128), kPersistentCtas, st, sp));
    S.e(PS_CONV1_FWD); }
  SRL_TRY(S.join(LANE_PACK));      // conv1's weight copy comes from the frame-conversion kernel; conv2 is the first reader of the re-packed copies
  { RConv2Fwd::Params q{maps.hi.a1p0_w, maps.hi.a1p1_w, maps.hi.w2k, maps.lo.a1p0_w, maps.lo.a1p1_w, maps.lo.w2k, p.b2, buf.hi.a2, buf.lo.a2, frames};
    S.b(PS_CONV2_FWD); SRL_TRY(res_fwd_launch<RConv2Fwd>(q, cdiv(frames * 100, 128), kPersistentCtas, st, sp)); S.e(PS_CONV2_FWD); }
  }
  { RConv3Fwd::Params q{maps.hi.a2_w, maps.hi.w3k, maps.lo.a2_w, maps.lo.w3k, p.b3, buf.hi.a3, buf.lo.a3, frames};
    S.b(PS_CONV3_FWD); SRL_TRY(res_fwd_launch<RConv3Fwd>(q, cdiv(frames * 81, 128), kPersistentCtas, st, sp)); S.e(PS_CONV3_FWD); }
  { TFcFwd::Params q{maps.hi.a3m128, maps.hi.wfk, maps.lo.a3m128, maps.lo.wfk, buf.hpart, frames};
    static_assert(TFcFwd::SPLITS == FC_SPLITS, "split count");
    S.b(PS_FC_FWD);
    if (sp) SRL_TRY((igemm_tma_launch<TFcFwd, 1>(q, dim3(cdiv(frames, 128), 8 * FC_SPLITS), st)));
    else SRL_TRY((igemm_tma_launch<TFcFwd, 0>(q, dim3(cdiv(frames, 128), 8 * FC_SPLITS), st)));
    S.e(PS_FC_FWD); }
  return cudaSuccess;
}

cudaError_t encoder_backward(int frames, const EncoderBuffers& buf, const ParamPtrs& g, const TmaMaps& maps, int mode,
                             const StepStreams& S, BwdParts parts, bool a3t_done) {
  if (frames <= 0) return cudaSuccess;
  if ((mode != 0 && mode != 1) || !maps.valid) return cudaErrorInvalidValue;
  const int sp = mode;
  if (sp && !buf.lo.wpack) return cudaErrorInvalidValue;
  const bool do_fc = parts & BWD_FC, do_conv = parts & BWD_CONV;
  // The wgrad GEMMs only feed the optimizer: each runs on its own lane beside the dgrad chain (dh -> da3 -> da2 -> da1) and beside
  // each other.
  const cudaStream_t st = S.main, s1 = S.lane(LANE_FC_WGRAD), s2 = S.lane(LANE_CONV3_WGRAD), s3 = S.lane(LANE_CONV2_WGRAD);
  if (do_fc) {
    SRL_TRY(S.fork(LANE_FC_WGRAD));
    { const bool native = !sp && buf.a3t != nullptr;          // bf16 mode: B operand = a3 transposed into fc.weight's column order, 256-column tiles
      S.b(PS_FC_WGRAD);
      if (native) {
        if (!a3t_done) SRL_TRY(launch_a3_transpose(buf.hi.a3, buf.a3t, frames, s1));
        TFcWgradN::Params q{maps.hi.dhm64, maps.a3tm64, g.wf, g.bf, frames};
        SRL_TRY((igemm_tma_launch<TFcWgradN, 0>(q, dim3(1, 4 * (TFcWgradN::NCT + 1)), s1)));
      } else {
        TFcWgrad::Params q{maps.hi.dhm64, maps.hi.a3m64, maps.lo.dhm64, maps.lo.a3m64, g.wf, g.bf, frames};
        if (sp) SRL_TRY((igemm_tma_launch<TFcWgrad, 1>(q, dim3(1, 4 * 50), s1))); else SRL_TRY((igemm_tma_launch<TFcWgrad, 0>(q, dim3(1, 4 * 50), s1)));
      }
      S.e(PS_FC_WGRAD); }
    { TFcDgrad::Params q{maps.hi.dhm128, maps.hi.wfd, maps.lo.dhm128, maps.lo.wfd, buf.hi.a3, buf.hi.da3, buf.lo.da3, frames};
      S.b(PS_FC_DGRAD);
      if (sp) SRL_TRY((igemm_tma_launch<TFcDgrad, 1>(q, dim3(cdiv(frames, 128), 49), st))); else SRL_TRY((igemm_tma_launch<TFcDgrad, 0>(q, dim3(cdiv(frames, 128), 49), st)));
      S.e(PS_FC_DGRAD); }
    // the fc_wgrad lane also holds the head wgrad that the learner step forked there before this call: this join ends both
    if (!do_conv) SRL_TRY(S.join(LANE_FC_WGRAD));
  }
  if (!do_conv) return cudaSuccess;
  SRL_TRY(S.fork(LANE_CONV3_WGRAD));
  float* part3 = buf.wgrad_part;
  float* part2 = part3 + (size_t)WG_PART_CTAS * WSP_W3;
  float* part1 = part2 + (size_t)WG_PART_CTAS * WSP_W2;
  int n3 = 0, n2 = 0, n1 = 0;       // CTAs (partial slices) of the three wgrad launches
  { RConv3Wgrad::Params q{maps.hi.a2_w, maps.hi.da3g_b, maps.lo.a2_w, maps.lo.da3g_b, part3, frames * 81, 0};
    S.b(PS_CONV3_WGRAD); SRL_TRY(res_wgrad_launch<RConv3Wgrad>(q, side_wgrad_ctas(), s2, &n3, sp)); S.e(PS_CONV3_WGRAD); }
  // lanes: each side layer is reduced on its own lane as soon as its wgrad ends; collapsed: all three reduces run at the end,
  // together in the conv_wgrad_finalize profile slot
  if (!S.collapsed) SRL_TRY(launch_wgrad_reduce<WgradReduce3>(part3, n3, g.w3, g.b3, s2));
  { RConv3Dgrad::Params q{maps.hi.da3g_w, maps.hi.w3d, maps.lo.da3g_w, maps.lo.w3d, buf.hi.a2, buf.hi.da2, buf.lo.da2, frames};
    S.b(PS_CONV3_DGRAD); SRL_TRY(res_fwd_launch<RConv3Dgrad>(q, cdiv(frames * 81, 128), bwd_ctas(), st, sp)); S.e(PS_CONV3_DGRAD); }
  SRL_TRY(S.fork(LANE_CONV2_WGRAD));
  { RConv2Wgrad::Params q{maps.hi.a1p0_w, maps.hi.a1p1_w, maps.hi.da2g_b, maps.lo.a1p0_w, maps.lo.a1p1_w, maps.lo.da2g_b, part2, frames * 100, 0};
    S.b(PS_CONV2_WGRAD); SRL_TRY(res_wgrad_launch<RConv2Wgrad>(q, side_wgrad_ctas(), s3, &n2, sp)); S.e(PS_CONV2_WGRAD); }
  if (!S.collapsed) SRL_TRY(launch_wgrad_reduce<WgradReduce2>(part2, n2, g.w2, g.b2, s3));
  { RConv2Dgrad::Params q{maps.hi.da2g_w, maps.hi.w2d, maps.lo.da2g_w, maps.lo.w2d, buf.hi.a1, buf.hi.da1, buf.lo.da1, frames, buf.NF};
    S.b(PS_CONV2_DGRAD); SRL_TRY(res_fwd_launch<RConv2Dgrad>(q, cdiv(frames * 100, 128), bwd_ctas(), st, sp)); S.e(PS_CONV2_DGRAD); }
  { RConv1Wgrad::Params q{maps.xs_w, maps.hi.da1g_b, maps.lo.da1g_b, part1, frames * 441, 0};
    S.b(PS_CONV1_WGRAD); SRL_TRY(res_wgrad_launch<RConv1Wgrad>(q, bwd_ctas(), st, &n1, sp)); S.e(PS_CONV1_WGRAD); }
  S.b(PS_WGRAD_FINALIZE);
  if (S.collapsed) {
    SRL_TRY(launch_wgrad_reduce<WgradReduce3>(part3, n3, g.w3, g.b3, st));
    SRL_TRY(launch_wgrad_reduce<WgradReduce2>(part2, n2, g.w2, g.b2, st));
  }
  SRL_TRY(launch_wgrad_reduce<WgradReduce1>(part1, n1, g.w1, g.b1, st));
  S.e(PS_WGRAD_FINALIZE);
  // the fc_wgrad lane (with the learner step's head wgrad) only if this call ran the fc part: a BWD_FC call joined it already
  if (do_fc) SRL_TRY(S.join(LANE_FC_WGRAD));
  SRL_TRY(S.join(LANE_CONV3_WGRAD));
  SRL_TRY(S.join(LANE_CONV2_WGRAD));
  return cudaSuccess;
}

}  // namespace srl
