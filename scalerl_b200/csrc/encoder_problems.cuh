// Helpers shared by the TMA GEMM problems (res_problems.cuh, tma_problems.cuh) and the fused encoder front (enc_fused.cuh):
// bf16 packing, the u8 -> bf16 frame conversion and ReLU masks.
#pragma once
#include "common.cuh"

namespace srl {

typedef __nv_bfloat16 bf16;

SRL_DEVINL uint4 ldg16(const void* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }

// 8 consecutive u8 (two aligned u32 words) -> 8 bf16 (exact: 0..255 fit the 8-bit significand)
SRL_DEVINL uint4 u8x8_to_bf16x8(uint32_t w0, uint32_t w1) {
  float f[8];
  f[0] = __uint_as_float(__byte_perm(w0, 0x4B000000u, 0x7540)) - 8388608.f;
  f[1] = __uint_as_float(__byte_perm(w0, 0x4B000000u, 0x7541)) - 8388608.f;
  f[2] = __uint_as_float(__byte_perm(w0, 0x4B000000u, 0x7542)) - 8388608.f;
  f[3] = __uint_as_float(__byte_perm(w0, 0x4B000000u, 0x7543)) - 8388608.f;
  f[4] = __uint_as_float(__byte_perm(w1, 0x4B000000u, 0x7540)) - 8388608.f;
  f[5] = __uint_as_float(__byte_perm(w1, 0x4B000000u, 0x7541)) - 8388608.f;
  f[6] = __uint_as_float(__byte_perm(w1, 0x4B000000u, 0x7542)) - 8388608.f;
  f[7] = __uint_as_float(__byte_perm(w1, 0x4B000000u, 0x7543)) - 8388608.f;
  return make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
}

// conv1's operand window from u8 frames: 150 rows (128 positions + 22 halo rows of the 21x21 space-to-depth grid) x 64 channels
// (c, dy, dx) = eight 16-byte chunks, SWIZZLE_128B, the layout TMA gives a window of xs.  SLOTS * 8 threads fill it: thread
// (gp = t & 7, rb = t >> 3) converts chunk gp = (c = gp >> 1, dy = 2 (gp & 1), 2 (gp & 1) + 1) of rows rb, rb + SLOTS, ...: two
// 4-byte runs, dx = 0..3 of source rows 4Y + dy and 4Y + dy + 1 at byte 4X, 8 bf16 exactly as obs_s2d_kernel converts them.
// The source is a u8 image of whole 336-byte source-row groups (Y = 0, 1, ...) in every channel plane; window row r is position
// q0 + r of the image (Y = q / 21, X = q % 21) and positions at or past qend are zero.  load() reads the image into registers,
// store() writes the window and hands every chunk of a position before qend to f(row, v).
template <int SLOTS>
struct S2dWindow {
  static constexpr int ROWS = 150, K = (ROWS + SLOTS - 1) / SLOTS;
  uint32_t w0[K], w1[K], valid = 0;
  // img: the image at the thread's channel plane c, source row 2 (gp & 1).  Shared-pipe loads (ld.shared, in order with the mbarrier
  // waits around them) on 32-bit addresses; a row past qend keeps zero words, which convert to +0
  SRL_DEVINL void load(const uint8_t* img, int rb, int q0, int qend) {
    const uint32_t base = smem_u32(img);
    int q = q0 + rb, Y = q / 21, X = q - Y * 21;
#pragma unroll
    for (int k = 0; k < K; ++k) {
      w0[k] = 0u; w1[k] = 0u;
      if (rb + SLOTS * k < ROWS && q < qend) {
        const uint32_t a = base + Y * 336 + 4 * X;
        asm volatile("ld.shared.b32 %0, [%1];" : "=r"(w0[k]) : "r"(a) : "memory");
        asm volatile("ld.shared.b32 %0, [%1];" : "=r"(w1[k]) : "r"(a + 84) : "memory");
        valid |= 1u << k;
      }
      q += SLOTS; X += SLOTS % 21; Y += SLOTS / 21;
      if (X >= 21) { X -= 21; Y += 1; }
    }
  }
  template <class F>
  SRL_DEVINL void store(uint8_t* win, int gp, int rb, F&& f) const {
    const uint32_t base = smem_u32(win);
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int row = rb + SLOTS * k;
      if (SLOTS * (k + 1) <= ROWS || row < ROWS) {        // every slot has rows 0 .. ROWS / SLOTS - 1
        const uint4 v = u8x8_to_bf16x8(w0[k], w1[k]);
        if ((valid >> k) & 1) f(row, v);
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(base + swz128(row, gp)), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
                     : "memory");
      }
    }
  }
};

SRL_DEVINL void store_bf16x16(bf16* dst, const float (&v)[16]) {
  uint4 a = make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
  uint4 b = make_uint4(pack_bf16x2(v[8], v[9]), pack_bf16x2(v[10], v[11]), pack_bf16x2(v[12], v[13]), pack_bf16x2(v[14], v[15]));
  reinterpret_cast<uint4*>(dst)[0] = a;
  reinterpret_cast<uint4*>(dst)[1] = b;
}
// v[j] *= (mask[j] > 0) for 16 bf16 mask values
SRL_DEVINL void relu_mask16(const bf16* mask, float (&v)[16]) {
  uint4 a = ldg16(mask), b = ldg16(mask + 8);
  const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (!(bf16_lo(w[i]) > 0.f)) v[2 * i] = 0.f;
    if (!(bf16_hi(w[i]) > 0.f)) v[2 * i + 1] = 0.f;
  }
}

// same with the 32 mask bytes already in registers (prefetched before the accumulator was waited for)
SRL_DEVINL void relu_mask16_pre(const uint4 (&m)[2], float (&v)[16]) {
  const uint32_t w[8] = {m[0].x, m[0].y, m[0].z, m[0].w, m[1].x, m[1].y, m[1].z, m[1].w};
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (!(bf16_lo(w[i]) > 0.f)) v[2 * i] = 0.f;
    if (!(bf16_hi(w[i]) > 0.f)) v[2 * i + 1] = 0.f;
  }
}
SRL_DEVINL void ld_mask16(const bf16* mask, uint4 (&m)[2]) { m[0] = ldg16(mask); m[1] = ldg16(mask + 8); }
// two bf16 values x, each kept where its bf16 mask value is > 0 and +0 elsewhere
SRL_DEVINL uint32_t relu_mask_bf16x2(uint32_t x, uint32_t m) {
  return (bf16_lo(m) > 0.f ? x & 0xFFFFu : 0u) | (bf16_hi(m) > 0.f ? x & 0xFFFF0000u : 0u);
}

}  // namespace srl
