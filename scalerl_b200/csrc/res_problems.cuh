// Resident-window problem definitions (see igemm_res.cuh) for conv1 / conv2 / conv3: forward, dgrad, wgrad.
//
// Row layouts (all bf16, 64 channels = 128 B per row, frames concatenated; "grid" = spatial grid of the conv input):
//   xs   [NF*441]   21x21 grid of conv1 (space-to-depth frame)            channel = (c,dy,dx)
//   a1   [2][NF*100] two row-parity planes of conv1's output, 10x10 grid of conv2: plane hp, row n*100 + (h>>1)*10 + (w>>1),
//                   channel = (w&1)*32 + c          (a stride-2 tap of conv2 = a unit row shift inside one plane)
//   a2   [NF*81]    9x9 grid of conv3
//   a3   [NF*49]    dense (the fc input)
//   da3g [NB*81]    d(conv3 out) on conv3's 9x9 grid, zeros outside the 7x7 valid outputs (those zeros ARE the padding of dgrad)
//   da2g [NB*100]   d(conv2 out) on conv2's 10x10 grid, zeros outside 9x9
//   da1g [NB*441]   d(conv1 out) on conv1's 21x21 grid, zeros outside 20x20; 32 channels = 64 B per row (SWIZZLE_64B tiles)
#pragma once
#include "igemm_res.cuh"
#include "encoder_problems.cuh"

namespace srl {

// bf16 store of 16 accumulator values; in the split (fp32-accurate) mode also the low tensor: lo = bf16(v - bf16(v))
template <int SPLIT>
SRL_DEVINL void store_act16(bf16* hi, bf16* lo, size_t elem_off, const float (&v)[16]) {
  store_bf16x16(hi + elem_off, v);
  if constexpr (SPLIT) {
    float r[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) r[j] = v[j] - __bfloat162float(__float2bfloat16_rn(v[j]));
    store_bf16x16(lo + elem_off, r);
  }
}

// ================================================================================================ forward
struct RConv1Fwd {   // 2x2 s1 over xs (== 8x8 s4 over the frame): taps (kh2,kw2) -> shifts {0, 1, 21, 22}
  static constexpr int KID = 11;        // diagnostics timeline id
  static constexpr int BN = 32, NT = 4, NWIN = 1, WROWS = 128 + 22, STAGES = 4, SPLIT_STAGES = 4;
  static constexpr bool A_LO = false;        // the frames are exact in bf16: only the weights have a low tensor
  struct Params { SRL_TMAP in0; SRL_TMAP w; SRL_TMAP w_lo; const float* bias; bf16* out; bf16* out_lo; int NF; int NFS; };   // NF frames now, NFS = frames the a1 planes are strided for
  // conv1's K-major weight copy (w1k) is written by the frame-conversion kernel's extra blocks (obs_s2d_kernel, encoder.cu), not by
  // pack_weights_kernel: conv1 then depends only on its stream predecessor and never waits for the re-pack (encoder_forward joins the
  // re-pack stream only before conv2); the weight tiles are therefore loaded AFTER griddepcontrol.wait
  static constexpr bool W_AFTER_WAIT = true;
  static constexpr int U8_BYTES = 0;        // the windows come from TMA loads of xs (FromFrames: converted from the frames)
  struct FromFrames;                        // the same GEMM fed straight from the u8 frames
  SRL_DEVINL static void prefetch(const Params& p) { tma_prefetch_desc(&p.in0); tma_prefetch_desc(&p.w); }
  SRL_DEVINL static int num_tiles(const Params& p) { return (p.NF * 441 + 127) >> 7; }
  SRL_DEVINL static constexpr int tap_win(int) { return 0; }
  SRL_DEVINL static constexpr int tap_shift(int j) { return (j >> 1) * 21 + (j & 1); }
  SRL_DEVINL static void load_windows(const Params& p, int t, uint8_t* dst, int, uint64_t* bar, bool) { tma_load_2d(dst, &p.in0, bar, 0, t * 128); }
  SRL_DEVINL static void prefetch16(const Params&, int, int, int, uint4 (&)[2]) {}
  // bf16 mode: the tile's 128 positions x 32 channels (64 B each) are staged in shared memory and leave as 16-byte pieces, four per
  // position, consecutive lanes on consecutive pieces: positions ow, ow + 1 fill one 128-byte a1 row, so a warp stores 512
  // contiguous bytes of an output row where a row per thread touched 16 rows per store
  static constexpr int TILE_ROWB = 80;
  SRL_DEVINL static void prefetch_tile(const Params&, int, int, uint4 (&)[BN / 16][2]) {}
  SRL_DEVINL static void epilogue_tile(const Params& p, int t, int wt, const float (&acc)[2][BN / 2], uint8_t* img, int bar,
                                       const uint4 (&)[BN / 16][2]) {
    wg_acc_stage_bf16<BN, TILE_ROWB>(acc, img, wt, bar, [&](int c, float v) { return fmaxf(fmaf(v, 1.0f / 255.0f, __ldg(p.bias + c)), 0.f); });
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      const int e = s * 128 + wt, q = e >> 2, k = e & 3;
      const int Q = t * 128 + q, n = Q / 441, r = Q - n * 441, oh = r / 21, ow = r - oh * 21;
      if (n >= p.NF || oh >= 20 || ow >= 20) continue;
      const size_t prow = (size_t)(oh & 1) * p.NFS * 100 + (size_t)n * 100 + (oh >> 1) * 10 + (ow >> 1);
      *reinterpret_cast<uint4*>(p.out + prow * 64 + (ow & 1) * 32 + k * 8) = *reinterpret_cast<const uint4*>(img + q * TILE_ROWB + k * 16);
    }
  }
  template <int SPLIT>
  SRL_DEVINL static void epilogue16(const Params& p, int t, int row, int c0, float (&v)[16], const uint4 (&)[2]) {
    const int Q = t * 128 + row, n = Q / 441, r = Q - n * 441, oh = r / 21, ow = r - oh * 21;
    if (n >= p.NF || oh >= 20 || ow >= 20) return;
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = fmaxf(fmaf(v[j], 1.0f / 255.0f, __ldg(p.bias + c0 + j)), 0.f);
    const size_t prow = (size_t)(oh & 1) * p.NFS * 100 + (size_t)n * 100 + (oh >> 1) * 10 + (ow >> 1);    // plane stride: the buffer's frame capacity
    store_act16<SPLIT>(p.out, p.out_lo, prow * 64 + (ow & 1) * 32 + c0, v);
  }
};

// conv1's forward fed straight from the u8 frames (bf16 mode, 16-byte aligned frames).  The producer warpgroup builds each window in
// shared memory: warp 8 brings in the source rows it covers (one bulk copy per frame and channel plane), warps 9-11 convert them into
// the SWIZZLE_128B window a TMA load of xs would give (S2dWindow) and write its rows 0..127 -- the tile's own positions -- to xs, conv1
// wgrad's operand, instead of reading xs back.  The MMAs and the epilogue are RConv1Fwd's on the same operand bytes.
struct RConv1Fwd::FromFrames : RConv1Fwd {
  static constexpr int SPAN = 9;                    // rows of the 21x21 grid (or of two frames' grids) a 150-row window touches, at most
  static constexpr int U8_PLANE = SPAN * 336;       // one channel plane of the staged source rows: a grid row is 4 source rows of 84 B
  static constexpr int U8_BYTES = 4 * U8_PLANE;     // per ring stage
  static constexpr int CONV_SLOTS = 12;             // converter threads (warps 9-11) / 8 chunks per row
  struct Params : RConv1Fwd::Params { const uint8_t* obs; bf16* xs; };
  SRL_DEVINL static void prefetch(const Params& p) { tma_prefetch_desc(&p.w); }
  // grid rows r0 .. r1 of tile t's window (positions t * 128 .. t * 128 + 149, clipped to the frames), plane c at dst + c * U8_PLANE
  SRL_DEVINL static void load_u8(const Params& p, int t, uint8_t* dst, uint64_t* bar) {
    const int q0 = t * 128, q1 = min(q0 + WROWS, p.NF * 441) - 1, r0 = q0 / 21, r1 = q1 / 21;
    mbar_arrive_expect_tx(bar, (r1 - r0 + 1) * 4 * 336);
    for (int ra = r0; ra <= r1;) {                  // a window straddles at most two frames
      const int n = ra / 21, rz = min(r1, n * 21 + 20);
      const uint8_t* src = p.obs + (size_t)n * 28224 + (ra - n * 21) * 336;
      for (int c = 0; c < 4; ++c) bulk_load_1d(dst + c * U8_PLANE + (ra - r0) * 336, src + c * 7056, (rz - ra + 1) * 336, bar);
      ra = rz + 1;
    }
  }
};

struct RConv2Fwd {   // 4x4 s2 over a1: tap j = (kh, kww): plane kh&1, shift (kh>>1)*10 + kww, K-block = (kh, kw in {2kww, 2kww+1}, c)
  static constexpr int KID = 12;        // diagnostics timeline id
  static constexpr bool W_AFTER_WAIT = false;
  static constexpr int U8_BYTES = 0;        // the windows come from TMA loads
  static constexpr int BN = 64, NT = 8, NWIN = 2, WROWS = 128 + 11, STAGES = 3, SPLIT_STAGES = 1;
  static constexpr bool A_LO = true;
  struct Params { SRL_TMAP in0; SRL_TMAP in1; SRL_TMAP w; SRL_TMAP in0_lo; SRL_TMAP in1_lo; SRL_TMAP w_lo; const float* bias; bf16* out; bf16* out_lo; int NF; };
  SRL_DEVINL static void prefetch(const Params& p) { tma_prefetch_desc(&p.in0); tma_prefetch_desc(&p.in1); tma_prefetch_desc(&p.w); }
  SRL_DEVINL static int num_tiles(const Params& p) { return (p.NF * 100 + 127) >> 7; }
  SRL_DEVINL static constexpr int tap_win(int j) { return (j >> 1) & 1; }
  SRL_DEVINL static constexpr int tap_shift(int j) { return (j >> 2) * 10 + (j & 1); }
  SRL_DEVINL static void load_windows(const Params& p, int t, uint8_t* dst, int win_bytes, uint64_t* bar, bool lo) {
    tma_load_2d(dst, lo ? &p.in0_lo : &p.in0, bar, 0, t * 128);
    tma_load_2d(dst + win_bytes, lo ? &p.in1_lo : &p.in1, bar, 0, t * 128);
  }
  SRL_DEVINL static void prefetch16(const Params&, int, int, int, uint4 (&)[2]) {}
  // bf16 mode: the tile's 128 positions x 64 channels are staged in shared memory and leave as 16-byte pieces, eight per position,
  // consecutive lanes on consecutive pieces: a warp stores four whole a2 rows, consecutive along a valid run of 9 positions, where a
  // row per thread touched 32 rows per store.  The 18 KB image fits the row hand-off's buffer: shared memory and ring depth are unchanged
  static constexpr int TILE_ROWB = 144;
  SRL_DEVINL static void prefetch_tile(const Params&, int, int, uint4 (&)[BN / 16][2]) {}
  SRL_DEVINL static void epilogue_tile(const Params& p, int t, int wt, const float (&acc)[2][BN / 2], uint8_t* img, int bar,
                                       const uint4 (&)[BN / 16][2]) {
    wg_acc_stage_bf16<BN, TILE_ROWB>(acc, img, wt, bar, [&](int c, float v) { return fmaxf(v + __ldg(p.bias + c), 0.f); });
#pragma unroll
    for (int s = 0; s < 8; ++s) {
      const int e = s * 128 + wt, q = e >> 3, k = e & 7;
      const int Q = t * 128 + q, n = Q / 100, r = Q - n * 100, oh = r / 10, ow = r - oh * 10;
      if (n >= p.NF || oh >= 9 || ow >= 9) continue;
      *reinterpret_cast<uint4*>(p.out + ((size_t)n * 81 + oh * 9 + ow) * 64 + k * 8) = *reinterpret_cast<const uint4*>(img + q * TILE_ROWB + k * 16);
    }
  }
  template <int SPLIT>
  SRL_DEVINL static void epilogue16(const Params& p, int t, int row, int c0, float (&v)[16], const uint4 (&)[2]) {
    const int Q = t * 128 + row, n = Q / 100, r = Q - n * 100, oh = r / 10, ow = r - oh * 10;
    if (n >= p.NF || oh >= 9 || ow >= 9) return;
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = fmaxf(v[j] + __ldg(p.bias + c0 + j), 0.f);
    store_act16<SPLIT>(p.out, p.out_lo, ((size_t)n * 81 + oh * 9 + ow) * 64 + c0, v);
  }
};

struct RConv3Fwd {   // 3x3 s1 over a2: tap (kh,kw) -> shift kh*9 + kw
  static constexpr int KID = 13;        // diagnostics timeline id
  static constexpr bool W_AFTER_WAIT = false;
  static constexpr int U8_BYTES = 0;        // the windows come from TMA loads
  static constexpr int BN = 64, NT = 9, NWIN = 1, WROWS = 128 + 20, STAGES = 4, SPLIT_STAGES = 2;
  static constexpr bool A_LO = true;
  struct Params { SRL_TMAP in0; SRL_TMAP w; SRL_TMAP in0_lo; SRL_TMAP w_lo; const float* bias; bf16* out; bf16* out_lo; int NF; };
  SRL_DEVINL static void prefetch(const Params& p) { tma_prefetch_desc(&p.in0); tma_prefetch_desc(&p.w); }
  SRL_DEVINL static int num_tiles(const Params& p) { return (p.NF * 81 + 127) >> 7; }
  SRL_DEVINL static constexpr int tap_win(int) { return 0; }
  SRL_DEVINL static constexpr int tap_shift(int j) { return (j / 3) * 9 + j % 3; }
  SRL_DEVINL static void load_windows(const Params& p, int t, uint8_t* dst, int, uint64_t* bar, bool lo) { tma_load_2d(dst, lo ? &p.in0_lo : &p.in0, bar, 0, t * 128); }
  SRL_DEVINL static void prefetch16(const Params&, int, int, int, uint4 (&)[2]) {}
  // bf16 mode: staged tile as in RConv2Fwd; a warp stores four whole a3 rows, consecutive along a valid run of 7 positions
  static constexpr int TILE_ROWB = 144;
  SRL_DEVINL static void prefetch_tile(const Params&, int, int, uint4 (&)[BN / 16][2]) {}
  SRL_DEVINL static void epilogue_tile(const Params& p, int t, int wt, const float (&acc)[2][BN / 2], uint8_t* img, int bar,
                                       const uint4 (&)[BN / 16][2]) {
    wg_acc_stage_bf16<BN, TILE_ROWB>(acc, img, wt, bar, [&](int c, float v) { return fmaxf(v + __ldg(p.bias + c), 0.f); });
#pragma unroll
    for (int s = 0; s < 8; ++s) {
      const int e = s * 128 + wt, q = e >> 3, k = e & 7;
      const int Q = t * 128 + q, n = Q / 81, r = Q - n * 81, oh = r / 9, ow = r - oh * 9;
      if (n >= p.NF || oh >= 7 || ow >= 7) continue;
      *reinterpret_cast<uint4*>(p.out + ((size_t)n * 49 + oh * 7 + ow) * 64 + k * 8) = *reinterpret_cast<const uint4*>(img + q * TILE_ROWB + k * 16);
    }
  }
  template <int SPLIT>
  SRL_DEVINL static void epilogue16(const Params& p, int t, int row, int c0, float (&v)[16], const uint4 (&)[2]) {
    const int Q = t * 128 + row, n = Q / 81, r = Q - n * 81, oh = r / 9, ow = r - oh * 9;
    if (n >= p.NF || oh >= 7 || ow >= 7) return;
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = fmaxf(v[j] + __ldg(p.bias + c0 + j), 0.f);
    store_act16<SPLIT>(p.out, p.out_lo, ((size_t)n * 49 + oh * 7 + ow) * 64 + c0, v);
  }
};

// ================================================================================================ dgrad
struct RConv3Dgrad {   // da2[ih,iw] = sum_{kh,kw} da3g[(ih-kh),(iw-kw)] W3[:, :, kh, kw]: shifts -(kh*9+kw); window starts 20 rows early
  static constexpr int KID = 14;        // diagnostics timeline id
  static constexpr bool W_AFTER_WAIT = false;
  static constexpr int U8_BYTES = 0;        // the windows come from TMA loads
  static constexpr int BN = 64, NT = 9, NWIN = 1, WROWS = 128 + 20, STAGES = 4, SPLIT_STAGES = 2;
  static constexpr bool A_LO = true;
  struct Params { SRL_TMAP in0; SRL_TMAP w; SRL_TMAP in0_lo; SRL_TMAP w_lo; const bf16* act; bf16* dx; bf16* dx_lo; int NB; };
  SRL_DEVINL static void prefetch(const Params& p) { tma_prefetch_desc(&p.in0); tma_prefetch_desc(&p.w); }
  SRL_DEVINL static int num_tiles(const Params& p) { return (p.NB * 81 + 127) >> 7; }
  SRL_DEVINL static constexpr int tap_win(int) { return 0; }
  SRL_DEVINL static constexpr int tap_shift(int j) { return 20 - ((j / 3) * 9 + j % 3); }
  SRL_DEVINL static void load_windows(const Params& p, int t, uint8_t* dst, int, uint64_t* bar, bool lo) { tma_load_2d(dst, lo ? &p.in0_lo : &p.in0, bar, 0, t * 128 - 20); }
  SRL_DEVINL static void prefetch16(const Params& p, int t, int row, int c0, uint4 (&m)[2]) {
    const int Q = t * 128 + row;
    if (Q < p.NB * 81) ld_mask16(p.act + (size_t)Q * 64 + c0, m);                  // a2 lives on the same 9x9 grid
  }
  // bf16 mode: the tile (128 positions x 64 channels) is staged in shared memory and leaves as 16-byte pieces e = s * 128 + wt
  // (position q = e >> 3, piece k = e & 7): the tile's mask is one contiguous 16 KB run of a2 and each position's 128 bytes are one
  // da2g row, so a warp loads 512 contiguous bytes of mask and stores four whole da2g rows where a row per thread touched 32 rows per
  // instruction.  Masking the rounded value gives the bits of rounding the masked one.
  static constexpr int TILE_ROWB = 144;
  SRL_DEVINL static void prefetch_tile(const Params& p, int t, int wt, uint4 (&m)[BN / 16][2]) {
#pragma unroll
    for (int s = 0; s < 8; ++s) {
      const int e = s * 128 + wt, Q = t * 128 + (e >> 3);
      if (Q < p.NB * 81) m[s >> 1][s & 1] = ldg16(p.act + (size_t)Q * 64 + (e & 7) * 8);
    }
  }
  SRL_DEVINL static void epilogue_tile(const Params& p, int t, int wt, const float (&acc)[2][BN / 2], uint8_t* img, int bar,
                                       const uint4 (&m)[BN / 16][2]) {
    wg_acc_stage_bf16<BN, TILE_ROWB>(acc, img, wt, bar, [](int, float v) { return v; });
#pragma unroll
    for (int s = 0; s < 8; ++s) {
      const int e = s * 128 + wt, q = e >> 3, k = e & 7;
      const int Q = t * 128 + q, n = Q / 81, r = Q - n * 81, ih = r / 9, iw = r - ih * 9;
      if (n >= p.NB) continue;
      const uint4 x = *reinterpret_cast<const uint4*>(img + q * TILE_ROWB + k * 16), mk = m[s >> 1][s & 1];
      *reinterpret_cast<uint4*>(p.dx + ((size_t)n * 100 + ih * 10 + iw) * 64 + k * 8) =
          make_uint4(relu_mask_bf16x2(x.x, mk.x), relu_mask_bf16x2(x.y, mk.y), relu_mask_bf16x2(x.z, mk.z), relu_mask_bf16x2(x.w, mk.w));
    }
  }
  template <int SPLIT>
  SRL_DEVINL static void epilogue16(const Params& p, int t, int row, int c0, float (&v)[16], const uint4 (&m)[2]) {
    const int Q = t * 128 + row, n = Q / 81, r = Q - n * 81, ih = r / 9, iw = r - ih * 9;
    if (n >= p.NB) return;
    relu_mask16_pre(m, v);
    store_act16<SPLIT>(p.dx, p.dx_lo, ((size_t)n * 100 + ih * 10 + iw) * 64 + c0, v);           // da2g: conv2's 10x10 grid
  }
};

struct RConv2Dgrad {   // the 4 stride-parity classes share A (da2g at (i'-kh', j'-kw')): one N = 4 x 32 GEMM; shifts -(kh'*10 + kw')
  static constexpr int KID = 15;        // diagnostics timeline id
  static constexpr bool W_AFTER_WAIT = false;
  static constexpr int U8_BYTES = 0;        // the windows come from TMA loads
  static constexpr int BN = 128, NT = 4, NWIN = 1, WROWS = 128 + 11, STAGES = 3, SPLIT_STAGES = 2;
  static constexpr bool A_LO = true;
  struct Params { SRL_TMAP in0; SRL_TMAP w; SRL_TMAP in0_lo; SRL_TMAP w_lo; const bf16* act; bf16* dx; bf16* dx_lo; int NB; int NF; };
  SRL_DEVINL static void prefetch(const Params& p) { tma_prefetch_desc(&p.in0); tma_prefetch_desc(&p.w); }
  SRL_DEVINL static int num_tiles(const Params& p) { return (p.NB * 100 + 127) >> 7; }
  SRL_DEVINL static constexpr int tap_win(int) { return 0; }
  SRL_DEVINL static constexpr int tap_shift(int j) { return 11 - ((j >> 1) * 10 + (j & 1)); }
  SRL_DEVINL static void load_windows(const Params& p, int t, uint8_t* dst, int, uint64_t* bar, bool lo) { tma_load_2d(dst, lo ? &p.in0_lo : &p.in0, bar, 0, t * 128 - 11); }
  SRL_DEVINL static void prefetch16(const Params& p, int t, int row, int c0, uint4 (&m)[2]) {
    const int Q = t * 128 + row, cls = c0 >> 5, c = c0 & 31;
    if (Q < p.NB * 100) ld_mask16(p.act + ((size_t)(cls >> 1) * p.NF * 100 + Q) * 64 + (cls & 1) * 32 + c, m);   // a1 plane ph, same row Q
  }
  // bf16 mode: the tile (128 positions x 4 classes x 32 channels) is staged in shared memory; it leaves as 16-byte pieces
  // e = s * 128 + wt (ph = e >> 10, position q = (e >> 3) & 127, piece k = e & 7 of the 128 bytes (pw, c) of row q, plane ph).
  // Those 128 bytes are the a1 row the ReLU mask comes from and the two da1g rows (2i + ph, 2j + pw) they go to, and position q + 1
  // continues both two rows on: a warp loads 512 contiguous bytes of mask and stores 512 contiguous bytes of da1g where a row per
  // thread touched 32 rows per instruction.  Masking the rounded value gives the bits of rounding the masked one.
  static constexpr int TILE_ROWB = 272;
  SRL_DEVINL static void prefetch_tile(const Params& p, int t, int wt, uint4 (&m)[BN / 16][2]) {
#pragma unroll
    for (int s = 0; s < 16; ++s) {
      const int e = s * 128 + wt, ph = e >> 10, Q = t * 128 + ((e >> 3) & 127);
      if (Q < p.NB * 100) m[s >> 1][s & 1] = ldg16(p.act + ((size_t)ph * p.NF * 100 + Q) * 64 + (e & 7) * 8);
    }
  }
  SRL_DEVINL static void epilogue_tile(const Params& p, int t, int wt, const float (&acc)[2][BN / 2], uint8_t* img, int bar,
                                       const uint4 (&m)[BN / 16][2]) {
    wg_acc_stage_bf16<BN, TILE_ROWB>(acc, img, wt, bar, [](int, float v) { return v; });
#pragma unroll
    for (int s = 0; s < 16; ++s) {
      const int e = s * 128 + wt, ph = e >> 10, q = (e >> 3) & 127, k = e & 7;
      const int Q = t * 128 + q, n = Q / 100, r = Q - n * 100, i = r / 10, j = r - i * 10;
      if (n >= p.NB) continue;
      const uint4 x = *reinterpret_cast<const uint4*>(img + q * TILE_ROWB + ph * 128 + k * 16), mk = m[s >> 1][s & 1];
      *reinterpret_cast<uint4*>(p.dx + ((size_t)n * 441 + (2 * i + ph) * 21 + 2 * j) * 32 + k * 8) =
          make_uint4(relu_mask_bf16x2(x.x, mk.x), relu_mask_bf16x2(x.y, mk.y), relu_mask_bf16x2(x.z, mk.z), relu_mask_bf16x2(x.w, mk.w));
    }
  }
  template <int SPLIT>
  SRL_DEVINL static void epilogue16(const Params& p, int t, int row, int c0, float (&v)[16], const uint4 (&m)[2]) {
    const int Q = t * 128 + row, n = Q / 100, r = Q - n * 100, i = r / 10, j = r - i * 10;
    if (n >= p.NB) return;
    const int cls = c0 >> 5, c = c0 & 31, ph = cls >> 1, pw = cls & 1;
    relu_mask16_pre(m, v);
    store_act16<SPLIT>(p.dx, p.dx_lo, ((size_t)n * 441 + (2 * i + ph) * 21 + 2 * j + pw) * 32 + c, v);   // da1g: conv1's 21x21 grid, 32-channel rows
  }
};

// ================================================================================================ wgrad
// Every wgrad CTA stores its accumulators (and bias sums) in its own slice of the per-CTA partials, PART floats at
// ws + blockIdx.x * PART, in the kernels' native [tap-block][row][co] order followed by the bias; conv_wgrad_reduce_kernel
// (encoder.cu, one launch per layer) adds the slices in CTA order straight into the PyTorch-layout weight gradient and the bias gradient.
// Tap block b = 64 rows of dW (one m64 wgmma accumulator) = window rows starting blk_shift(b) in window blk_win(b).
struct RConv3Wgrad {   // block b = tap b.  ws: [10 taps][64 c][64 co] fp32 (co contiguous; the tenth block is not written), db3
  static constexpr int KID = 21;        // diagnostics timeline id
  static constexpr int NBLK = 9, CWG = 3, NWIN = 1, WROWS = 128 + 20, STAGES = 3, SPLIT_STAGES = 2;
  static constexpr bool A_LO = true;
  static constexpr bool SMEM_BIAS = false;     // db3 from an all-ones wgmma (bf16 mode; the split mode sums the dY columns)
  static constexpr int BIAS_CH = 64, DY_CH = 64;
  static constexpr int PART = WSP_W3;
  struct Params { SRL_TMAP in0; SRL_TMAP dy; SRL_TMAP in0_lo; SRL_TMAP dy_lo; float* ws; int P; int chunks_per_cta; };
  SRL_DEVINL static void prefetch(const Params& p) { tma_prefetch_desc(&p.in0); tma_prefetch_desc(&p.dy); }
  SRL_DEVINL static constexpr int blk_win(int) { return 0; }
  SRL_DEVINL static constexpr int blk_shift(int b) { return (b / 3) * 9 + b % 3; }
  SRL_DEVINL static void load_windows(const Params& p, int chunk, uint8_t* dst, int, uint64_t* bar, bool lo) { tma_load_2d(dst, lo ? &p.in0_lo : &p.in0, bar, 0, chunk * 128); }
};

struct RConv2Wgrad {   // block b = (kh = b >> 1, kww = b & 1): rows = (kw = 2kww + wp, c), row-parity plane kh & 1
  static constexpr int KID = 22;        // diagnostics timeline id
  static constexpr int NBLK = 8, CWG = 2, NWIN = 2, WROWS = 128 + 11, STAGES = 3, SPLIT_STAGES = 1;
  static constexpr bool A_LO = true;
  static constexpr bool SMEM_BIAS = true;
  static constexpr int BIAS_CH = 64, DY_CH = 64;
  static constexpr int PART = WSP_W2;
  struct Params { SRL_TMAP in0; SRL_TMAP in1; SRL_TMAP dy; SRL_TMAP in0_lo; SRL_TMAP in1_lo; SRL_TMAP dy_lo; float* ws; int P; int chunks_per_cta; };   // ws: [4 kh][128 (kw,c)][64 co]
  SRL_DEVINL static void prefetch(const Params& p) { tma_prefetch_desc(&p.in0); tma_prefetch_desc(&p.in1); tma_prefetch_desc(&p.dy); }
  SRL_DEVINL static constexpr int blk_win(int b) { return (b >> 1) & 1; }
  SRL_DEVINL static constexpr int blk_shift(int b) { return (b >> 2) * 10 + (b & 1); }
  SRL_DEVINL static void load_windows(const Params& p, int chunk, uint8_t* dst, int win_bytes, uint64_t* bar, bool lo) {
    tma_load_2d(dst, lo ? &p.in0_lo : &p.in0, bar, 0, chunk * 128);
    tma_load_2d(dst + win_bytes, lo ? &p.in1_lo : &p.in1, bar, 0, chunk * 128);
  }
};

struct RConv1Wgrad {   // block b = (kh2 = b >> 1, kw2 = b & 1): rows = (c, dy, dx)
  static constexpr int KID = 23;        // diagnostics timeline id
  static constexpr int NBLK = 4, CWG = 2, NWIN = 1, WROWS = 128 + 22, STAGES = 5, SPLIT_STAGES = 3;
  static constexpr bool A_LO = false;          // the frames are exact in bf16
  static constexpr bool SMEM_BIAS = true;
  static constexpr int BIAS_CH = 32;
  static constexpr int DY_CH = 32;             // da1g rows are 32 channels (64 B): SWIZZLE_64B dY tiles, N = 32 MMAs
  static constexpr int PART = WSP_W1;
  struct Params { SRL_TMAP in0; SRL_TMAP dy; SRL_TMAP dy_lo; float* ws; int P; int chunks_per_cta; };   // ws: [2 kh2][128 (kw2,c,dy,dx)][32 co]
  SRL_DEVINL static void prefetch(const Params& p) { tma_prefetch_desc(&p.in0); tma_prefetch_desc(&p.dy); }
  SRL_DEVINL static constexpr int blk_win(int) { return 0; }
  SRL_DEVINL static constexpr int blk_shift(int b) { return (b >> 1) * 21 + (b & 1); }
  SRL_DEVINL static void load_windows(const Params& p, int chunk, uint8_t* dst, int, uint64_t* bar, bool) { tma_load_2d(dst, &p.in0, bar, 0, chunk * 128); }
};

}  // namespace srl
