// TMA box programs + epilogues of the fc layer's three GEMMs (see igemm_tma.cuh for the mainloop, encoder.cu for the
// tensor maps; the conv layers are in res_problems.cuh).  Reference: scalerl/algorithms/utils/atari_model.py:46,100-101.
#pragma once
#include "igemm_tma.cuh"
#include "encoder_problems.cuh"   // store_bf16x16, relu_mask16, bf16 helpers

namespace srl {

#define SRL_TMAP alignas(64) CUtensorMap

// ============================================================================================ fc
struct TFcFwd {
  static constexpr int KID = 31;        // diagnostics timeline id
  static constexpr bool PREFETCH = false;   // split-K partials; grid.y = 8 N-tiles x FC_SPLITS, ty = nt*FC_SPLITS + split
  static constexpr int BN = 64, STAGES = 4, SPLITS = 4;
  static constexpr bool A_MN = false, B_MN = false, ZERO_INIT = false;
  static constexpr int KROWS = 64;
  struct Params { SRL_TMAP a3m; SRL_TMAP w; SRL_TMAP a3m_lo; SRL_TMAP w_lo; float* out; int M; };
  SRL_DEVINL static void prefetch(const Params& p) { tma_prefetch_desc(&p.a3m); tma_prefetch_desc(&p.w); }
  SRL_DEVINL static int kb_begin(int split) { return (49 * split) / SPLITS; }
  SRL_DEVINL static void issue_split(const Params& p, int tm, int ty, int kb, uint8_t* st, int a_bytes, int half, uint64_t* bar) {
    const int k = (kb_begin(ty % SPLITS) + kb) * 64;
    mbar_arrive_expect_tx(bar, 2 * (128 * 128 + 64 * 128));
    tma_load_2d(st, &p.a3m, bar, k, tm * 128);
    tma_load_2d(st + a_bytes, &p.w, bar, k, (ty / SPLITS) * 64);
    tma_load_2d(st + half, &p.a3m_lo, bar, k, tm * 128);
    tma_load_2d(st + half + a_bytes, &p.w_lo, bar, k, (ty / SPLITS) * 64);
  }
  template <int SPLIT>
  SRL_DEVINL static void epilogue16(const Params& p, int tm, int ty, int row, int c0, float (&v)[16]) { epilogue16(p, tm, ty, row, c0, v); }
  SRL_DEVINL static int num_kblocks(const Params&, int, int ty) { const int sp = ty % SPLITS; return kb_begin(sp + 1) - kb_begin(sp); }
  SRL_DEVINL static void issue(const Params& p, int tm, int ty, int kb, uint8_t* sA, uint8_t* sB, uint64_t* bar) {
    const int k = (kb_begin(ty % SPLITS) + kb) * 64;
    mbar_arrive_expect_tx(bar, 128 * 128 + 64 * 128);
    tma_load_2d(sA, &p.a3m, bar, k, tm * 128);
    tma_load_2d(sB, &p.w, bar, k, (ty / SPLITS) * 64);
  }
  SRL_DEVINL static void epilogue16(const Params& p, int tm, int ty, int row, int c0, float (&v)[16]) {
    const int m = tm * 128 + row;
    if (m >= p.M) return;
    float4* o = reinterpret_cast<float4*>(p.out + ((size_t)(ty % SPLITS) * p.M + m) * 512 + (ty / SPLITS) * 64 + c0);
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
  }
  // bf16 mode: the 128 x 64 fp32 tile leaves as 16-byte pieces e = s * 256 + t (row q = e >> 4, piece k = e & 15): a warp stores
  // two whole 256-byte row pieces of hpart, where a row per thread touched 32 rows 2 KB apart per store
  static constexpr int TILE_ROWB = 4 * BN + 32;
  SRL_DEVINL static void epilogue_tile(const Params& p, int tm, int ty, int t, const uint8_t* img, const uint4 (&)[1][2]) {
    float* out = p.out + (size_t)(ty % SPLITS) * p.M * 512 + (ty / SPLITS) * 64;
#pragma unroll
    for (int s = 0; s < 8; ++s) {
      const int e = s * 256 + t, q = e >> 4, k = e & 15, m = tm * 128 + q;
      if (m < p.M) *reinterpret_cast<float4*>(out + (size_t)m * 512 + k * 4) = *reinterpret_cast<const float4*>(img + q * TILE_ROWB + k * 16);
    }
  }
};

struct TFcDgrad {
  static constexpr int KID = 32;        // diagnostics timeline id
  static constexpr bool PREFETCH = true;   // da3[m][i] = (dh[m][:] . Wfc[:][i]) * (a3 > 0); grid = (ceil(M/128), 49)
  static constexpr int BN = 64, STAGES = 4;
  static constexpr bool A_MN = false, B_MN = false, ZERO_INIT = false;
  static constexpr int KROWS = 64;
  struct Params { SRL_TMAP dhm; SRL_TMAP w; SRL_TMAP dhm_lo; SRL_TMAP w_lo; const bf16* a3; bf16* da3; bf16* da3_lo; int M; };
  SRL_DEVINL static void prefetch(const Params& p) { tma_prefetch_desc(&p.dhm); tma_prefetch_desc(&p.w); }
  SRL_DEVINL static int num_kblocks(const Params&, int, int) { return 8; }
  SRL_DEVINL static void issue_split(const Params& p, int tm, int ty, int kb, uint8_t* st, int a_bytes, int half, uint64_t* bar) {
    mbar_arrive_expect_tx(bar, 2 * (128 * 128 + 64 * 128));
    tma_load_2d(st, &p.dhm, bar, kb * 64, tm * 128);
    tma_load_2d(st + a_bytes, &p.w, bar, kb * 64, ty * 64);
    tma_load_2d(st + half, &p.dhm_lo, bar, kb * 64, tm * 128);
    tma_load_2d(st + half + a_bytes, &p.w_lo, bar, kb * 64, ty * 64);
  }
  SRL_DEVINL static void issue(const Params& p, int tm, int ty, int kb, uint8_t* sA, uint8_t* sB, uint64_t* bar) {
    mbar_arrive_expect_tx(bar, 128 * 128 + 64 * 128);
    tma_load_2d(sA, &p.dhm, bar, kb * 64, tm * 128);
    tma_load_2d(sB, &p.w, bar, kb * 64, ty * 64);
  }
  SRL_DEVINL static void prefetch16(const Params& p, int tm, int ty, int row, int c0, uint4 (&mk)[2]) {
    const int m = tm * 128 + row;
    if (m < p.M) ld_mask16(p.a3 + (size_t)m * 3136 + ty * 64 + c0, mk);
  }
  SRL_DEVINL static void epilogue16(const Params& p, int tm, int ty, int row, int c0, float (&v)[16], const uint4 (&mk)[2]) {
    epilogue16<0>(p, tm, ty, row, c0, v, mk);
  }
  template <int SPLIT>
  SRL_DEVINL static void epilogue16(const Params& p, int tm, int ty, int row, int c0, float (&v)[16], const uint4 (&mk)[2]) {
    const int m = tm * 128 + row;
    if (m >= p.M) return;
    relu_mask16_pre(mk, v);
    // N-tile ty == one output pixel hw of conv3; da3g lives on conv3's 9x9 input grid (zeros outside the 7x7 outputs)
    const size_t o = ((size_t)m * 81 + (ty / 7) * 9 + ty % 7) * 64 + c0;
    store_bf16x16(p.da3 + o, v);
    if constexpr (SPLIT) {
      float r[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) r[j] = v[j] - __bfloat162float(__float2bfloat16_rn(v[j]));
      store_bf16x16(p.da3_lo + o, r);
    }
  }
  // bf16 mode: the tile (128 frames x 64 channels of one pixel) leaves as 16-byte pieces e = s * 256 + t (frame q = e >> 3, channels
  // 8k.. with k = e & 7): a warp loads four whole 128-byte mask rows of a3 and stores four whole da3 pixel rows, where a row per
  // thread touched 32 frames 10,368 bytes apart per store.  Masking the rounded value gives the bits of rounding the masked one.
  static constexpr int TILE_ROWB = 4 * BN + 32;
  SRL_DEVINL static void prefetch_tile(const Params& p, int tm, int ty, int t, uint4 (&mk)[2][2]) {
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      const int e = s * 256 + t, m = tm * 128 + (e >> 3);
      if (m < p.M) mk[s >> 1][s & 1] = ldg16(p.a3 + (size_t)m * 3136 + ty * 64 + (e & 7) * 8);
    }
  }
  SRL_DEVINL static void epilogue_tile(const Params& p, int tm, int ty, int t, const uint8_t* img, const uint4 (&mk)[2][2]) {
    bf16* out = p.da3 + ((ty / 7) * 9 + ty % 7) * 64;
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      const int e = s * 256 + t, q = e >> 3, k = e & 7, m = tm * 128 + q;
      if (m >= p.M) continue;
      const float4 a = *reinterpret_cast<const float4*>(img + q * TILE_ROWB + k * 32), b = *reinterpret_cast<const float4*>(img + q * TILE_ROWB + k * 32 + 16);
      const uint4 w = mk[s >> 1][s & 1];
      *reinterpret_cast<uint4*>(out + (size_t)m * 81 * 64 + k * 8) =
          make_uint4(relu_mask_bf16x2(pack_bf16x2(a.x, a.y), w.x), relu_mask_bf16x2(pack_bf16x2(a.z, a.w), w.y),
                     relu_mask_bf16x2(pack_bf16x2(b.x, b.y), w.z), relu_mask_bf16x2(pack_bf16x2(b.z, b.w), w.w));
    }
  }
};

SRL_DEVINL void fill_ones(uint8_t* dst, int bytes, int tid) {   // bf16 1.0 = 0x3F80
  uint4* q = reinterpret_cast<uint4*>(dst);
  for (int i = tid; i < bytes / 16; i += IGT_THREADS) q[i] = make_uint4(0x3F803F80u, 0x3F803F80u, 0x3F803F80u, 0x3F803F80u);
}

// (h,w,c)-ordered column tiles: used by the fp32-accurate split mode only (no low twin of a3t); the bf16 mode runs TFcWgradN below
struct TFcWgrad {
  static constexpr int KID = 33;        // diagnostics timeline id
  static constexpr bool PREFETCH = false;   // grid = (1, 4*50): ty = hw*4 + jt, hw == 49 is the ones slice (B = ones -> dbfc); stage = 64 frames
  static constexpr int BN = 64, STAGES = 4, KROWS = 64, TILE_ROWB = 0;
  static constexpr bool A_MN = true, B_MN = true, ZERO_INIT = true;
  struct Params { SRL_TMAP dhm; SRL_TMAP a3m; SRL_TMAP dhm_lo; SRL_TMAP a3m_lo; float* dw; float* db; int M; };
  SRL_DEVINL static void prefetch(const Params& p) { tma_prefetch_desc(&p.dhm); tma_prefetch_desc(&p.a3m); }
  // split mode: the ones slice keeps B lo = 0 (zero-initialised once, never loaded), so only dh hi/lo . ones contribute
  SRL_DEVINL static void issue_split(const Params& p, int, int ty, int kb, uint8_t* st, int a_bytes, int half, uint64_t* bar) {
    const int hw = ty >> 2, j0 = (ty & 3) * 128;
    mbar_arrive_expect_tx(bar, (hw < 49 ? 6 : 4) * 64 * 128);
    tma_load_2d(st, &p.dhm, bar, j0, kb * 64);
    tma_load_2d(st + KROWS * 128, &p.dhm, bar, j0 + 64, kb * 64);
    tma_load_2d(st + half, &p.dhm_lo, bar, j0, kb * 64);
    tma_load_2d(st + half + KROWS * 128, &p.dhm_lo, bar, j0 + 64, kb * 64);
    if (hw < 49) {
      tma_load_2d(st + a_bytes, &p.a3m, bar, hw * 64, kb * 64);
      tma_load_2d(st + half + a_bytes, &p.a3m_lo, bar, hw * 64, kb * 64);
    }
  }
  template <int SPLIT>
  SRL_DEVINL static void epilogue16(const Params& p, int tm, int ty, int row, int c0, float (&v)[16]) { epilogue16(p, tm, ty, row, c0, v); }
  SRL_DEVINL static bool zero_cta(int) { return true; }
  SRL_DEVINL static int num_kblocks(const Params& p, int, int) { return (p.M + 63) >> 6; }
  SRL_DEVINL static void init_smem(const Params&, int, int ty, uint8_t* stage, int tid) {
    if ((ty >> 2) == 49) fill_ones(stage + 2 * KROWS * 128, KROWS * 128, tid);
  }
  SRL_DEVINL static void issue(const Params& p, int, int ty, int kb, uint8_t* sA, uint8_t* sB, uint64_t* bar) {
    const int hw = ty >> 2, j0 = (ty & 3) * 128;
    mbar_arrive_expect_tx(bar, (hw < 49 ? 3 : 2) * 64 * 128);
    tma_load_2d(sA, &p.dhm, bar, j0, kb * 64);
    tma_load_2d(sA + KROWS * 128, &p.dhm, bar, j0 + 64, kb * 64);
    if (hw < 49) tma_load_2d(sB, &p.a3m, bar, hw * 64, kb * 64);
  }
  SRL_DEVINL static void epilogue16(const Params& p, int, int ty, int row, int c0, float (&v)[16]) {
    const int j = (ty & 3) * 128 + row, hw = ty >> 2;
    if (hw < 49) {
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) p.dw[(size_t)j * 3136 + (c0 + jj) * 49 + hw] = v[jj];
    } else if (c0 == 0) {
      p.db[j] = v[0];
    }
  }
};

// The fc weight gradient in fc.weight's own column order (bf16 mode): B operand = a3t [frames][64*49] (a3 transposed, encoder.cu), one CTA =
// 128 rows j x 256 CONSECUTIVE columns -> N = 256 MMAs run at the tensor array's own rate (128 clk, section 4.1: N = 64 costs 48 clk for a quarter
// of the work), dh is re-read 13 times instead of 49, and a thread stores 64 float4 in a row.  grid = (1, 4 * 14): ty = ct*4 + jt; column tile
// ct < 13 (the last one holds 64 valid columns, the rest of its B tile is never loaded and its columns are not stored), ct == 13 = the bias slice
// (B block 0 = ones -> column 0 of the accumulator = dbfc).
struct TFcWgradN {
  static constexpr int KID = 36;
  static constexpr bool PREFETCH = false;
  static constexpr int BN = 256, STAGES = 4, KROWS = 64, NCT = 13;
  static constexpr bool A_MN = true, B_MN = true, ZERO_INIT = true;
  struct Params { SRL_TMAP dhm; SRL_TMAP a3tm; float* dw; float* db; int M; };
  SRL_DEVINL static void prefetch(const Params& p) { tma_prefetch_desc(&p.dhm); tma_prefetch_desc(&p.a3tm); }
  SRL_DEVINL static bool zero_cta(int ty) { return (ty >> 2) == NCT; }          // only the bias slice needs defined B tiles everywhere
  SRL_DEVINL static int num_kblocks(const Params& p, int, int) { return (p.M + 63) >> 6; }
  SRL_DEVINL static void init_smem(const Params&, int, int ty, uint8_t* stage, int tid) {
    if ((ty >> 2) == NCT) fill_ones(stage + 2 * KROWS * 128, KROWS * 128, tid);
  }
  SRL_DEVINL static void issue(const Params& p, int, int ty, int kb, uint8_t* sA, uint8_t* sB, uint64_t* bar) {
    const int ct = ty >> 2, j0 = (ty & 3) * 128;
    const int nb = ct < NCT ? (ct == NCT - 1 ? 1 : 4) : 0;                       // 64-column blocks of a3t this tile owns (3136 = 12 * 256 + 64)
    mbar_arrive_expect_tx(bar, (2 + nb) * 64 * 128);
    tma_load_2d(sA, &p.dhm, bar, j0, kb * 64);
    tma_load_2d(sA + KROWS * 128, &p.dhm, bar, j0 + 64, kb * 64);
    for (int q = 0; q < nb; ++q) tma_load_2d(sB + q * KROWS * 128, &p.a3tm, bar, ct * 256 + q * 64, kb * 64);
  }
  SRL_DEVINL static void epilogue16(const Params& p, int, int ty, int row, int c0, float (&v)[16]) {
    const int j = (ty & 3) * 128 + row, ct = ty >> 2, col = ct * 256 + c0;
    if (ct < NCT) {
      if (col < 3136) {
        float4* d = reinterpret_cast<float4*>(p.dw + (size_t)j * 3136 + col);
#pragma unroll
        for (int q = 0; q < 4; ++q) d[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
      }
    } else if (c0 == 0) {
      p.db[j] = v[0];
    }
  }
  // bf16 mode: the 128 x 256 fp32 tile (128 KB, in the stage ring) leaves as 16-byte pieces, consecutive threads on consecutive pieces
  // of a dW row: a warp stores 512 contiguous bytes, where a row per thread touched 32 rows 12,544 bytes apart per store.  The last
  // column tile holds 64 valid columns (16 pieces per row); the bias slice stores column 0 as db.
  static constexpr int TILE_ROWB = 4 * BN + 32;
  SRL_DEVINL static void epilogue_tile(const Params& p, int, int ty, int t, const uint8_t* img, const uint4 (&)[1][2]) {
    const int j0 = (ty & 3) * 128, ct = ty >> 2;
    if (ct == NCT) {
      if (t < 128) p.db[j0 + t] = *reinterpret_cast<const float*>(img + t * TILE_ROWB);
      return;
    }
    float* dw = p.dw + (size_t)j0 * 3136 + ct * 256;
    const int lg = ct == NCT - 1 ? 4 : 6;                         // log2 of the valid 16-byte pieces per row
#pragma unroll 8
    for (int e = t; e < 128 << lg; e += 256) {
      const int q = e >> lg, k = e & ((1 << lg) - 1);
      *reinterpret_cast<float4*>(dw + (size_t)q * 3136 + k * 4) = *reinterpret_cast<const float4*>(img + q * TILE_ROWB + k * 16);
    }
  }
};

}  // namespace srl
