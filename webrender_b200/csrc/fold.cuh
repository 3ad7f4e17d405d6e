// fold.cuh — a run of plain solid premultiplied-over layers as per-channel lookup tables.
//
// In a simple solid batch (BatchInfo::simple) every layer maps each 8-bit channel of a pixel through a
// function of that channel alone:  d' = min(255, ((d * (255 - a) + 255) >> 8) + s)  (wr_premult_over_pair).
// A run of such layers is therefore, per channel, a map u8 -> u8: 4 x 256 entries, built by blending the
// 256 possible inputs through the run once.  Where every command of the batch covers a whole 128x8 tile
// (the tile lies inside the common cover, BatchInfo::cx0..cy1), the tile's result is one table lookup per
// channel — bit for bit what blending the layers in order gives, for valid and over-range colours alike.
//
// Table layout: entry [ch * 256 + v], ch in pixel byte order (B, G, R, A).  The batch's command list is
// cut into up to WR_FOLD_CTAS x WR_FOLD_SEGS contiguous segments, each folded over the 256 inputs on its own
// (one warp each on the device) and the segment tables composed in batch order.
#pragma once
#include "blend.cuh"
#include "cmd.cuh"
#include "wrcu_internal.h"

#define WR_FOLD_SEGS 32  // segments per CTA of wr_fold_solid (a warp each)
#define WR_FOLD_CTAS 8   // CTAs of wr_fold_solid
#define WR_FOLD_ENTRIES (4 * 256)
// Device memory per batch: the tables, then the partial tables of the fold's CTAs.
#define WR_FOLD_SLOT ((1 + WR_FOLD_CTAS) * WR_FOLD_ENTRIES)

// Blend constants of a solid command for wr_fast_blend8: (255 - A, 255 + 256 * (B | R << 16),
// 255 + 256 * (G | A << 16), 0).
WRD uint4 wr_solid_consts(const CmdHot& c) {
  const uint32_t srb = (uint32_t)c.col[0] | ((uint32_t)c.col[2] << 16);  // B | R<<16
  const uint32_t sga = (uint32_t)c.col[1] | ((uint32_t)c.col[3] << 16);  // G | A<<16
  return make_uint4(255u - c.col[3], 0x00FF00FFu + (srb << 8), 0x00FF00FFu + (sga << 8), 0u);
}

// Tiles (in tile units, half-open) of the batch's tile grid — the bounding box clamped to the target, as
// wr_raster_solid_premult walks it — that lie wholly inside the common cover.  Empty: x1 <= x0 or y1 <= y0.
WRD int4 wr_cover_tiles(const BatchInfo& bi, const TargetDev& t) {
  const int bx0 = max(bi.bx0, 0) / WRCU_TILE_W, by0 = max(bi.by0, 0) / WRCU_TILE_H;
  const int bx1 = (min(bi.bx1, t.w) + WRCU_TILE_W - 1) / WRCU_TILE_W;
  const int by1 = (min(bi.by1, t.h) + WRCU_TILE_H - 1) / WRCU_TILE_H;
  const int cx0 = (max(bi.cx0, 0) + WRCU_TILE_W - 1) / WRCU_TILE_W, cy0 = (max(bi.cy0, 0) + WRCU_TILE_H - 1) / WRCU_TILE_H;
  const int cx1 = max(bi.cx1, 0) / WRCU_TILE_W, cy1 = max(bi.cy1, 0) / WRCU_TILE_H;
  return make_int4(max(bx0, cx0), max(by0, cy0), min(bx1, cx1), min(by1, cy1));
}

// Segment `s` of `nseg` of a list of n commands: [*s0, *s1).
WRD int wr_fold_nseg(int n) { return min(n, WR_FOLD_CTAS * WR_FOLD_SEGS); }
WRD void wr_fold_segment(int n, int nseg, int s, int* s0, int* s1) {
  *s0 = (int)((long long)n * s / nseg);
  *s1 = (int)((long long)n * (s + 1) / nseg);
}

// One lane's slice of a table: the inputs v0 .. v0+7 of all four channels, as the (B,R) / (G,A) pairs
// wr_fast_blend8 works on.
WRD void wr_fold_init(uint32_t* rb, uint32_t* ga, int v0) {
#pragma unroll
  for (int p = 0; p < 8; p++) rb[p] = ga[p] = (uint32_t)(v0 + p) * 0x00010001u;
}
WRD void wr_fold_store(const uint32_t* rb, const uint32_t* ga, int v0, uint8_t* tab) {
#pragma unroll
  for (int p = 0; p < 8; p++) {
    tab[0 * 256 + v0 + p] = (uint8_t)rb[p];
    tab[1 * 256 + v0 + p] = (uint8_t)ga[p];
    tab[2 * 256 + v0 + p] = (uint8_t)(rb[p] >> 16);
    tab[3 * 256 + v0 + p] = (uint8_t)(ga[p] >> 16);
  }
}

// Entry e of the composition of nseg segment tables (segs[s * WR_FOLD_ENTRIES + ...], applied in order).
WRD uint8_t wr_fold_compose(const uint8_t* segs, int nseg, int e) {
  const int base = e & ~255;
  int x = e & 255;
  for (int s = 0; s < nseg; s++) x = segs[s * WR_FOLD_ENTRIES + base + x];
  return (uint8_t)x;
}

// A pixel through the tables.
WRD uint32_t wr_fold_px(const uint8_t* lut, uint32_t p) {
  return (uint32_t)lut[p & 255] | ((uint32_t)lut[256 + ((p >> 8) & 255)] << 8) |
         ((uint32_t)lut[512 + ((p >> 16) & 255)] << 16) | ((uint32_t)lut[768 + (p >> 24)] << 24);
}

#ifdef WRCU_HOSTEMU
// The device fold (wr_fold_solid) step by step on the host: every segment, every lane's slice, then the
// composition (in one pass: the device's per-CTA then across-CTA composition gives the same tables, as
// composition is associative).  Folds the commands the tile kernel keeps (x1 > x0).
static void wr_fold_host(const CmdHot* hot, int n, bool premul_valid, uint8_t* out) {
  std::vector<uint8_t> segs((size_t)WR_FOLD_CTAS * WR_FOLD_SEGS * WR_FOLD_ENTRIES);
  const int nseg = wr_fold_nseg(n);
  for (int s = 0; s < nseg; s++) {
    int s0, s1;
    wr_fold_segment(n, nseg, s, &s0, &s1);
    for (int lane = 0; lane < 32; lane++) {
      uint32_t rb[8], ga[8];
      wr_fold_init(rb, ga, lane * 8);
      for (int i = s0; i < s1; i++) {
        if (hot[i].x1 <= hot[i].x0) continue;
        const uint4 k = wr_solid_consts(hot[i]);
        if (premul_valid) wr_fast_blend8<true>(rb, ga, k.x, k.y, k.z);
        else wr_fast_blend8<false>(rb, ga, k.x, k.y, k.z);
      }
      wr_fold_store(rb, ga, lane * 8, segs.data() + (size_t)s * WR_FOLD_ENTRIES);
    }
  }
  for (int e = 0; e < WR_FOLD_ENTRIES; e++) out[e] = wr_fold_compose(segs.data(), nseg, e);
}
#endif
