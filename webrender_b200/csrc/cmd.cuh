// cmd.cuh — DrawCmd records: the output of the per-instance "setup" kernels
// (the reference's vertex stage + draw_quad set-up, swgl/src/rasterize.h:
// 1549-1632) and the input of the tile raster kernels.
//
// A command is split into a 32-byte HOT part that every tile CTA streams
// through shared memory (coverage rect, flags, z, packed colour) and a COLD
// part that only the CTAs actually covered by the instance read from L2
// (AA ramps, clip-mask placement, interpolation frame, sampler parameters).
#pragma once
#include <stdint.h>
#include "wrcu_internal.h"

enum : uint32_t {
  CMD_MASK = 1u << 1,       // SWGL_CLIP_FLAG_MASK   (blend.h:345)
  CMD_AA = 1u << 2,         // SWGL_CLIP_FLAG_AA
  CMD_TEXTURED = 1u << 3,   // fragment samples sColor0
  CMD_OUT_RRRR = 1u << 4,   // QF_IS_MASK: output_color.rrrr
  CMD_SUBPIXEL_TEXT = 1u << 8, // swgl_blendSubpixelText override
  CMD_DROP_SHADOW = 1u << 7, // swgl_blendDropShadow override; colour in CmdCold.i[0..1]
  CMD_CONST_COLOR = 1u << 6, // fragment output is the constant colour in CmdHot.col
  CMD_GENERAL = 1u << 9,    // screen edges not axis-aligned: per-row spans from the edge walk (GenQuad)
  CMD_CLIP_DIST = 1u << 10,  // gl_ClipDistance in interpolants 2..5 bounds every span (rasterize.h:566-596)
  CMD_COPY = 1u << 11,      // composite: an opaque / premultiplied-over 1:1 rectangle copy, drawn by wr_composite_copy when
                            // the batch allows it (BatchInfo::all_copy)
  CMD_RUNS = 1u << 12,      // has failing-sample bitmaps (CmdCold::fail_off): its depth runs are reproduced
  CMD_SPAN_SOLID = 1u << 5, // span body is drawn by swgl_commitSolid* (mask folded into colour before AA)
  CMD_ORDERED = 1u << 14,   // text: set by wr_raster_glyphs on a command it leaves to the ordered tile kernel (one it cannot draw, or
                            // that overlaps an earlier such command); the tile kernel then draws only these
  CMD_DONE = 1u << 15,      // text: drawn by wr_raster_glyphs (set after its pixels, release semantics)
  CMD_PERSP = 1u << 13,     // w differs between the vertices: draw_perspective (rasterize.h:1064-1545) — a clipped convex
                            // polygon (PerspPoly in the row-table pool, CmdCold::row_off), per-row spans from its edge walk,
                            // z/w and the interpolants (scaled by 1/w) stepped per sample; always set together with CMD_GENERAL
};

struct __align__(16) CmdHot {
  short x0, y0, x1, y1;  // half-open pixel rect; empty rect == skipped instance
  uint32_t flags;
  uint32_t z;            // 24-bit depth of the quad (rasterize.h:1587-1594)
  uint16_t col[4];       // B,G,R,A 16-bit lanes (round_pixel of v_color)
  short aa_left_end;     // leftAA.end   (rasterize.h:546)
  short aa_right_start;  // rightAA.start
  uint32_t cold;         // index of the CmdCold record
};
static_assert(sizeof(CmdHot) == 32, "CmdHot must be 32 bytes");

#define WR_NI 6  // interpolated floats per vertex (cs_clip_box_shadow: vLocalPos + vUv)

struct __align__(16) CmdCold {
  // AA coverage ramps: dist = start + x*slope per edge (rasterize.h:511-519)
  float aa_l0, aa_ls, aa_r0, aa_rs;
  // clip mask: texel for fb pixel (x,y) = mask[(y-cmy)*pitch + (x-cmx)]
  const uint8_t* mask_ptr;
  int mask_pitch;
  short cmx, cmy;
  // Interpolation frame of the (screen-axis-aligned) quad: left/right edge x,
  // top y, 1/height, and interpolants at the four edge end points.
  float xl, xr, yt, yscale;
  float i_lt[WR_NI], i_lb[WR_NI], i_rt[WR_NI], i_rb[WR_NI];
  // kind-specific
  float f[8];   // e.g. uv sample bounds
  int32_t i[4];
  float g[40];  // large kind-specific block (rounded-rect clip geometry, ...)
  // CMD_GENERAL: the quad's screen vertices (interpolants per vertex are then in
  // i_lt, i_lb, i_rt, i_rb = vertices 0..3), its clip rect, and the edge walk of
  // draw_quad_spans (rasterize.h:783-1054) recorded as events: from row `row`
  // on, the l-chain edge is l0->l1 (initialised at row lrow) and the r-chain edge
  // r0->r1 (initialised at row rrow).
  float gpx[4], gpy[4];
  float gclip[4];
  struct { short row, lrow, rrow; uint8_t l0, l1, r0, r1; } gev[6];
  int gn_ev, gflipped, gaa_mask;
  // Row table (axis-aligned quads of >= WR_ROW_TAB_MIN rows with interpolants): the edge
  // interpolants of every row, 2*row_n floats per row (left, right per interpolant) from float
  // offset row_off of RasterArgs.row_tab; -1 = none, wr_row_interp walks the sums itself.
  int row_off;
  int row_n;
  // Depth runs: word offset of this command's failing-sample bitmaps in the batch's pool (-1 = none):
  // per row of the hot rect 1 + fail_w words — [0] the number of failing samples inside the row's span,
  // then bit i of the bitmap = sample hot.x0 + i fails the depth test (or lies outside the row's span).
  int fail_off, fail_w, rpad;
};

// CMD_PERSP: the polygon draw_perspective hands to draw_perspective_spans — up to 4 + 6 vertices after
// clip_side (rasterize.h:1289-1420), in screen space with w = 1/clip.w, the vertex interpolants, the
// clipped AA edge mask, the clip rect and the edge walk recorded as events (as CmdCold::gev).
#define WR_PP_MAXV 10
#define WR_PP_MAXEV 14
struct PerspPoly {
  int nump, n_ev, flipped, aa_mask;
  float clip[4];
  float px[WR_PP_MAXV], py[WR_PP_MAXV], pz[WR_PP_MAXV], pw[WR_PP_MAXV];
  float interp[WR_PP_MAXV][WR_NI];
  struct { short row, lrow, rrow; uint8_t l0, l1, r0, r1; } ev[WR_PP_MAXEV];
};
#define WR_PP_FLOATS ((int)((sizeof(PerspPoly) + 15) / 16 * 4))

// Per-(command,row) state of a perspective polygon (wr_persp_row): the left / right Edge of
// draw_perspective_spans at this row — (x, z, w) and which polygon edge each is on — and the span's
// z/w start and step (rasterize.h:1236-1252).
struct PerspRow {
  const PerspPoly* poly;
  float lx, lz, lw, rx, rz, rw;
  float step_scale, x0f;   // 1 / (right.x - left.x), span.start + 0.5 - left.x
  float zw0[2], step_zw[2];
  int lv0, lv1, lrow, rv0, rv1, rrow;
};

// Per-(command,row) state of a general quad, computed by wr_general_row.
struct GenRow {
  float lx, rx;                      // left.x / right.x at this row
  float aa_l0, aa_ls, aa_r0, aa_rs;  // AA ramps of this row
  int lv0, lv1, lrow, rv0, rv1, rrow;  // (final) left/right edge: vertices and init row
};

// Per-batch info written by the setup kernel.
struct BatchInfo {
  int bx0, by0, bx1, by1;  // bounding box of all commands
  int unsupported;         // instances the setup kernel had to reject
  int simple;              // 1 while every command is a plain solid quad (no mask/AA/texture, lanes<=255)
  int premul_valid;        // 1 while every command's colour lanes are <= its alpha lane
  int tile_counter;        // dynamic tile scheduler of the generic raster kernel
  int n_ordered;           // text: commands wr_raster_glyphs left to the tile kernel (CMD_ORDERED)
  int all_copy;            // composite: 1 while no two commands of the batch overlap: CMD_COPY commands go to wr_composite_copy
  int glyph_ticket;        // text: next glyph wr_raster_glyphs hands to a warp
  int n_noncopy;           // composite: drawn commands that are not CMD_COPY (0: the tile kernel has nothing to do)
  int cx0, cy0, cx1, cy1;  // common cover: the rect every drawn command contains (max of x0/y0, min of x1/y1);
                           // reduced over the commands of simple batches only (see fold.cuh)
  int fold_ticket;         // wr_fold_solid: CTAs that have written their partial tables (the last one composes them)
};
#define WR_ROW_TAB_MIN 4   // glyph rows (~12) too: the per-(command,row,tile) walk was a third of the text kernel
