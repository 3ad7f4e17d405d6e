// raster.cuh — tile-resident raster kernels.
//
// The reference draws a batch instance by instance: for each instance every
// row, every span, every 4-pixel chunk is read-modify-written in the
// framebuffer (swgl/src/rasterize.h:783-1054, blend.h:416).  On a GPU that
// shape would serialise on memory: N overlapping instances = N passes over
// the same bytes.  Here the loop nest is inverted: one CTA owns a 128x8-pixel
// tile of the render target, keeps its pixels in registers (4 pixels/thread),
// streams the batch's command list through shared memory IN BATCH ORDER (order
// matters for blending), applies fragment + blend stage per pixel, and writes
// the tile once.  DRAM sees each target byte at most once in and once out per
// batch, however many layers the batch stacks.
//
// Thread mapping: 256 threads = 8 warps; warp w owns tile row w (128 px =
// 512 B contiguous for RGBA8 → one fully coalesced 16-byte vector access per
// lane); lane l owns pixels [4l, 4l+4).
#pragma once
#include "blend.cuh"
#include "cmd.cuh"
#include "sample.cuh"
#include "texspan.cuh"
#include "wrcu_internal.h"
#include "repeat_add.cuh"
#include "fold.cuh"

struct RasterArgs {
  TargetDev tgt;
  const CmdHot* hot;
  const CmdCold* cold;
  const BatchInfo* info;
  int n;
  int blend;        // wrcu_blend
  int depth_mode;   // wrcu_depth
  Px blend_color;   // glBlendColor in lane order
  TexView color0;   // sColor0
  TexView color1;   // sColor1 (brush_mix_blend source, YUV chroma plane)
  TexView color2;   // sColor2 (third YUV plane)
  int fast_eligible;  // host-side part of the solid-premult fast-path test
  const float4* gbuf_f;  // gpu_buffer_f (gradient LUTs)
  int n_gbuf_f;
  const float4* gpu_cache;  // component-transfer tables
  int n_gpu_cache;
  const GenRow* gen;  // per-thread row state of the current CMD_GENERAL command
  const PerspRow* persp;  // ... of the current CMD_PERSP command (nullptr otherwise): varyings are w * interp_perspective
  const uint32_t* tile_mask;  // bitmask bins (see SetupArgs), nullptr = scan every command
  const uint32_t* wide_mask;
  const uint32_t* tile_any;  // see SetupArgs
  int any_words;
  uint32_t* tile_ord;    // glyph-major text: bit t = an ordered command (CMD_ORDERED) touches tile t (binned batches)
  int glyph_major;       // the batch went through wr_raster_glyphs first: the tile kernel draws only CMD_ORDERED commands
  int lane_rows;         // the lanes of a warp hold different (command,row)s: no warp-cooperative walks in the row set-up
  int strip_seg;         // > 0: strip mode of the tile kernel — work items are runs of this many adjacent tiles of a tile row
  int bin_words, bin_tiles_x;
  const float* row_tab;  // row tables written by the setup kernel (CmdCold::row_off)
  // Depth runs (rasterize.h:601-657): with depth testing on, the reference draws each maximal run of
  // passing samples of a span as a span of its own.  rl != nullptr while a run AFTER the first of a
  // (command,row) is being shaded: the four chunk lanes of every interpolant (rl[lane * WR_NI + i]) as
  // the walk over the earlier runs left them.  fail_pool: per (command,row) bitmaps of failing samples
  // written by wr_depth_fail_rows (CmdCold::fail_off).
  const float* rl;
  const uint32_t* fail_pool;
  const void* tmaps;     // device table of CUtensorMap records, indexed by TexView::tmap_id
  int copy_eligible;     // composite: a copy-class batch (BatchInfo::all_copy) is drawn by wr_composite_copy
  int tmap_acquire;      // tensor-map table slots have been reused: acquire each map before use (tma.cuh)
  int pdl_early;         // programmatic dependent launch: this kernel may read its commands (written by the set-up
                         // launch, which finished earlier) before the kernel ahead of it in the stream has completed
  uint8_t* fold;         // solid batches: the batch's 4 x 256 lookup tables (fold.cuh), written by wr_fold_solid
                         // ahead of wr_raster_solid_premult; nullptr when no fold was launched
};

#define CHUNK_CMDS 256
// Programmatic dependent launch (griddepcontrol): raster kernels of a submission are launched with
// programmaticStreamSerialization, each lets its successor start at once and itself waits for its predecessor
// only where it first touches pixels — the command scan of batch k+1 overlaps the pixels of batch k.  Both
// instructions do nothing in a kernel launched the ordinary way.
#ifdef WRCU_HOSTEMU
static inline void wr_pdl_launch_dependents() {}
static inline void wr_pdl_wait() {}
#else
__device__ __forceinline__ void wr_pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void wr_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
#endif

// AA weight of pixel x for the current command (DO_AA, blend.h:433-445, with
// the span set-up of aa_span, rasterize.h:546-557).  Chunks of 4 start at the
// span start c.x0.
WRD int wr_aa_weight(const RasterArgs& a, const CmdHot& c, const CmdCold& k, int x) {
  int j = (x - c.x0) & 3;
  int xc = x - j;
  int opaque = max((int)c.aa_right_start - (int)c.aa_left_end - 3, 0);
  int off = xc - c.aa_left_end;
  if (off >= 0 && off < opaque) return 256;
  const bool gen = (c.flags & CMD_GENERAL) != 0;
  const float l0 = gen ? a.gen->aa_l0 : k.aa_l0, ls = gen ? a.gen->aa_ls : k.aa_ls;
  const float r0 = gen ? a.gen->aa_r0 : k.aa_r0, rs = gen ? a.gen->aa_rs : k.aa_rs;
  float offs = (float)(c.aa_left_end + j);
  float left = __fadd_rn(l0, __fmul_rn(offs, ls));
  float right = __fadd_rn(r0, __fmul_rn(offs, rs));
  float fo = (float)off;
  float dist = wr_clamp(wr_min(__fadd_rn(left, __fmul_rn(ls, fo)),
                               __fadd_rn(right, __fmul_rn(rs, fo))),
                        0.0f, 256.0f);
  return wr_round_pixel(dist, 1.0f);
}

// Interpolants of a screen-axis-aligned quad.  The reference walks the left and
// right edges row by row, adding the per-row slope each time (Edge::nextRow,
// rasterize.h:880-884), then derives the span's start value and per-pixel step
// (rasterize.h:1003-1017).  wr_row_interp reproduces that running sum exactly:
// it starts from the Edge constructor's value at the first row and adds the
// slope (y - y0) times — warp-uniform work, once per (command,row).
// One edge of the walk at row y: Edge(y_init, p0, p1, interp0, interp1) followed by
// (y - init row) nextRow() steps (rasterize.h:851-884).
WRD void wr_gen_edge_x(const CmdCold& k, int v0, int v1, int init_row, int y, float* x, float* slope) {
  float ys = (float)init_row + 0.5f;
  float yScale = 1.0f / wr_max(k.gpy[v1] - k.gpy[v0], 1.0f / 256);
  float xs = (k.gpx[v1] - k.gpx[v0]) * yScale;
  float xx = k.gpx[v0] + (ys - k.gpy[v0]) * xs;
  xx = wr_repeat_add(xx, xs, y - init_row);
  *x = xx;
  *slope = xs;
}
WRD const float* wr_gen_vertex_interp(const CmdCold& k, int v) {
  return v == 0 ? k.i_lt : v == 1 ? k.i_lb : v == 2 ? k.i_rt : k.i_rb;
}

// aa_span + the edge state of draw_quad_spans for row y of a general quad.
// Fills g and the row's span in `out` (a copy of the hot record); false = empty.
WRD_SHARED bool wr_general_row(const CmdCold& k, const CmdHot& c, int y, GenRow& g, CmdHot& out) {
  int e = 0;
  for (int i = 1; i < k.gn_ev; i++)
    if (k.gev[i].row <= y) e = i;
  const int l0 = k.gev[e].l0, l1 = k.gev[e].l1, r0 = k.gev[e].r0, r1 = k.gev[e].r1;
  float lcx, lcs, rcx, rcs;  // l-chain / r-chain edge x and slope
  wr_gen_edge_x(k, l0, l1, k.gev[e].lrow, y, &lcx, &lcs);
  wr_gen_edge_x(k, r0, r1, k.gev[e].rrow, y, &rcx, &rcs);
  // edgeMask: Edge(.., edgeIndex = l1i) for the l-chain, r0i for the r-chain
  int lcm = (k.gaa_mask >> l1) & 1, rcm = (k.gaa_mask >> r0) & 1;
  float leftx, lefts, rightx, rights;
  int lmask, rmask;
  if (k.gflipped) {
    leftx = rcx; lefts = rcs; lmask = rcm; rightx = lcx; rights = lcs; rmask = lcm;
    g.lv0 = r0; g.lv1 = r1; g.lrow = k.gev[e].rrow; g.rv0 = l0; g.rv1 = l1; g.rrow = k.gev[e].lrow;
  } else {
    leftx = lcx; lefts = lcs; lmask = lcm; rightx = rcx; rights = rcs; rmask = rcm;
    g.lv0 = l0; g.lv1 = l1; g.lrow = k.gev[e].lrow; g.rv0 = r0; g.rv1 = r1; g.rrow = k.gev[e].rrow;
  }
  g.lx = leftx;
  g.rx = rightx;
  const float cx0 = k.gclip[0], cx1 = k.gclip[2];
  float cs0 = wr_clamp(wr_min(wr_min(k.gpx[l0], k.gpx[l1]), wr_min(k.gpx[r0], k.gpx[r1])), cx0, cx1);
  float cs1 = wr_clamp(wr_max(wr_max(k.gpx[l0], k.gpx[l1]), wr_max(k.gpx[r0], k.gpx[r1])), cx0, cx1);
  int sx0, sx1;
  out = c;
  if (!(c.flags & CMD_AA)) {
    sx0 = (int)floorf(wr_clamp(leftx, cs0, cs1) + 0.5f);
    sx1 = (int)floorf(wr_clamp(rightx, cs0, cs1) + 0.5f);
  } else {
    int la0, la1, ra0, ra1;
    if (lmask) {
      float rad = 0.5f * fabsf(lefts);
      la0 = (int)floorf(wr_clamp(leftx - rad, cs0, cs1));
      la1 = (int)ceilf(wr_clamp(leftx + rad, cs0, cs1));
      float dx = (-1.0f * 256.0f) * (1.0f / sqrtf(1.0f + lefts * lefts));
      g.aa_l0 = 128.0f + dx * (leftx - 0.5f);
      g.aa_ls = -dx;
    } else {
      la0 = la1 = (int)floorf(wr_clamp(leftx, cs0, cs1) + 0.5f);
      g.aa_l0 = 256.0f;
      g.aa_ls = 0.0f;
    }
    if (rmask) {
      float rad = 0.5f * fabsf(rights);
      ra0 = (int)floorf(wr_clamp(rightx - rad, cs0, cs1));
      ra1 = (int)ceilf(wr_clamp(rightx + rad, cs0, cs1));
      float dx = (1.0f * 256.0f) * (1.0f / sqrtf(1.0f + rights * rights));
      g.aa_r0 = 128.0f + dx * (rightx - 0.5f);
      g.aa_rs = -dx;
    } else {
      ra0 = ra1 = (int)floorf(wr_clamp(rightx, cs0, cs1) + 0.5f);
      g.aa_r0 = 256.0f;
      g.aa_rs = 0.0f;
    }
    out.aa_left_end = (short)la1;
    out.aa_right_start = (short)ra0;
    sx0 = la0;
    sx1 = ra1;
  }
  out.x0 = (short)sx0;
  out.x1 = (short)sx1;
  return sx1 > sx0;
}

// ---- perspective (draw_perspective_spans, rasterize.h:1064-1283) -------------------------------------
#ifdef WRCU_HOSTEMU
#define WRD_NOINLINE_R static
#else
#define WRD_NOINLINE_R __device__ __noinline__
#endif
// One Edge of the perspective walk at row y: Edge(y_init, p0, p1, ..) + (y - init row) nextRow() steps.
WRD void wr_persp_edge(const PerspPoly& P, int v0, int v1, int init_row, int y, float* x, float* z, float* w, float* xslope) {
  const float ys = (float)init_row + 0.5f;
  const float yScale = 1.0f / wr_max(P.py[v1] - P.py[v0], 1.0f / 256);
  const float dy = ys - P.py[v0];
  const float xs = (P.px[v1] - P.px[v0]) * yScale, zs = (P.pz[v1] - P.pz[v0]) * yScale, ws = (P.pw[v1] - P.pw[v0]) * yScale;
  *x = wr_repeat_add(P.px[v0] + dy * xs, xs, y - init_row);
  *z = wr_repeat_add(P.pz[v0] + dy * zs, zs, y - init_row);
  *w = wr_repeat_add(P.pw[v0] + dy * ws, ws, y - init_row);
  *xslope = xs;
}
// The row's edges, aa_span and the z/w set-up of the span.  Fills g (AA ramps, as wr_general_row), pr and the
// row's span in `out`; false = empty.
WRD_NOINLINE_R bool wr_persp_row(const float* row_tab, const CmdCold& k, const CmdHot& c, int y, GenRow& g, PerspRow& pr, CmdHot& out) {
  const PerspPoly& P = *(const PerspPoly*)(row_tab + k.row_off);
  int e = 0;
  for (int i = 1; i < P.n_ev; i++)
    if (P.ev[i].row <= y) e = i;
  const int l0 = P.ev[e].l0, l1 = P.ev[e].l1, r0 = P.ev[e].r0, r1 = P.ev[e].r1;
  float lcx, lcz, lcw, lcs, rcx, rcz, rcw, rcs;
  wr_persp_edge(P, l0, l1, P.ev[e].lrow, y, &lcx, &lcz, &lcw, &lcs);
  wr_persp_edge(P, r0, r1, P.ev[e].rrow, y, &rcx, &rcz, &rcw, &rcs);
  const int lcm = (P.aa_mask >> l1) & 1, rcm = (P.aa_mask >> r0) & 1;
  float leftx, lefts, rightx, rights;
  int lmask, rmask;
  if (P.flipped) {
    leftx = rcx; lefts = rcs; lmask = rcm; rightx = lcx; rights = lcs; rmask = lcm;
    pr.lz = rcz; pr.lw = rcw; pr.rz = lcz; pr.rw = lcw;
    pr.lv0 = r0; pr.lv1 = r1; pr.lrow = P.ev[e].rrow; pr.rv0 = l0; pr.rv1 = l1; pr.rrow = P.ev[e].lrow;
  } else {
    leftx = lcx; lefts = lcs; lmask = lcm; rightx = rcx; rights = rcs; rmask = rcm;
    pr.lz = lcz; pr.lw = lcw; pr.rz = rcz; pr.rw = rcw;
    pr.lv0 = l0; pr.lv1 = l1; pr.lrow = P.ev[e].lrow; pr.rv0 = r0; pr.rv1 = r1; pr.rrow = P.ev[e].rrow;
  }
  pr.poly = &P;
  pr.lx = leftx;
  pr.rx = rightx;
  g.lx = leftx;
  g.rx = rightx;
  const float cx0 = P.clip[0], cx1 = P.clip[2];
  const float cs0 = wr_clamp(wr_min(wr_min(P.px[l0], P.px[l1]), wr_min(P.px[r0], P.px[r1])), cx0, cx1);
  const float cs1 = wr_clamp(wr_max(wr_max(P.px[l0], P.px[l1]), wr_max(P.px[r0], P.px[r1])), cx0, cx1);
  int sx0, sx1;
  out = c;
  if (!(c.flags & CMD_AA)) {
    sx0 = (int)floorf(wr_clamp(leftx, cs0, cs1) + 0.5f);
    sx1 = (int)floorf(wr_clamp(rightx, cs0, cs1) + 0.5f);
  } else {
    int la0, la1, ra0, ra1;
    if (lmask) {
      float rad = 0.5f * fabsf(lefts);
      la0 = (int)floorf(wr_clamp(leftx - rad, cs0, cs1));
      la1 = (int)ceilf(wr_clamp(leftx + rad, cs0, cs1));
      float dx = (-1.0f * 256.0f) * (1.0f / sqrtf(1.0f + lefts * lefts));
      g.aa_l0 = 128.0f + dx * (leftx - 0.5f);
      g.aa_ls = -dx;
    } else {
      la0 = la1 = (int)floorf(wr_clamp(leftx, cs0, cs1) + 0.5f);
      g.aa_l0 = 256.0f;
      g.aa_ls = 0.0f;
    }
    if (rmask) {
      float rad = 0.5f * fabsf(rights);
      ra0 = (int)floorf(wr_clamp(rightx - rad, cs0, cs1));
      ra1 = (int)ceilf(wr_clamp(rightx + rad, cs0, cs1));
      float dx = (1.0f * 256.0f) * (1.0f / sqrtf(1.0f + rights * rights));
      g.aa_r0 = 128.0f + dx * (rightx - 0.5f);
      g.aa_rs = -dx;
    } else {
      ra0 = ra1 = (int)floorf(wr_clamp(rightx, cs0, cs1) + 0.5f);
      g.aa_r0 = 256.0f;
      g.aa_rs = 0.0f;
    }
    out.aa_left_end = (short)la1;
    out.aa_right_start = (short)ra0;
    sx0 = la0;
    sx1 = ra1;
  }
  out.x0 = (short)sx0;
  out.x1 = (short)sx1;
  if (sx1 <= sx0) return false;
  float stepScale = 1.0f / (rightx - leftx);
  if (!isfinite(stepScale)) stepScale = 0.0f;
  pr.step_scale = stepScale;
  pr.x0f = (float)sx0 + 0.5f - leftx;
  pr.step_zw[0] = (pr.rz - pr.lz) * stepScale;
  pr.step_zw[1] = (pr.rw - pr.lw) * stepScale;
  pr.zw0[0] = pr.lz + pr.step_zw[0] * pr.x0f;
  pr.zw0[1] = pr.lw + pr.step_zw[1] * pr.x0f;
  return true;
}
// gl_FragCoord.z / .w (c = 0 / 1) of the sample `rel` pixels into the span: lane j of init_interp(zw, stepZW),
// advanced one step_perspective() per chunk (program.h:145-148).
WRD_NOINLINE_R float wr_persp_zw(const PerspRow& pr, int c, int rel) {
  float v = pr.zw0[c];
  const float st = pr.step_zw[c];
  for (int s = 0; s < (rel & 3); s++) v = __fadd_rn(v, st);
  return wr_repeat_add(v, __fmul_rn(st, 4.0f), rel >> 2);
}
// interp_perspective of the sample: lane j of init_interp(o, step) + one interp_step per chunk
// (glsl-to-cxx read_perspective_inputs / step_perspective_inputs)
WRD_NOINLINE_R float wr_persp_lane(float o, float step, int rel) {
  float v = o;
  for (int s = 0; s < (rel & 3); s++) v = __fadd_rn(v, step);
  return wr_repeat_add(v, __fmul_rn(step, 4.0f), rel >> 2);
}
// left.interp / right.interp of the walk at this row (interpolants pre-multiplied by the vertices' 1/w)
WRD_NOINLINE_R void wr_persp_edge_interp(const PerspRow& pr, int i, int y, float* li, float* ri) {
  const PerspPoly& P = *pr.poly;
  {
    const float lsc = 1.0f / wr_max(P.py[pr.lv1] - P.py[pr.lv0], 1.0f / 256);
    const float i0 = P.interp[pr.lv0][i] * P.pw[pr.lv0], i1 = P.interp[pr.lv1][i] * P.pw[pr.lv1];
    const float sl = (i1 - i0) * lsc;
    *li = wr_repeat_add(i0 + ((float)pr.lrow + 0.5f - P.py[pr.lv0]) * sl, sl, y - pr.lrow);
  }
  {
    const float rsc = 1.0f / wr_max(P.py[pr.rv1] - P.py[pr.rv0], 1.0f / 256);
    const float i0 = P.interp[pr.rv0][i] * P.pw[pr.rv0], i1 = P.interp[pr.rv1][i] * P.pw[pr.rv1];
    const float sr = (i1 - i0) * rsc;
    *ri = wr_repeat_add(i0 + ((float)pr.rrow + 0.5f - P.py[pr.rv0]) * sr, sr, y - pr.rrow);
  }
}

template <int N>
WRD void wr_row_interp_raw(const RasterArgs& a, const CmdCold& k, const CmdHot& c, int y, float* o, float* step,
                           float* li_out, float* ri_out) {
  if (c.flags & CMD_PERSP) {
    const PerspRow& pr = *a.persp;
#pragma unroll
    for (int i = 0; i < N; i++) {
      float li, ri;
      wr_persp_edge_interp(pr, i, y, &li, &ri);
      if (li_out) { li_out[i] = li; ri_out[i] = ri; }
      const float st = (ri - li) * pr.step_scale;
      step[i] = st;
      o[i] = li + st * pr.x0f;
    }
    return;
  }
  if (c.flags & CMD_GENERAL) {
    // left.interp / right.interp of the walk at this row, then the span's start
    // value and per-pixel step (rasterize.h:1003-1017)
    const GenRow& g = *a.gen;
    float stepScale = __fdiv_rn(1.0f, __fsub_rn(g.rx, g.lx));
    if (!isfinite(stepScale)) stepScale = 0.0f;
    float x0f = __fsub_rn(__fadd_rn((float)c.x0, 0.5f), g.lx);
    const float* l0i = wr_gen_vertex_interp(k, g.lv0);
    const float* l1i = wr_gen_vertex_interp(k, g.lv1);
    const float* r0i = wr_gen_vertex_interp(k, g.rv0);
    const float* r1i = wr_gen_vertex_interp(k, g.rv1);
    float lys = (float)g.lrow + 0.5f, rys = (float)g.rrow + 0.5f;
    float lsc = 1.0f / wr_max(k.gpy[g.lv1] - k.gpy[g.lv0], 1.0f / 256);
    float rsc = 1.0f / wr_max(k.gpy[g.rv1] - k.gpy[g.rv0], 1.0f / 256);
#pragma unroll
    for (int i = 0; i < N; i++) {
      float sl = (l1i[i] - l0i[i]) * lsc, sr = (r1i[i] - r0i[i]) * rsc;
      float li = l0i[i] + (lys - k.gpy[g.lv0]) * sl;
      float ri = r0i[i] + (rys - k.gpy[g.rv0]) * sr;
      li = wr_repeat_add(li, sl, y - g.lrow);
      ri = wr_repeat_add(ri, sr, y - g.rrow);
      if (li_out) { li_out[i] = li; ri_out[i] = ri; }
      float st = (ri - li) * stepScale;
      step[i] = st;
      o[i] = li + st * x0f;
    }
    return;
  }
  float y0c = (float)c.y0 + 0.5f;
  float dy = __fsub_rn(y0c, k.yt);
  float stepScale = __fdiv_rn(1.0f, __fsub_rn(k.xr, k.xl));
  if (!isfinite(stepScale)) stepScale = 0.0f;
  float x0f = __fsub_rn(__fadd_rn((float)c.x0, 0.5f), k.xl);
  int rows = y - c.y0;
  if (k.row_off >= 0 && k.row_n == N) {
    // the setup kernel already walked the edge sums of every row of this command
    const float* t = a.row_tab + k.row_off + (size_t)rows * (2 * N);
#pragma unroll
    for (int i = 0; i < N; i++) {
      float li = __ldg(t + 2 * i), ri = __ldg(t + 2 * i + 1);
      if (li_out) { li_out[i] = li; ri_out[i] = ri; }
      float st = __fmul_rn(__fsub_rn(ri, li), stepScale);
      step[i] = st;
      o[i] = __fadd_rn(li, __fmul_rn(st, x0f));
    }
    return;
  }
#ifndef WRCU_HOSTEMU
  // The 2N edge sums are independent and the whole warp is here (row_setup is
  // warp-uniform): lane l < 2N walks one of them, the results are broadcast.
  // One walk's worth of instructions instead of 2N.  (Not where lanes hold different rows:
  // RasterArgs::lane_rows, the glyph-major kernel.)
  if (!a.lane_rows) {
  const int wlane = threadIdx.x & 31;
  float walked = 0.0f;
  if (wlane < 2 * N) {
    const int i = wlane >> 1;
    const float* top = (wlane & 1) ? k.i_rt : k.i_lt;
    const float* bot = (wlane & 1) ? k.i_rb : k.i_lb;
    float sl = __fmul_rn(__fsub_rn(bot[i], top[i]), k.yscale);
    walked = wr_repeat_add(__fadd_rn(top[i], __fmul_rn(dy, sl)), sl, rows);
  }
#pragma unroll
  for (int i = 0; i < N; i++) {
    float li = __shfl_sync(0xFFFFFFFFu, walked, 2 * i);
    float ri = __shfl_sync(0xFFFFFFFFu, walked, 2 * i + 1);
    if (li_out) { li_out[i] = li; ri_out[i] = ri; }
    float st = __fmul_rn(__fsub_rn(ri, li), stepScale);
    step[i] = st;
    o[i] = __fadd_rn(li, __fmul_rn(st, x0f));
  }
  return;
  }
#endif
#pragma unroll
  for (int i = 0; i < N; i++) {
    float sl = __fmul_rn(__fsub_rn(k.i_lb[i], k.i_lt[i]), k.yscale);
    float sr = __fmul_rn(__fsub_rn(k.i_rb[i], k.i_rt[i]), k.yscale);
    float li = __fadd_rn(k.i_lt[i], __fmul_rn(dy, sl));
    float ri = __fadd_rn(k.i_rt[i], __fmul_rn(dy, sr));
    li = wr_repeat_add(li, sl, rows);
    ri = wr_repeat_add(ri, sr, rows);
    if (li_out) { li_out[i] = li; ri_out[i] = ri; }
    float st = __fmul_rn(__fsub_rn(ri, li), stepScale);
    step[i] = st;
    o[i] = __fadd_rn(li, __fmul_rn(st, x0f));
  }
}

template <int N>
WRD void wr_row_interp(const RasterArgs& a, const CmdCold& k, const CmdHot& c, int y, float* o, float* step,
                       float* li_out = nullptr, float* ri_out = nullptr) {
  wr_row_interp_raw<N>(a, k, c, y, o, step, li_out, ri_out);
  if (a.rl) {  // a later depth run of this row: lane 0 continues from the walk, not from the span equation
#pragma unroll
    for (int i = 0; i < N; i++) o[i] = a.rl[i];
  }
}

// The chunk lanes across a passing depth run of n pixels (draw_depth_span, rasterize.h:612-657): the
// `drawn` pixels a span shader committed advance them in one step (DISPATCH_DRAW_SPAN:
// step_interp_inputs(drawn), swgl_ext.h:1916-1923), every remaining chunk — a partial tail included —
// by one interp_step per run().  `is` = interp_step = 4 * step.
WRD float wr_run_advance(float v, float is, int n, int drawn) {
  if (drawn > 0) v = __fadd_rn(v, __fmul_rn(is, __fmul_rn((float)drawn, 0.25f)));
  return wr_repeat_add(v, is, (n - drawn + 3) >> 2);
}
// ... and across the failed samples up to the next run: skip(skip - pad), pad = what the partial tail
// chunk of the previous run over-advanced (rasterize.h:649-656).
WRD float wr_run_skip(float v, float is, int prev_len, int skip) {
  const int pad = (prev_len & 3) ? 4 - (prev_len & 3) : 0;
  return __fadd_rn(v, __fmul_rn(is, __fmul_rn((float)(skip - pad), 0.25f)));
}
// How a shader takes part in the depth-run walk: n = interpolants per vertex its Row is built from
// (0: the shader's source does not depend on them), drawn() = pixels of the run its span shader
// committed (from the Row that row_setup built for that run).
template <class S> struct WrRun {
  enum { n = 0 };
  WRD_MEMBER int drawn(const typename S::Row&) { return 0; }
};

// The walk itself, shared by the tile kernel and the host emulation: begin() before a run is shaded
// (sets a.rl), end() after it with the run's span-shader pixel count.
template <class S>
struct WrRunWalk {
  enum { NL = WrRun<S>::n };
  float lanes[4 * WR_NI];
  float is[WR_NI];
  bool first;
  int prev_end, prev_len;
  WRD_METHOD void reset() { first = true; prev_end = 0; prev_len = 0; }
  WRD_METHOD void begin(RasterArgs& a, const CmdCold& k, const CmdHot& cr, int y) {
    a.rl = nullptr;
    if (NL == 0) return;
    if (first) {
      // leading failed samples are skipped before init_span: the first run's interpolants come from the
      // span equation at its own start (rasterize.h:984-1017), its lanes accumulate as init_interp does
      float o[NL ? NL : 1], st[NL ? NL : 1];
      wr_row_interp<(NL ? NL : 1)>(a, k, cr, y, o, st);
#pragma unroll
      for (int i = 0; i < NL; i++) {
        is[i] = __fmul_rn(st[i], 4.0f);
        float v = o[i];
        lanes[i] = v;
        v = __fadd_rn(v, st[i]); lanes[WR_NI + i] = v;
        v = __fadd_rn(v, st[i]); lanes[2 * WR_NI + i] = v;
        v = __fadd_rn(v, st[i]); lanes[3 * WR_NI + i] = v;
      }
      return;
    }
#pragma unroll
    for (int j = 0; j < 4; j++)
#pragma unroll
      for (int i = 0; i < NL; i++) lanes[j * WR_NI + i] = wr_run_skip(lanes[j * WR_NI + i], is[i], prev_len, (int)cr.x0 - prev_end);
    a.rl = lanes;
  }
  WRD_METHOD void end(RasterArgs& a, const CmdHot& cr, int drawn) {
    const int n = (int)cr.x1 - (int)cr.x0;
#pragma unroll
    for (int j = 0; j < 4; j++)
#pragma unroll
      for (int i = 0; i < NL; i++) lanes[j * WR_NI + i] = wr_run_advance(lanes[j * WR_NI + i], is[i], n, drawn);
    first = false;
    prev_end = cr.x1;
    prev_len = n;
    a.rl = nullptr;
  }
};

// Value of interpolant lanes at pixel x of the span: lane j of chunk k.  Chunk
// offset accumulates sequentially as init_interp does (glsl.h:3083-3088), then
// the chunk advance is one multiply-add (step_interp_inputs(drawn) after a
// span body; exact for the 1:1 mappings that dominate).
template <int N>
WRD void wr_interp_at_plain(const float* o, const float* step, int rel, float* out) {  // setup kernels: no depth runs
  int j = rel & 3;
  float kf = (float)(rel >> 2);
#pragma unroll
  for (int i = 0; i < N; i++) {
    float v = o[i];
    for (int s = 0; s < j; s++) v = __fadd_rn(v, step[i]);
    v = __fadd_rn(v, __fmul_rn(__fmul_rn(step[i], 4.0f), kf));
    out[i] = v;
  }
}
template <int N>
WRD void wr_interp_at(const RasterArgs& a, const float* o, const float* step, int rel, float* out) {
  if (a.persp) {  // varying = w * interp_perspective, w = 1 / gl_FragCoord.w of the sample
    const float w = 1.0f / wr_persp_zw(*a.persp, 1, rel);
#pragma unroll
    for (int i = 0; i < N; i++) out[i] = wr_persp_lane(o[i], step[i], rel) * w;
    return;
  }
  int j = rel & 3;
  float kf = (float)(rel >> 2);
#pragma unroll
  for (int i = 0; i < N; i++) {
    float v = o[i];
    if (a.rl) v = a.rl[j * WR_NI + i];                              // a later depth run: the lanes as the walk left them
    else for (int s = 0; s < j; s++) v = __fadd_rn(v, step[i]);    // init_interp lanes first,
    v = __fadd_rn(v, __fmul_rn(__fmul_rn(step[i], 4.0f), kf));     // then interp_step * chunks
    out[i] = v;
  }
}

// clip_distance_range (rasterize.h:566-596) for row y of a command whose vertex stage wrote
// gl_ClipDistance (interpolants 2..5): narrows the row's span [c.x0, c.x1).  Warp-uniform.
WRD_SHARED bool wr_clip_dist_row(const RasterArgs& a, const CmdCold& k, CmdHot& c, int y) {
  float o[6], st[6], li[6], ri[6];
  wr_row_interp<6>(a, k, c, y, o, st, li, ri);
  const bool gen = (c.flags & CMD_GENERAL) != 0;
  const float lx = gen ? a.gen->lx : k.xl, rx = gen ? a.gen->rx : k.xr;
  float start_m = -1.0e30f, end_m = 1.0e30f;
#pragma unroll
  for (int i = 2; i < 6; i++) {
    const float lc = li[i], rc = ri[i];
    const float clipStep = (rc - lc) / (rx - lx);
    const float clipDist = wr_clamp(lx - lc * (1.0f / clipStep), 0.0f, 1.0e6f);
    const float s_ = clipStep > 0.0f ? clipDist : (lc < 0.0f ? 1.0e6f : 0.0f);
    const float e_ = clipStep < 0.0f ? clipDist : (rc >= 0.0f ? 1.0e6f : 0.0f);
    start_m = wr_max(start_m, s_);
    end_m = wr_min(end_m, e_);
  }
  const int cs = (int)floorf(start_m + 0.5f), ce = (int)floorf(end_m + 0.5f);
  const int x0 = max((int)c.x0, cs), x1 = min((int)c.x1, ce);
  if (x1 <= x0) return false;
  c.x0 = (short)x0;
  c.x1 = (short)x1;
  return true;
}

// Fragment-path interpolants: the reference advances varyings once per 4-pixel
// chunk (v += interp_step, glsl-to-cxx step_interp_inputs), a running sum.
// wr_chunk_base walks that sum to the first chunk a tile touches (warp-uniform,
// once per command/row/tile); wr_chunk_lane finishes the walk for one pixel
// (at most 32 more additions inside a 128-pixel tile).
template <int N>
WRD int wr_chunk_base(const RasterArgs& a, const float* o, const float* step, const CmdHot& c, int tx0, float (*base)[N]) {
  int kb = max(0, (max(tx0, (int)c.x0) - (int)c.x0) >> 2);
#pragma unroll
  for (int i = 0; i < N; i++) {
    float is = __fmul_rn(step[i], 4.0f);
    float v = o[i];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      // init_interp: lane j of chunk 0 = lane j-1 + step (glsl.h:3083-3088);
      // every later chunk adds interp_step to each lane
      float l = a.rl ? a.rl[j * WR_NI + i] : v;
      l = wr_repeat_add(l, is, kb);
      base[j][i] = l;
      v = __fadd_rn(v, step[i]);
    }
  }
  return kb;
}
// lane j (0..3) of chunk k >= kb, given the lanes of chunk kb in base
template <int N>
WRD void wr_chunk_lane(const RasterArgs& a, const float (*base)[N], const float* step, int kb, int k, int j, float* out) {
#pragma unroll
  for (int i = 0; i < N; i++) {
    float is = __fmul_rn(step[i], 4.0f);
    float v = base[j][i];
    for (int s = kb; s < k; s++) v = __fadd_rn(v, is);
    out[i] = v;
  }
  if (a.persp) {  // the sums above are interp_perspective: the varying is w times that
    const float w = 1.0f / wr_persp_zw(*a.persp, 1, 4 * k + j);
#pragma unroll
    for (int i = 0; i < N; i++) out[i] = out[i] * w;
  }
}

// ---- fragment stage: ps_quad_textured -------------------------------------------
// (webrender/res/ps_quad_textured.glsl:39-64, ps_quad.glsl:406-417).  The first
// len&~3 pixels of a span are drawn by swgl_drawSpanRGBA8 (solid commit or
// swgl_commitTextureLinearColorRGBA8), the rest by the fragment shader.
struct QuadShader {
  struct Row {
    float o[2], step[2];
    TexRow tr;
  };
  WRD_MEMBER void row_setup(const RasterArgs& a, const CmdHot& c, int y, int tx0, bool rgba, Row& r) {
    r.tr.mode = TEX_NONE;
    r.tr.body_len = 0;
    if (!(c.flags & CMD_TEXTURED)) return;
    const CmdCold& k = a.cold[c.cold];
    wr_row_interp<2>(a, k, c, y, r.o, r.step);
    int len = c.x1 - c.x0;
    int body_len = (rgba && len >= 4 && !(c.flags & CMD_OUT_RRRR) && !a.persp) ? (len & ~3) : 0;  // (no span shaders under perspective)
    float u[4], v[4];
    for (int j = 0; j < 4; j++) {
      float uv[2];
      wr_interp_at<2>(a, r.o, r.step, j, uv);
      u[j] = uv[0];
      v[j] = uv[1];
    }
    wr_tex_row_setup(a.color0, k.f, false, body_len, u, v, max(tx0, (int)c.x0) - (int)c.x0, r.tr);
  }
  WRD_MEMBER Px source(const RasterArgs& a, const CmdHot& c, const Row& r, int x, int, bool rgba) {
    Px col{c.col[0], c.col[1], c.col[2], c.col[3]};
    const int len = c.x1 - c.x0;
    int rel = x - c.x0;
    if (!(c.flags & CMD_TEXTURED)) {
      // swgl_drawSpanRGBA8 commits v_color for the span body even for mask quads;
      // only the fragment-shader tail applies .rrrr.  R8 targets have no span
      // shader: always the fragment path.
      if (c.flags & CMD_OUT_RRRR) {
        int body_len0 = (rgba && len >= 4 && !a.persp) ? (len & ~3) : 0;
        if (rel >= body_len0) col.b = col.g = col.a = col.r;
      }
      return col;
    }
    const TexView& t = a.color0;
    if (rel < r.tr.body_len) return px_apply_color(wr_tex_body(t, r.tr, rel), col);
    // fragment path: fs_sample_color0 (sample_color0.glsl:25-31), v_color == 1
    const CmdCold& k = a.cold[c.cold];
    float uv[2];
    wr_interp_at<2>(a, r.o, r.step, rel, uv);
    float tex[4];
    wr_tex_fragment(t, wr_clamp(uv[0], k.f[0], k.f[2]), wr_clamp(uv[1], k.f[1], k.f[3]), tex);
    Px o;
    if (c.flags & CMD_OUT_RRRR) {
      int rr = wr_round_pixel(tex[0], 255.0f) & 0xFFFF;
      o = Px{rr, rr, rr, rr};
    } else {
      o.r = wr_round_pixel(tex[0], 255.0f) & 0xFFFF;
      o.g = wr_round_pixel(tex[1], 255.0f) & 0xFFFF;
      o.b = wr_round_pixel(tex[2], 255.0f) & 0xFFFF;
      o.a = wr_round_pixel(tex[3], 255.0f) & 0xFFFF;
    }
    return o;
  }
};

template <> struct WrRun<QuadShader> {
  enum { n = 2 };
  WRD_MEMBER int drawn(const QuadShader::Row& r) { return r.tr.body_len; }
};

// One pixel of one command through depth test, fragment stage, AA/mask
// modifiers and the blend stage.  Shared by the tile kernel and (tests only) the
// host emulation.  px = packed destination pixel (RGBA8) or value (R8).
template <class S, int FMT>
WRD void wr_shade_pixel(const RasterArgs& a, const CmdHot& c, const typename S::Row& row, int xx, int y,
                        bool use_depth, uint32_t& px, uint32_t& zb, bool& dirty, bool& zdirty) {
  if (use_depth) {
    uint32_t z = c.z;
    // perspective: z varies per sample — packDepth() of the stepped gl_FragCoord.z (rasterize.h:345-347, 695-716)
    if (a.persp) z = (uint32_t)(int)(wr_persp_zw(*a.persp, 0, xx - (int)c.x0) * 16777215.0f);
    if (!((int)z <= (int)zb)) return;  // GL_LEQUAL (check_depth compares sign-extended I32 lanes)
    if (a.depth_mode == WRCU_DEPTH_TEST_WRITE) { zb = z; zdirty = true; }
  }
  Px src = S::source(a, c, row, xx, y, FMT == WRCU_FMT_RGBA8);
  if (a.blend != WRCU_BLEND_NONE) {
    if (c.flags & (CMD_AA | CMD_MASK)) {
      const CmdCold& k = a.cold[c.cold];
      // Order of the two source modifiers: the blend stage applies AA then the
      // clip mask (blend.h:447-461); commit_masked_solid_span (swgl_ext.h:10-24)
      // — whole chunks of solid spans — folds the mask into the colour first.
      int len = c.x1 - c.x0;
      bool mask_first = (c.flags & CMD_SPAN_SOLID) && (xx - c.x0) < (len >= 4 ? (len & ~3) : 0);
      int mk = 255;
      if (c.flags & CMD_MASK) mk = __ldg(k.mask_ptr + (size_t)(y - k.cmy) * k.mask_pitch + (xx - k.cmx));
      if ((c.flags & CMD_MASK) && mask_first) {
        if (FMT == WRCU_FMT_RGBA8) src = px_scale255(src, mk);
        else src.r = wr_muldiv255(src.r, mk);
      }
      if (c.flags & CMD_AA) {
        int aa = wr_aa_weight(a, c, k, xx);
        if (FMT == WRCU_FMT_RGBA8) src = px_scale256(src, aa);
        else src.r = wr_muldiv256(src.r, aa);
      }
      if ((c.flags & CMD_MASK) && !mask_first) {
        if (FMT == WRCU_FMT_RGBA8) src = px_scale255(src, mk);
        else src.r = wr_muldiv255(src.r, mk);
      }
    }
    if (FMT == WRCU_FMT_RGBA8) {
      int key = a.blend;
      Px kc = a.blend_color;
      if (c.flags & (CMD_DROP_SHADOW | CMD_SUBPIXEL_TEXT)) {  // SWGL_CLIP_FLAG_BLEND_OVERRIDE (rasterize.h:410-413)
        const CmdCold& k = a.cold[c.cold];
        key = (c.flags & CMD_DROP_SHADOW) ? WRCU_BLEND__DROP_SHADOW : WRCU_BLEND__SUBPIXEL_TEXT;
        kc = Px{k.i[0] & 0xFFFF, (k.i[0] >> 16) & 0xFFFF, k.i[1] & 0xFFFF, (k.i[1] >> 16) & 0xFFFF};
      }
      px = px_pack(wr_blend_rgba8(key, src, px_unpack(px), kc));
    }
    else px = wr_pack16(wr_blend_r8(a.blend, src.r, (int)px));
  } else {
    if (FMT == WRCU_FMT_RGBA8) px = px_pack(src);
    else px = wr_pack16(src.r);
  }
  dirty = true;
}

#ifdef WRCU_HOSTEMU
// tests only: the same per-pixel code, pixel by pixel, commands in batch order
template <class S, int FMT>
static void wr_raster(const RasterArgs& a) {
  const BatchInfo bi = *a.info;
  if (a.fast_eligible && bi.simple) return;
  for (int y = 0; y < a.tgt.h; y++) {
    uint8_t* rowp = a.tgt.color + (size_t)y * a.tgt.color_pitch;
    uint32_t* zrow = a.tgt.depth ? (uint32_t*)((uint8_t*)a.tgt.depth + (size_t)y * a.tgt.depth_pitch) : nullptr;
    const bool use_depth = a.depth_mode != WRCU_DEPTH_OFF && zrow != nullptr;
    for (int i = 0; i < a.n; i++) {
      CmdHot c = a.hot[i];
      if (y < c.y0 || y >= c.y1) continue;
      GenRow g;
      PerspRow prow;
      RasterArgs ar = a;
      ar.gen = &g;
      ar.persp = nullptr;
      if (c.flags & CMD_PERSP) {
        const CmdHot c0 = c;
        if (!wr_persp_row(a.row_tab, a.cold[c0.cold], c0, y, g, prow, c)) continue;
        ar.persp = &prow;
      } else if (c.flags & CMD_GENERAL) {
        const CmdHot c0 = c;
        if (!wr_general_row(a.cold[c0.cold], c0, y, g, c)) continue;
      }
      if ((c.flags & CMD_CLIP_DIST) && !wr_clip_dist_row(ar, ar.cold[c.cold], c, y)) continue;
      typename S::Row row;
      // With depth testing on, every maximal run of passing samples is drawn as a span of its own
      // (draw_depth_span, rasterize.h:612-657): chunk phase, span-shader body and tail restart at the run.
      WrRunWalk<S> walk;
      walk.reset();
      int xs = c.x0;
      while (xs < c.x1) {
        CmdHot cr = c;
        if (use_depth && !ar.persp) {
          while (xs < c.x1 && !(c.z <= zrow[xs])) xs++;
          int s0 = xs;
          while (xs < c.x1 && c.z <= zrow[xs]) xs++;
          if (xs == s0) break;
          cr.x0 = (short)s0;
          cr.x1 = (short)xs;
          walk.begin(ar, ar.cold[c.cold], cr, y);
        } else {
          xs = c.x1;
        }
        const RasterArgs& a = ar;  // shadows: the shaders see the row state
        int drawn = 0;
        for (int tx0 = (cr.x0 / WRCU_TILE_W) * WRCU_TILE_W; tx0 < cr.x1; tx0 += WRCU_TILE_W) {
          S::row_setup(a, cr, y, tx0, FMT == WRCU_FMT_RGBA8, row);
          if (tx0 <= cr.x0) drawn = WrRun<S>::drawn(row);
          for (int xx = max((int)cr.x0, tx0); xx < min((int)cr.x1, tx0 + WRCU_TILE_W); xx++) {
            uint32_t px = FMT == WRCU_FMT_RGBA8 ? ((uint32_t*)rowp)[xx] : rowp[xx];
            uint32_t zb = use_depth ? zrow[xx] : 0;
            bool dirty = false, zdirty = false;
            wr_shade_pixel<S, FMT>(a, cr, row, xx, y, use_depth, px, zb, dirty, zdirty);
            if (dirty) { if (FMT == WRCU_FMT_RGBA8) ((uint32_t*)rowp)[xx] = px; else rowp[xx] = (uint8_t)px; }
            if (zdirty) zrow[xx] = zb;
          }
        }
        if (use_depth && !ar.persp) walk.end(ar, cr, drawn);
      }
    }
  }
}
static void wr_fold_solid(const RasterArgs& a) {
  const BatchInfo bi = *a.info;
  const int4 cov = wr_cover_tiles(bi, a.tgt);
  if (!bi.simple || cov.z <= cov.x || cov.w <= cov.y) return;
  wr_fold_host(a.hot, a.n, bi.premul_valid != 0, a.fold);
}
// Pixels of tiles inside the common cover go through the fold's tables (when one was launched), every
// other pixel through the commands in batch order: disjoint pixel sets, so the order between them is free.
static void wr_raster_solid_premult(const RasterArgs& a) {
  const BatchInfo bi = *a.info;
  if (!bi.simple) return;
  int4 cov = make_int4(0, 0, 0, 0);
  if (a.fold) {
    cov = wr_cover_tiles(bi, a.tgt);
    cov = make_int4(cov.x * WRCU_TILE_W, cov.y * WRCU_TILE_H, cov.z * WRCU_TILE_W, cov.w * WRCU_TILE_H);
    if (cov.z <= cov.x || cov.w <= cov.y) cov = make_int4(0, 0, 0, 0);
  }
  for (int y = cov.y; y < cov.w; y++) {
    uint32_t* rowp = (uint32_t*)(a.tgt.color + (size_t)y * a.tgt.color_pitch);
    for (int x = cov.x; x < cov.z; x++) rowp[x] = wr_fold_px(a.fold, rowp[x]);
  }
  for (int i = 0; i < a.n; i++) {
    const CmdHot c = a.hot[i];
    uint32_t srb = (uint32_t)c.col[0] | ((uint32_t)c.col[2] << 16), sga = (uint32_t)c.col[1] | ((uint32_t)c.col[3] << 16);
    uint32_t cc = 255u - c.col[3];
    for (int y = c.y0; y < c.y1; y++) {
      uint32_t* rowp = (uint32_t*)(a.tgt.color + (size_t)y * a.tgt.color_pitch);
      for (int x = c.x0; x < c.x1; x++) {
        if (y >= cov.y && y < cov.w && x >= cov.x && x < cov.z) continue;
        uint32_t p = rowp[x];
        uint32_t rb = wr_premult_over_pair(p & 0x00FF00FFu, srb, cc);
        uint32_t ga = wr_premult_over_pair((p >> 8) & 0x00FF00FFu, sga, cc);
        rowp[x] = rb | (ga << 8);
      }
    }
  }
}
#else
// Shaders whose Row holds only warp-uniform state (nothing computed for "this lane's pixels") may have
// narrow spans shaded one pixel per lane (see wr_raster_tile).
template <class S> struct WrNarrowSpans { enum { v = 0 }; };

// first index in [from, to) of a bit equal to `want` in the bitmap `w`; `to` when there is none (warp-uniform)
WRD int wr_bits_next(const uint32_t* w, int from, int to, bool want) {
  while (from < to) {
    uint32_t v = __ldg(w + (from >> 5));
    if (!want) v = ~v;
    v &= 0xFFFFFFFFu << (from & 31);
    if (v) return min((from & ~31) + __ffs((int)v) - 1, to);
    from = (from & ~31) + 32;
  }
  return to;
}

// Row state across the tiles of a row.  A full-width surface (a video frame, a page-wide gradient) crosses 30 tiles
// of a 4K row and S::row_setup — edge interpolants, quantised start lanes, filter selection — is the same work in each
// of them.  In STRIP mode (RasterArgs::strip_seg) a CTA takes a run of horizontally adjacent tiles and walks it left
// to right; its warps stay on their rows, so a shader that says its Row can serve a later tile of the same
// (command,row) (WrRowReuse<S>::ok) has it kept instead of rebuilt.
template <class S> struct WrRowReuse {
  enum { v = 0 };
  WRD_MEMBER bool ok(const typename S::Row&) { return false; }
};
template <class S> struct WrRowCache {
  typename S::Row row;
  int cold, y;  // the (command,row) `row` was built for; cold < 0: none
};

// ---- the generic tile kernel (any command kind via the shader policy S, any
// blend key).  S::row_setup computes per-(command,row) constants once per warp
// (all 32 lanes of a warp share the row, so the work is warp-uniform);
// S::source returns the fragment stage's output for one pixel as 16-bit lanes.
template <class S, int FMT, bool RUNS>
WRD void wr_raster_tile(RasterArgs& a, const int tx0, const int ty0, CmdHot* sh, int* wsum, unsigned short* list,
                        const bool skip_copy, WrRowCache<S>& cache) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int x = tx0 + lane * 4, y = ty0 + warp;
  const bool row_ok = y < a.tgt.h;
  GenRow grow;
  PerspRow prow;
  a.gen = &grow;
  a.persp = nullptr;
  uint32_t px[4] = {0, 0, 0, 0};
  uint32_t zb[4] = {0, 0, 0, 0};
  bool loaded = false, dirty = false, zdirty = false;
  uint8_t* rowp = a.tgt.color + (size_t)y * a.tgt.color_pitch;
  uint32_t* zrow = a.tgt.depth ? (uint32_t*)((uint8_t*)a.tgt.depth + (size_t)y * a.tgt.depth_pitch) : nullptr;
  const bool use_depth = a.depth_mode != WRCU_DEPTH_OFF && zrow != nullptr;
  const bool cover_ok = a.blend == WRCU_BLEND_NONE && a.depth_mode == WRCU_DEPTH_OFF;

  // Commands are taken in chunks of CHUNK_CMDS.  With bitmask bins the tile's mask words for
  // 8192 commands at a time are staged in shared memory first, so empty chunks are skipped
  // without touching global memory or a barrier.
  for (int sbase = 0; sbase < a.n; sbase += WRCU_THREADS * 32) {
  const int send = min(a.n, sbase + WRCU_THREADS * 32);
  // With bitmask bins the set bits of the tile's mask words (one word per thread, 8192 commands per
  // pass) are expanded into an ordered index list in shared memory; the chunk loop below then runs
  // over that list, so a sparse batch (text: a few dozen of 6000 glyphs per tile) costs one chunk
  // instead of a scan over every 256-command chunk.
  int n_items = send - sbase;
  const bool listed = a.tile_mask != nullptr;
  if (listed) {
    const int wi = (sbase >> 5) + (int)threadIdx.x;
    uint32_t word = wi < a.bin_words
        ? (__ldg(a.tile_mask + (size_t)((ty0 / WRCU_TILE_H) * a.bin_tiles_x + tx0 / WRCU_TILE_W) * a.bin_words + wi) |
           __ldg(a.wide_mask + wi))
        : 0u;
    const int cnt = __popc(word);
    int incl = cnt;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int t = __shfl_up_sync(0xFFFFFFFFu, incl, d);
      if (lane >= d) incl += t;
    }
    __syncthreads();  // previous pass / tile done with wsum and the list
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    int pos = incl - cnt;
    n_items = 0;
#pragma unroll
    for (int w = 0; w < WRCU_THREADS / 32; w++) {
      const int v = wsum[w];
      if (w < warp) pos += v;
      n_items += v;
    }
    while (word) {
      const int b = __ffs((int)word) - 1;
      word &= word - 1;
      list[pos++] = (unsigned short)(threadIdx.x * 32 + b);
    }
    __syncthreads();
  }
  for (int ib = 0; ib < n_items; ib += CHUNK_CMDS) {
    // Binning: each thread tests one command of the chunk against this tile; the
    // survivors' indices are compacted in batch order (ballot + prefix sum), so
    // the pixel loop only visits commands that touch the tile.
    const int m = min(CHUNK_CMDS, n_items - ib);
    int keep = 0;
    CmdHot mine;
    const bool candidate = (int)threadIdx.x < m;
    const int cidx = candidate ? (listed ? sbase + (int)list[ib + threadIdx.x] : sbase + ib + (int)threadIdx.x) : 0;
    bool cover = false;
    if (candidate) {
      mine = a.hot[cidx];
      keep = mine.x1 > tx0 && mine.x0 < tx0 + WRCU_TILE_W && mine.y1 > ty0 && mine.y0 < ty0 + WRCU_TILE_H &&
             mine.x1 > mine.x0 && !(skip_copy && (mine.flags & CMD_COPY)) &&
             (!a.glyph_major || (mine.flags & CMD_ORDERED));
      // Hidden-surface removal inside a batch: with blending and depth off a command that
      // overwrites every writable pixel of this tile makes all earlier commands of the batch
      // invisible here, so the pixel loop can start at the last such command.
      cover = keep && cover_ok &&
              !(mine.flags & (CMD_MASK | CMD_AA | CMD_GENERAL | CMD_CLIP_DIST | CMD_DROP_SHADOW | CMD_SUBPIXEL_TEXT)) &&
              mine.x0 <= max(tx0, a.tgt.cx0) && mine.x1 >= min(tx0 + WRCU_TILE_W, a.tgt.cx1) &&
              mine.y0 <= max(ty0, a.tgt.cy0) && mine.y1 >= min(ty0 + WRCU_TILE_H, a.tgt.cy1);
    }
    const unsigned bal = __ballot_sync(0xFFFFFFFFu, keep);
    __syncthreads();  // previous chunk fully consumed
    if (lane == 0) wsum[warp] = __popc(bal);
    if (threadIdx.x == 0) wsum[WRCU_THREADS / 32] = 0;
    __syncthreads();
    int off = 0, total = 0;
#pragma unroll
    for (int w = 0; w < WRCU_THREADS / 32; w++) {
      const int v = wsum[w];
      if (w < warp) off += v;
      total += v;
    }
    const int slot = off + __popc(bal & ((1u << lane) - 1u));
    if (keep) sh[slot] = mine;
    if (cover) atomicMax(&wsum[WRCU_THREADS / 32], slot);
    __syncthreads();
    const int first_cmd = wsum[WRCU_THREADS / 32];
    for (int i = first_cmd; i < total; i++) {
      CmdHot c = sh[i];
      if (!row_ok || y < c.y0 || y >= c.y1) continue;          // warp-uniform
      const int bit0 = c.x0;  // sample of bit 0 of the command's failing-sample bitmaps (the hot rect's x0)
      a.persp = nullptr;
      if (c.flags & CMD_PERSP) {
        // perspective polygon: span, z/w and edge state of this row from its edge walk (warp-uniform)
        const CmdHot c0 = c;
        if (!wr_persp_row(a.row_tab, a.cold[c0.cold], c0, y, grow, prow, c)) continue;
        if (c.x1 <= tx0 || c.x0 >= tx0 + WRCU_TILE_W) continue;
        a.persp = &prow;
      } else if (c.flags & CMD_GENERAL) {
        // rotated quad: this row's span comes from the edge walk (warp-uniform)
        const CmdHot c0 = c;
        if (!wr_general_row(a.cold[c0.cold], c0, y, grow, c)) continue;
        if (c.x1 <= tx0 || c.x0 >= tx0 + WRCU_TILE_W) continue;
      }
      if (c.flags & CMD_CLIP_DIST) {
        if (!wr_clip_dist_row(a, a.cold[c.cold], c, y)) continue;
        if (c.x1 <= tx0 || c.x0 >= tx0 + WRCU_TILE_W) continue;
      }
      if (!loaded) {
        // lazy tile load: first command that touches this row
        loaded = true;
        wr_pdl_wait();  // the kernel ahead of this one in the stream may still be writing these pixels
        if (FMT == WRCU_FMT_RGBA8) {
          uint4 v = *(const uint4*)(rowp + (size_t)x * 4);
          px[0] = v.x; px[1] = v.y; px[2] = v.z; px[3] = v.w;
        } else {
          uint32_t v = *(const uint32_t*)(rowp + x);
          px[0] = v & 0xFF; px[1] = (v >> 8) & 0xFF; px[2] = (v >> 16) & 0xFF; px[3] = v >> 24;
        }
        if (use_depth) {
          uint4 v = *(const uint4*)(zrow + x);
          zb[0] = v.x; zb[1] = v.y; zb[2] = v.z; zb[3] = v.w;
        }
      }
      // (strip mode: the Row of the tile to the left, when this is still its command and the shader allows it)
      typename S::Row row_local;
      const bool cacheable = WrRowReuse<S>::v && a.strip_seg > 0 && !(c.flags & (CMD_GENERAL | CMD_PERSP | CMD_CLIP_DIST));
      typename S::Row& row = cacheable ? cache.row : row_local;
      // With depth testing on, each maximal run of passing samples of the row's span is drawn as a span of
      // its own (draw_depth_span, rasterize.h:612-657).  The runs are walked in order up to this tile
      // (warp-uniform; the failing-sample bitmap was written by wr_depth_fail_rows before this kernel
      // started), because a run's chunk lanes continue from the previous run's.  Without depth testing, or
      // when every sample of the span passes, the span is its only run.
      const CmdCold& kc = a.cold[c.cold];
      const uint32_t* frow = (RUNS && use_depth && kc.fail_off >= 0)
          ? a.fail_pool + (size_t)kc.fail_off + (size_t)(y - (int)c.y0) * (kc.fail_w + 1) : nullptr;
      const bool runs = RUNS && frow && __ldg(frow) != 0u;
      WrRunWalk<S> walk;
      walk.reset();
      int xs = c.x0;
      for (;;) {
        CmdHot cr = c;
        bool here = true;
        if (runs) {
          if (xs >= c.x1) break;
          const int s0 = bit0 + wr_bits_next(frow + 1, xs - bit0, (int)c.x1 - bit0, false);
          if (s0 >= c.x1 || s0 >= tx0 + WRCU_TILE_W) break;
          const int e0 = bit0 + wr_bits_next(frow + 1, s0 - bit0, (int)c.x1 - bit0, true);
          xs = e0;
          here = e0 > tx0;
          if (WrRun<S>::n == 0 && !here) continue;  // nothing carries over from runs left of the tile
          cr.x0 = (short)s0;
          cr.x1 = (short)e0;
          walk.begin(a, kc, cr, y);
        }
        // (for a run left of the tile only its span-shader pixel count is needed)
        if (cacheable && !runs && cache.cold == (int)c.cold && cache.y == y && WrRowReuse<S>::ok(cache.row)) {
          // kept from the tile to the left
        } else {
          S::row_setup(a, cr, y, here ? tx0 : ((int)cr.x0 & ~(WRCU_TILE_W - 1)), FMT == WRCU_FMT_RGBA8, row);
          if (cacheable) { cache.cold = runs ? -1 : (int)c.cold; cache.y = y; }
        }
        if (here) {
          const CmdHot& c = cr;
      const int nxs = max((int)c.x0, tx0), nw = min((int)c.x1, tx0 + WRCU_TILE_W) - nxs;
      if (WrNarrowSpans<S>::v && nw <= 32) {
        // Narrow span (a glyph row is ~12 pixels): with 4 pixels per lane only 3-4 lanes would work
        // through four pixel slots.  Instead lane i takes pixel nxs + i: the destination pixels are
        // gathered from their owners, shaded in ONE slot, and scattered back.  (Only for shaders
        // whose Row is warp-uniform — S::source must not depend on which lane asks.)
        const int gx = nxs + lane - tx0;  // tile-relative pixel of this lane
        const int owner = (gx >> 2) & 31, slot = gx & 3;
        uint32_t g0 = __shfl_sync(0xFFFFFFFFu, px[0], owner), g1 = __shfl_sync(0xFFFFFFFFu, px[1], owner);
        uint32_t g2 = __shfl_sync(0xFFFFFFFFu, px[2], owner), g3 = __shfl_sync(0xFFFFFFFFu, px[3], owner);
        uint32_t mypx = slot == 0 ? g0 : (slot == 1 ? g1 : (slot == 2 ? g2 : g3));
        uint32_t myz = 0;
        if (use_depth) {
          uint32_t z0 = __shfl_sync(0xFFFFFFFFu, zb[0], owner), z1 = __shfl_sync(0xFFFFFFFFu, zb[1], owner);
          uint32_t z2 = __shfl_sync(0xFFFFFFFFu, zb[2], owner), z3 = __shfl_sync(0xFFFFFFFFu, zb[3], owner);
          myz = slot == 0 ? z0 : (slot == 1 ? z1 : (slot == 2 ? z2 : z3));
        }
        bool d1 = false, zd1 = false;
        if (lane < nw) wr_shade_pixel<S, FMT>(a, c, row, nxs + lane, y, use_depth, mypx, myz, d1, zd1);
        const unsigned dmask = __ballot_sync(0xFFFFFFFFu, d1), zmask = __ballot_sync(0xFFFFFFFFu, zd1);
        if (dmask | zmask) {
#pragma unroll
          for (int p = 0; p < 4; p++) {
            const int from = x + p - nxs;  // lane that shaded this pixel
            const uint32_t v = __shfl_sync(0xFFFFFFFFu, mypx, from & 31);
            const uint32_t vz = use_depth ? __shfl_sync(0xFFFFFFFFu, myz, from & 31) : 0u;
            if (from >= 0 && from < nw) {
              if ((dmask >> from) & 1u) { px[p] = v; dirty = true; }
              if ((zmask >> from) & 1u) { zb[p] = vz; zdirty = true; }
            }
          }
        }
      } else {
#pragma unroll
      for (int p = 0; p < 4; p++) {
        int xx = x + p;
        if (xx < c.x0 || xx >= c.x1) continue;
        wr_shade_pixel<S, FMT>(a, c, row, xx, y, use_depth, px[p], zb[p], dirty, zdirty);
      }
      }
        }
        if (!runs) break;
        walk.end(a, cr, WrRun<S>::drawn(row));
      }
    }
  }
  }  // super-chunk
  if (dirty) {
    if (FMT == WRCU_FMT_RGBA8) {
      *(uint4*)(rowp + (size_t)x * 4) = make_uint4(px[0], px[1], px[2], px[3]);
    } else {
      *(uint32_t*)(rowp + x) = px[0] | (px[1] << 8) | (px[2] << 16) | (px[3] << 24);
    }
  }
  if (zdirty) *(uint4*)(zrow + x) = make_uint4(zb[0], zb[1], zb[2], zb[3]);
}

// Persistent CTAs stride over the tiles of the batch's bounding box (known only
// on the device), so a batch that touches a small part of a large target costs
// a small launch, and a full-target batch fills the chip evenly.
// Resident CTAs per SM the kernel is compiled for (register budget = 65536 / (256 * v)): shaders whose
// work is latency-bound (many small commands) specialise this to 3.
template <class S> struct WrMinCtas { enum { v = 2 }; };

// RUNS: the variant that reproduces depth runs (launched for depth-tested batches of the kinds whose
// shading depends on them); the plain variant carries none of that code.
template <class S, int FMT, bool RUNS = false>
__global__ void __launch_bounds__(WRCU_THREADS, WrMinCtas<S>::v)
wr_raster(RasterArgs a) {
  __shared__ CmdHot sh[CHUNK_CMDS];
  __shared__ int wsum[WRCU_THREADS / 32 + 1];  // per-warp survivor counts + the last covering command
  wr_pdl_launch_dependents();
  if (!a.pdl_early) wr_pdl_wait();
  const BatchInfo bi = *a.info;
  if (a.fast_eligible && bi.simple) return;  // handled by wr_raster_solid_premult
  const bool skip_copy = a.copy_eligible && bi.all_copy;  // CMD_COPY commands are drawn by wr_composite_copy
  if (skip_copy && bi.n_noncopy == 0) return;
  if (a.glyph_major && bi.n_ordered == 0) return;  // wr_raster_glyphs drew the whole batch
  const uint32_t* any_map = a.glyph_major ? a.tile_ord : a.tile_any;
  const bool any_all = !a.glyph_major && a.tile_any && a.tile_any[a.any_words];
  const int bx0 = max(bi.bx0, 0) / WRCU_TILE_W, by0 = max(bi.by0, 0) / WRCU_TILE_H;
  const int bx1 = (min(bi.bx1, a.tgt.w) + WRCU_TILE_W - 1) / WRCU_TILE_W;
  const int by1 = (min(bi.by1, a.tgt.h) + WRCU_TILE_H - 1) / WRCU_TILE_H;
  const int nx = bx1 - bx0, n_tiles = nx * (by1 - by0);
  if (nx <= 0 || n_tiles <= 0) return;
  // tiles are handed out dynamically: their cost varies with what lands on them
  __shared__ int s_tile;
  __shared__ unsigned short list[WRCU_THREADS * 32];  // command indices of the tile's set mask bits, in order
  WrRowCache<S> cache;
  cache.cold = -1;
  cache.y = -1;
  if (WrRowReuse<S>::v && a.strip_seg > 0) {
    // strip mode: the work items are runs of strip_seg horizontally adjacent tiles, walked left to right
    const int segs = (nx + a.strip_seg - 1) / a.strip_seg, n_items = segs * (by1 - by0);
    for (;;) {
      if (threadIdx.x == 0) s_tile = atomicAdd(const_cast<int*>(&a.info->tile_counter), 1);
      __syncthreads();
      const int t = s_tile;
      if (t >= n_items) break;
      const int ty = by0 + t / segs, txa = bx0 + (t % segs) * a.strip_seg, txb = min(txa + a.strip_seg, bx1);
      cache.cold = -1;
      for (int tx = txa; tx < txb; tx++) {
        wr_raster_tile<S, FMT, RUNS>(a, tx * WRCU_TILE_W, ty * WRCU_TILE_H, sh, wsum, list, skip_copy, cache);
        __syncthreads();
      }
    }
    return;
  }
  for (;;) {
    if (threadIdx.x == 0) {
      // binned batches: pass over tiles no command touches (text: ~7 of 8 tiles of a 4K page) with one load each
      int tn;
      for (;;) {
        tn = atomicAdd(const_cast<int*>(&a.info->tile_counter), 1);
        if (tn >= n_tiles || !any_map || !a.tile_mask) break;
        const int tid = (by0 + tn / nx) * a.bin_tiles_x + bx0 + tn % nx;
        if (any_all || ((any_map[tid >> 5] >> (tid & 31)) & 1u)) break;
      }
      s_tile = tn;
    }
    __syncthreads();
    const int t = s_tile;
    if (t >= n_tiles) break;
    wr_raster_tile<S, FMT, RUNS>(a, (bx0 + t % nx) * WRCU_TILE_W, (by0 + t / nx) * WRCU_TILE_H, sh, wsum, list, skip_copy, cache);
    __syncthreads();
  }
}

// ---- depth runs: which samples of each (command,row) fail the depth test ---------------------------
// The reference keeps depth as runs per row and draws a span run by run (rasterize.h:5-257, 601-657);
// where a run starts decides chunk phase, span-shader body vs tail and the interpolant sums, and a run
// may start far left of the tile a CTA is drawing.  This kernel runs between the setup and the raster
// kernel and writes, for every command that asked for it (CmdCold::fail_off) and every row, the bitmap of
// failing samples over the command's hot rect:
//   fails(x) = x outside the row's span, or  z > depth_before_batch(x),
//              or (depth writes on) z > z' of an EARLIER command of this batch covering (x, y)
// — with LEQUAL and writes the depth a command sees is the minimum over what was there and everything
// drawn before it, whether those draws passed or not.  One CTA per command (earlier commands that can
// occlude it are collected once into shared memory), one warp per row.
#define WR_FAIL_CAND 1024
WRD bool wr_row_span_of(RasterArgs& ar, GenRow& g, const CmdHot& c0, int y, int& x0, int& x1) {
  if (y < c0.y0 || y >= c0.y1 || c0.x1 <= c0.x0) return false;
  CmdHot c = c0;
  const CmdCold& k = ar.cold[c0.cold];
  ar.gen = &g;
  if (c0.flags & CMD_PERSP) {
    PerspRow pr;
    if (!wr_persp_row(ar.row_tab, k, c0, y, g, pr, c)) return false;
  } else if ((c0.flags & CMD_GENERAL) && !wr_general_row(k, c0, y, g, c)) return false;
  if ((c.flags & CMD_CLIP_DIST) && !wr_clip_dist_row(ar, k, c, y)) return false;
  x0 = c.x0;
  x1 = c.x1;
  return x1 > x0;
}
__global__ void __launch_bounds__(256) wr_depth_fail_rows(RasterArgs a, uint32_t* pool) {
  // occluder candidates of the current command: index and hot rect (axis-aligned candidates are tested from
  // shared memory alone; CMD_GENERAL / CMD_CLIP_DIST ones re-derive their row span)
  __shared__ unsigned short cand[WR_FAIL_CAND];
  __shared__ short4 crect[WR_FAIL_CAND];
  __shared__ unsigned char cgen[WR_FAIL_CAND];
  __shared__ int ncand;
  wr_pdl_launch_dependents();
  wr_pdl_wait();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int G = (int)gridDim.x;
  RasterArgs ar = a;
  GenRow g;
  // Work items = groups of `nwarps` rows of the commands that carry bitmaps (CMD_RUNS), dealt round-robin to
  // the persistent CTAs: a tall command spreads over the grid, thousands of glyph-sized ones cost a CTA each.
  // The hot records are staged through shared memory 256 at a time: every CTA walks the whole list, and one
  // dependent global load per command (x 60 glyphs) was most of this kernel's time on small batches.
  // Many small commands (a text run: 60 glyphs of 12 rows) are dealt a CTA each instead (command-major): no CTA
  // walks the list at all.
  __shared__ CmdHot hot_sh[256];
  const bool cmd_major = a.n >= 48;
  int gbase = 0;
  for (int ci = cmd_major ? (int)blockIdx.x : 0; ci < a.n; ci += cmd_major ? G : 1) {
    CmdHot c0;
    if (cmd_major) {
      c0 = a.hot[ci];
    } else {
      if ((ci & 255) == 0) {
        __syncthreads();
        if (ci + (int)threadIdx.x < a.n) hot_sh[threadIdx.x] = a.hot[ci + threadIdx.x];
        __syncthreads();
      }
      c0 = hot_sh[ci & 255];
    }
    if (!(c0.flags & CMD_RUNS) || c0.x1 <= c0.x0) continue;  // CTA-uniform
    const int rows = (int)c0.y1 - (int)c0.y0, ngroups = (rows + nwarps - 1) / nwarps;
    int first = 0, gstride = 1;
    if (!cmd_major) {
      first = ((int)blockIdx.x - gbase % G + G) % G;
      gstride = G;
      gbase += ngroups;
      if (first >= ngroups) continue;  // none of this command's row groups is ours
    }
    const CmdCold& k = a.cold[c0.cold];
    int nc = 0;
    if (a.depth_mode == WRCU_DEPTH_TEST_WRITE) {
      __syncthreads();
      if (threadIdx.x == 0) ncand = 0;
      __syncthreads();
      for (int j = threadIdx.x; j < ci; j += blockDim.x) {
        const CmdHot o = a.hot[j];
        if (o.x1 > o.x0 && o.z < c0.z && o.x0 < c0.x1 && c0.x0 < o.x1 && o.y0 < c0.y1 && c0.y0 < o.y1) {
          const int p = atomicAdd(&ncand, 1);
          if (p < WR_FAIL_CAND) {
            cand[p] = (unsigned short)j;
            crect[p] = make_short4(o.x0, o.y0, o.x1, o.y1);
            cgen[p] = (o.flags & (CMD_GENERAL | CMD_CLIP_DIST)) ? 1 : 0;
          }
        }
      }
      __syncthreads();
      nc = ncand;
    }
    const int W = k.fail_w;
    for (int grp = first; grp < ngroups; grp += gstride) {
      const int r = grp * nwarps + warp;
      if (r >= rows) continue;
      const int y = (int)c0.y0 + r;
      int sx0 = 0, sx1 = 0;
      wr_row_span_of(ar, g, c0, y, sx0, sx1);
      uint32_t* out = pool + (size_t)k.fail_off + (size_t)r * (W + 1);
      const uint32_t* zrow = (const uint32_t*)((const uint8_t*)a.tgt.depth + (size_t)y * a.tgt.depth_pitch);
      int cnt = 0;
      for (int wb = 0; wb < W; wb += 32) {
        const int nwords = min(32, W - wb);
        uint32_t mine = 0;
        // eight words (256 samples) per step: the depth loads of a step are independent, so their latencies overlap
        for (int i0 = 0; i0 < nwords; i0 += 8) {
          uint32_t zv[8];
#pragma unroll
          for (int u = 0; u < 8; u++) {
            const int xx = (int)c0.x0 + (wb + i0 + u) * 32 + lane;
            zv[u] = (i0 + u < nwords && xx >= sx0 && xx < sx1) ? zrow[xx] : 0u;  // 0 fails every z > 0
          }
#pragma unroll
          for (int u = 0; u < 8; u++) {
            const int xx = (int)c0.x0 + (wb + i0 + u) * 32 + lane;
            const bool pass = i0 + u < nwords && xx >= sx0 && xx < sx1 && c0.z <= zv[u];
            const uint32_t bal = __ballot_sync(0xFFFFFFFFu, !pass);
            if (lane == i0 + u) mine = bal;
          }
        }
        const int wx0 = (int)c0.x0 + (wb + lane) * 32;  // first sample of this lane's word
        auto or_span = [&](int ox0, int ox1) {
          const int lo = max(ox0 - wx0, 0), hi = min(ox1 - wx0, 32);
          if (hi > lo) mine |= (hi - lo == 32) ? 0xFFFFFFFFu : (((1u << (hi - lo)) - 1u) << lo);
        };
        if (nc > WR_FAIL_CAND) {
          // more occluder candidates than the list holds: test every earlier command directly
          for (int j = 0; j < ci; j++) {
            const CmdHot o = a.hot[j];
            int ox0, ox1;
            if (o.z < c0.z && wr_row_span_of(ar, g, o, y, ox0, ox1)) or_span(ox0, ox1);
          }
        } else {
          for (int q = 0; q < nc; q++) {
            const short4 rc = crect[q];
            if (y < rc.y || y >= rc.w) continue;
            if (!cgen[q]) { or_span(rc.x, rc.z); continue; }
            const CmdHot o = a.hot[cand[q]];
            int ox0, ox1;
            if (wr_row_span_of(ar, g, o, y, ox0, ox1)) or_span(ox0, ox1);
          }
        }
        if (lane < nwords) {
          out[1 + wb + lane] = mine;
          const int lo = max(sx0 - wx0, 0), hi = min(sx1 - wx0, 32);
          if (hi > lo) cnt += __popc(mine & ((hi - lo == 32) ? 0xFFFFFFFFu : (((1u << (hi - lo)) - 1u) << lo)));
        }
      }
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) cnt += __shfl_xor_sync(0xFFFFFFFFu, cnt, d);
      if (lane == 0) out[0] = (uint32_t)cnt;
    }
  }
}

// ---- specialised hot kernel: solid quads, premultiplied-alpha over, no depth,
// no mask/AA (config B, the alpha-blend brush pass).
//
// Work decomposition.  A CTA of 128 threads owns a 128x8 tile; warp w holds rows
// w and w+4, lane l pixels [4l, 4l+4) of both: 8 pixels per thread, kept
// unpacked as (B,R) / (G,A) 16-bit lane pairs for the whole command list.
// CTAs are persistent and stride over the tiles of the batch's bounding box;
// the host sizes the grid so the tile count divides evenly over the resident
// CTAs (see wr_fast_grid).
//
// Per chunk of 128 commands the CTA first CLASSIFIES cooperatively — one
// command per thread against the tile: no overlap (dropped), full cover, or
// partial — and compacts the survivors in batch order into shared memory
// (ballot + prefix sum), together with the per-command blend constants.  The
// pixel loop then runs over survivors only; for a full-cover command it is
// branch-free.
//
// Arithmetic per 16-bit lane, c = 255 - src.a (blend.h:473-474, muldiv255):
//   dst' = dst + src - ((dst*src.a + dst) >> 8)  ==  ((dst*c + 255) >> 8) + src
// (exact: dst - floor(t/256) = ceil((256 dst - t)/256), t = dst*(src.a+1)).
// When every source lane <= src.a (a valid premultiplied colour) the sum cannot
// exceed 255, so `+ src` folds into the multiply-add's addend and the
// saturating pack disappears:   dst' = (dst*c + (255 + 256*src)) >> 8,
// i.e. one IMAD + one PRMT per lane pair = 4 instructions per pixel-layer.
// Batches with over-range colours (src > src.a) take the saturating variant.
#define FAST_THREADS 128
#define FAST_CHUNK 128

// `v0`, `v1`: this thread's pixels of the tile, loaded by the caller one tile ahead (software prefetch: the
// loads of tile t+1 are in flight while tile t is classified and blended — a shallow batch is a
// read-modify-write of the target at HBM speed, and the tile-at-a-time dependency chain
// load → blend → store would otherwise leave half the memory pipeline idle).
template <bool VALID>
WRD void wr_fast_tile(const RasterArgs& a, int tx0, int ty0, uint4* fa, int4* fb, int* wsum, const uint4 v0, const uint4 v1) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int x = tx0 + lane * 4;
  const int y0 = ty0 + warp, y1 = ty0 + warp + 4;
  uint8_t* p0 = a.tgt.color + (size_t)y0 * a.tgt.color_pitch + (size_t)x * 4;
  uint8_t* p1 = a.tgt.color + (size_t)y1 * a.tgt.color_pitch + (size_t)x * 4;
  uint32_t rb[8], ga[8];
  bool loaded = false, dirty = false;
  for (int base = 0; base < a.n; base += FAST_CHUNK) {
    // ---- classify + compact (one command per thread) ----
    int keep = 0;
    uint4 A = make_uint4(0, 0, 0, 0);
    int4 B = make_int4(0, 0, 0, 0);
    if (base + (int)threadIdx.x < a.n) {
      const CmdHot c = a.hot[base + threadIdx.x];
      keep = c.x1 > tx0 && c.x0 < tx0 + WRCU_TILE_W && c.y1 > ty0 && c.y0 < ty0 + WRCU_TILE_H && c.x1 > c.x0;
      A = wr_solid_consts(c);
      A.w = c.x0 <= tx0 && c.x1 >= tx0 + WRCU_TILE_W && c.y0 <= ty0 && c.y1 >= ty0 + WRCU_TILE_H;  // full cover
      B = make_int4(c.x0, c.x1, c.y0, c.y1);
    }
    const unsigned bal = __ballot_sync(0xFFFFFFFFu, keep);
    const unsigned balp = __ballot_sync(0xFFFFFFFFu, keep && !A.w);  // partial-cover survivors
    __syncthreads();  // previous chunk's readers are done with fa/fb/wsum
    if (lane == 0) wsum[warp] = __popc(bal) | (__popc(balp) << 16);
    __syncthreads();
    int off = 0, total = 0, partial = 0;
#pragma unroll
    for (int w = 0; w < FAST_THREADS / 32; w++) {
      const int v = wsum[w];
      if (w < warp) off += v & 0xFFFF;
      total += v & 0xFFFF;
      partial += v >> 16;
    }
    if (keep) {
      const int slot = off + __popc(bal & ((1u << lane) - 1u));
      fa[slot] = A;
      fb[slot] = B;
    }
    __syncthreads();
    if (total == 0) continue;
    if (!loaded) {
      loaded = true;  // first chunk with a command on this tile: unpack the prefetched pixels
      const uint32_t pv[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
      for (int p = 0; p < 8; p++) {
        rb[p] = pv[p] & 0x00FF00FFu;
        ga[p] = (pv[p] >> 8) & 0x00FF00FFu;
      }
    }
    // ---- blend the survivors in batch order ----
    if (partial == 0) {
      // every survivor covers the whole tile: no per-command branch at all
#pragma unroll 4
      for (int i = 0; i < total; i++) {
        const uint4 k = fa[i];
        wr_fast_blend8<VALID>(rb, ga, k.x, k.y, k.z);
      }
      dirty = true;
      continue;
    }
#pragma unroll 2
    for (int i = 0; i < total; i++) {
      const uint4 k = fa[i];
      if (k.w) {
        wr_fast_blend8<VALID>(rb, ga, k.x, k.y, k.z);
        dirty = true;
      } else {
        const int4 r = fb[i];
        const uint32_t srb = (k.y - 0x00FF00FFu) >> 8, sga = (k.z - 0x00FF00FFu) >> 8;
#pragma unroll
        for (int row = 0; row < 2; row++) {
          const int yy = row ? y1 : y0;
          if (yy < r.z || yy >= r.w || r.y <= x || r.x >= x + 4) continue;
#pragma unroll
          for (int p = 0; p < 4; p++) {
            if (x + p >= r.x && x + p < r.y) {
              rb[4 * row + p] = wr_premult_over_pair(rb[4 * row + p], srb, k.x);
              ga[4 * row + p] = wr_premult_over_pair(ga[4 * row + p], sga, k.x);
            }
          }
          dirty = true;
        }
      }
    }
  }
  if (dirty) {
    // rows past the target height exist in the allocation (textures are padded to
    // whole tiles), so both rows can be stored unconditionally
    *(uint4*)p0 = make_uint4(rb[0] | (ga[0] << 8), rb[1] | (ga[1] << 8), rb[2] | (ga[2] << 8), rb[3] | (ga[3] << 8));
    *(uint4*)p1 = make_uint4(rb[4] | (ga[4] << 8), rb[5] | (ga[5] << 8), rb[6] | (ga[6] << 8), rb[7] | (ga[7] << 8));
  }
}

// ---- shallow batches of plain solid quads: the streaming variant ---------------------------------------
// With a handful of layers the pass is a read-modify-write of the target at HBM speed and the tile
// machinery above (classification, compaction, three barriers per chunk, one tile in flight per CTA) is
// pure latency.  Here every thread owns 2 x 4 pixels (two 16-byte accesses in flight), the <= FLAT_MAX
// commands sit in shared memory, and a thread walks them in batch order testing coverage per pixel group —
// the classic elementwise shape; the grid covers the batch's bounding box only.  Same blend arithmetic.
#define FLAT_MAX 32
#define FLAT_THREADS 256
__global__ void __launch_bounds__(FLAT_THREADS) wr_raster_solid_flat(RasterArgs a) {
  __shared__ int4 rect[FLAT_MAX];
  __shared__ uint4 col[FLAT_MAX];
  wr_pdl_launch_dependents();
  wr_pdl_wait();
  const BatchInfo bi = *a.info;
  if (!bi.simple) return;  // mixed batch → generic kernel
  if (threadIdx.x < a.n) {
    const CmdHot c = a.hot[threadIdx.x];
    rect[threadIdx.x] = make_int4(c.x0, c.x1 > c.x0 ? c.x1 : c.x0, c.y0, c.y1);
    const uint32_t srb = (uint32_t)c.col[0] | ((uint32_t)c.col[2] << 16), sga = (uint32_t)c.col[1] | ((uint32_t)c.col[3] << 16);
    col[threadIdx.x] = make_uint4(255u - c.col[3], srb, sga, 0u);
  }
  __syncthreads();
  // the bounding box in units of 4 pixels x 2 rows
  const int gx0 = max(bi.bx0, 0) >> 2, gx1 = (min(bi.bx1, a.tgt.w) + 3) >> 2;
  const int gy0 = max(bi.by0, 0) >> 1, gy1 = (min(bi.by1, a.tgt.h) + 1) >> 1;
  const int gw = gx1 - gx0, gh = gy1 - gy0;
  if (gw <= 0 || gh <= 0) return;
  const long long total = (long long)gw * gh;
  for (long long g = (long long)blockIdx.x * FLAT_THREADS + threadIdx.x; g < total; g += (long long)gridDim.x * FLAT_THREADS) {
    const int x = (gx0 + (int)(g % gw)) * 4, y = (gy0 + (int)(g / gw)) * 2;
    uint4* p0 = (uint4*)(a.tgt.color + (size_t)y * a.tgt.color_pitch + (size_t)x * 4);
    uint4* p1 = (uint4*)(a.tgt.color + (size_t)(y + 1) * a.tgt.color_pitch + (size_t)x * 4);
    const uint4 v0 = *p0, v1 = *p1;  // (rows and columns past the target exist in the padded allocation)
    uint32_t px[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
    bool dirty = false;
    for (int i = 0; i < a.n; i++) {
      const int4 r = rect[i];
      if (r.y <= x || r.x >= x + 4 || r.w <= y || r.z >= y + 2) continue;
      const uint4 k = col[i];
#pragma unroll
      for (int q = 0; q < 8; q++) {
        const int xx = x + (q & 3), yy = y + (q >> 2);
        if (xx >= r.x && xx < r.y && yy >= r.z && yy < r.w) {
          const uint32_t rb = wr_premult_over_pair(px[q] & 0x00FF00FFu, k.y, k.x);
          const uint32_t ga = wr_premult_over_pair((px[q] >> 8) & 0x00FF00FFu, k.z, k.x);
          px[q] = rb | (ga << 8);
        }
      }
      dirty = true;
    }
    if (dirty) {
      *p0 = make_uint4(px[0], px[1], px[2], px[3]);
      *p1 = make_uint4(px[4], px[5], px[6], px[7]);
    }
  }
}

// ---- the lookup tables of a solid batch (fold.cuh) -----------------------------------------------------
// WR_FOLD_CTAS CTAs; warp w of CTA b folds segment b * WR_FOLD_SEGS + w of the command list over the 256
// inputs (lane l holds inputs 8l .. 8l+7 of all four channels as 16-bit lane pairs and applies the tile
// kernel's blend to them).  Each CTA composes its segment tables into a partial table; the last CTA to
// finish (a ticket in BatchInfo: no CTA ever waits for another) composes the partial tables in batch order.
// The work is n x 512 lane-pair multiply-adds and as many byte permutes: on one SM's integer pipes
// (64 per clock) 16 clocks per command: 8 us for config B's 1000 layers on one CTA; spread over 8 SMs, 1 us.
// Returns at once unless the batch is simple and a whole tile lies inside the common cover, the only place
// wr_raster_solid_premult reads the tables.
#define FOLD_THREADS (WR_FOLD_SEGS * 32)
static_assert(FOLD_THREADS == WR_FOLD_ENTRIES, "wr_fold_solid composes one table entry per thread");
static_assert(FAST_THREADS * 8 == WR_FOLD_ENTRIES, "wr_raster_solid_premult loads the tables 8 bytes per thread");

template <bool VALID>
__device__ __forceinline__ void wr_fold_warp(const CmdHot* hot, int s0, int s1, uint32_t* rb, uint32_t* ga) {
  const int lane = threadIdx.x & 31;
  for (int base = s0; base < s1; base += 32) {
    // 32 commands per round, loaded one per lane and handed to the whole warp by shuffles
    uint4 k = make_uint4(0, 0, 0, 0);
    bool keep = false;
    if (base + lane < s1) {
      const CmdHot c = hot[base + lane];
      keep = c.x1 > c.x0;  // what the tile kernel keeps: commands that draw nothing stay identity
      k = wr_solid_consts(c);
    }
    unsigned m = __ballot_sync(0xFFFFFFFFu, keep);
    while (m) {
      const int src = __ffs((int)m) - 1;
      m &= m - 1;
      wr_fast_blend8<VALID>(rb, ga, __shfl_sync(0xFFFFFFFFu, k.x, src), __shfl_sync(0xFFFFFFFFu, k.y, src),
                            __shfl_sync(0xFFFFFFFFu, k.z, src));
    }
  }
}

static_assert(WR_FOLD_CTAS * WR_FOLD_ENTRIES == FOLD_THREADS * 8, "the last CTA loads the partial tables 8 bytes per thread");

__global__ void __launch_bounds__(FOLD_THREADS) wr_fold_solid(RasterArgs a) {
  __shared__ __align__(16) uint8_t segs[WR_FOLD_SEGS * WR_FOLD_ENTRIES];
  __shared__ int s_last;
  wr_pdl_launch_dependents();
  wr_pdl_wait();
  const BatchInfo bi = *a.info;
  const int4 cov = wr_cover_tiles(bi, a.tgt);
  if (!bi.simple || cov.z <= cov.x || cov.w <= cov.y) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nseg = wr_fold_nseg(a.n), seg0 = blockIdx.x * WR_FOLD_SEGS;
  if (seg0 + warp < nseg) {
    int s0, s1;
    wr_fold_segment(a.n, nseg, seg0 + warp, &s0, &s1);
    uint32_t rb[8], ga[8];
    wr_fold_init(rb, ga, lane * 8);
    if (bi.premul_valid) wr_fold_warp<true>(a.hot, s0, s1, rb, ga);
    else wr_fold_warp<false>(a.hot, s0, s1, rb, ga);
    wr_fold_store(rb, ga, lane * 8, segs + warp * WR_FOLD_ENTRIES);
  }
  __syncthreads();
  uint8_t* part = a.fold + WR_FOLD_ENTRIES;  // the CTAs' partial tables, in CTA order
  part[blockIdx.x * WR_FOLD_ENTRIES + threadIdx.x] =
      wr_fold_compose(segs, min(max(nseg - seg0, 0), WR_FOLD_SEGS), threadIdx.x);
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(const_cast<int*>(&a.info->fold_ticket), 1) == WR_FOLD_CTAS - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  ((uint2*)segs)[threadIdx.x] = __ldcg((const uint2*)part + threadIdx.x);  // written by other CTAs: from L2
  __syncthreads();
  a.fold[threadIdx.x] = wr_fold_compose(segs, WR_FOLD_CTAS, threadIdx.x);
}

__global__ void __launch_bounds__(FAST_THREADS)
wr_raster_solid_premult(RasterArgs a) {
  __shared__ uint4 fa[FAST_CHUNK];
  __shared__ int4 fb[FAST_CHUNK];
  __shared__ int wsum[FAST_THREADS / 32];
  __shared__ __align__(16) uint8_t lut[WR_FOLD_ENTRIES];
  wr_pdl_launch_dependents();
  wr_pdl_wait();
  const BatchInfo bi = *a.info;
  if (!bi.simple) return;  // mixed batch → generic kernel
  // tiles of the batch's bounding box (clamped to the target)
  const int bx0 = max(bi.bx0, 0) / WRCU_TILE_W, by0 = max(bi.by0, 0) / WRCU_TILE_H;
  const int bx1 = (min(bi.bx1, a.tgt.w) + WRCU_TILE_W - 1) / WRCU_TILE_W;
  const int by1 = (min(bi.by1, a.tgt.h) + WRCU_TILE_H - 1) / WRCU_TILE_H;
  const int nx = bx1 - bx0, n_tiles = nx * (by1 - by0);
  if (nx <= 0 || n_tiles <= 0) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  auto tile_px = [&](int t, int row) {  // this thread's 16 bytes of row `row` (0 / 1 → tile rows warp, warp + 4)
    const int tx0 = (bx0 + t % nx) * WRCU_TILE_W, ty0 = (by0 + t / nx) * WRCU_TILE_H;
    return (uint4*)(a.tgt.color + (size_t)(ty0 + warp + 4 * row) * a.tgt.color_pitch + (size_t)(tx0 + lane * 4) * 4);
  };
  int t = blockIdx.x;
  uint4 n0 = make_uint4(0, 0, 0, 0), n1 = n0;
  if (t < n_tiles) { n0 = *tile_px(t, 0); n1 = *tile_px(t, 1); }
  // Tiles wholly inside the common cover take the fold's tables (when wr_fold_solid ran ahead of this kernel).
  // Their tile range stays in shared memory and is re-read per tile: held in registers through the tile loop
  // it takes the kernel from 72 to 80 registers, one resident CTA per SM fewer.
  __shared__ int s_cov[4];
  {
    const int4 c = a.fold ? wr_cover_tiles(bi, a.tgt) : make_int4(0, 0, 0, 0);
    if (threadIdx.x == 0) { s_cov[0] = c.x; s_cov[1] = c.y; s_cov[2] = c.z; s_cov[3] = c.w; }
    if (c.z > c.x && c.w > c.y) ((uint2*)lut)[threadIdx.x] = ((const uint2*)a.fold)[threadIdx.x];
  }
  __syncthreads();
  const volatile int* cov = s_cov;
  for (; t < n_tiles; t += gridDim.x) {
    const uint4 v0 = n0, v1 = n1;
    const int tn = t + gridDim.x;
    if (tn < n_tiles) { n0 = *tile_px(tn, 0); n1 = *tile_px(tn, 1); }  // next tile: issued now, used next iteration
    const int tx = bx0 + t % nx, ty = by0 + t / nx;
    if (tx >= cov[0] && tx < cov[2] && ty >= cov[1] && ty < cov[3]) {
      // every command of the batch covers this tile: the layers are the tables (no chunk classification)
      *tile_px(t, 0) = make_uint4(wr_fold_px(lut, v0.x), wr_fold_px(lut, v0.y), wr_fold_px(lut, v0.z), wr_fold_px(lut, v0.w));
      *tile_px(t, 1) = make_uint4(wr_fold_px(lut, v1.x), wr_fold_px(lut, v1.y), wr_fold_px(lut, v1.z), wr_fold_px(lut, v1.w));
      continue;
    }
    const int tx0 = tx * WRCU_TILE_W, ty0 = ty * WRCU_TILE_H;
    if (bi.premul_valid) wr_fast_tile<true>(a, tx0, ty0, fa, fb, wsum, v0, v1);
    else wr_fast_tile<false>(a, tx0, ty0, fa, fb, wsum, v0, v1);
  }
}
#endif  // !WRCU_HOSTEMU
