// setup_common.cuh — pieces of the reference's vertex stage shared by all
// kinds: data-table fetches (webrender/res/gpu_cache.glsl, gpu_buffer.glsl,
// render_task.glsl, transform.glsl) and draw_quad's screen-space set-up for
// screen-axis-aligned quads (swgl/src/rasterize.h:1549-1632, 783-941).
//
// Compiled with -fmad=false: every float expression below is evaluated as
// written, in IEEE fp32, in the same order as the GLSL / glsl.h source, so
// device rects and interpolants match the g++ build of SWGL bit for bit.
#pragma once
#include "blend.cuh"
#include "cmd.cuh"
#include "repeat_add.cuh"
#include "wrcu_internal.h"

#define WR_WIDE_TILES 64

struct SetupArgs {
  FrameTablesDev tabs;
  TargetDev tgt;
  const uint8_t* instances;
  int stride;
  int n;
  CmdHot* hot;
  CmdCold* cold;
  BatchInfo* info;
  BatchInfo* info_next;  // the NEXT batch's record, reset by this batch's setup kernel (ring of 4)
  // bitmask bins (large batches): bit i of tile_mask[tile * bin_words + i/32] = command i touches the tile;
  // commands covering more than WR_WIDE_TILES tiles set their bit in wide_mask instead
  uint32_t* tile_mask;
  uint32_t* wide_mask;
  // bit t of tile_any = some command's bit is set in tile t's mask; word any_words = a wide command exists.
  // Lets the raster kernel's tile scheduler pass over empty tiles with one load each.
  uint32_t* tile_any;
  int any_words;
  int bin_words, bin_tiles_x;
  int* err_counter;
  int blend_enabled;
  uint32_t features;
  int kind;  // WRCU_KIND_* (setup functions shared by several kinds)
  float* row_tab;   // row-table pool (see CmdCold::row_off), row_cap floats
  int row_cap;
  TexView color0;
  TexView color1;
  TexView color2;
  TexView clip_mask;
  const TexView* tex_list;  // wrcu_draw_composite_tiles: sColor0 of instance i (nullptr: color0 for all)
  int warp_per_inst;        // small batches: one WARP per instance (lane 0 runs the vertex stage, the warp fills its row table)
  int depth_runs;           // depth test on and the kind's shading depends on where passing runs start:
  int fail_cap;             //   commands get a failing-sample bitmap (CmdCold::fail_off) from a pool of fail_cap words
  int copy_ok;              // composite: blend off or premultiplied-alpha over, no depth → copy class possible
  int persp_ok;             // the kind's fragment stage is built for draw_perspective (per-sample 1/w); others are rejected
  int* pool_ctr;            // [0] floats of the row-table pool, [1] words of the depth-run bitmap pool handed out so far
                            // (shared by every batch of a submission: wrcu_api.cu flush_pending)
};

// A setup kernel = one thread per instance running <name>_one.  Under the host
// emulation (tests only) the same function is called in a plain loop.
WRD void wr_reset_batch_info(BatchInfo* info) {
  info->bx0 = 0x7fffffff; info->by0 = 0x7fffffff;
  info->bx1 = -0x7fffffff; info->by1 = -0x7fffffff;
  info->unsupported = 0;
  info->simple = 1;
  info->premul_valid = 1;
  info->tile_counter = 0;
  info->n_ordered = 0;
  info->all_copy = 1;
  info->glyph_ticket = 0;
  info->n_noncopy = 0;
  info->cx0 = -0x7fffffff; info->cy0 = -0x7fffffff;
  info->cx1 = 0x7fffffff; info->cy1 = 0x7fffffff;
  info->fold_ticket = 0;
}
// Each setup kernel also re-arms the per-batch record the NEXT draw will use
// (records rotate through a ring of 4; the one after the current was last read
// three draws ago), so no separate initialisation launch is needed per draw.
// Row tables.  The raster kernel needs, for every (command,row) it touches, the edge
// interpolants of that row — running sums down the quad's edges (rasterize.h:880-930).  A
// full-height quad is touched by ~30 tiles per row, each of which would otherwise re-walk
// the sums (wr_repeat_add, O(binades)); instead the setup kernel writes them once: after its
// 32 instances are emitted, the warp fills the table of each in turn, lanes split over the
// 2N edge sums x blocks of rows (a block starts with one wr_repeat_add, then plain additions —
// the reference's own sequence).
// tall commands: the 32 lanes split one command's 2N edge sums x blocks of rows
WRD_SHARED void wr_fill_row_table(const SetupArgs& a, int cidx, int lane) {
  const CmdHot c = a.hot[cidx];
  const CmdCold& k = a.cold[cidx];
  const int E = 2 * k.row_n, rows = c.y1 - c.y0;
  if (E <= 0 || E > 32) return;
  const int nblk = min(32 / E, (rows + 255) / 256);
  const int e = lane % E, blk = lane / E;
  if (blk >= nblk) return;
  const int per = (rows + nblk - 1) / nblk;
  const int r0 = blk * per, r1 = min(rows, r0 + per);
  if (r0 >= r1) return;
  const int i = e >> 1;
  const float top = (e & 1) ? k.i_rt[i] : k.i_lt[i], bot = (e & 1) ? k.i_rb[i] : k.i_lb[i];
  const float sl = __fmul_rn(__fsub_rn(bot, top), k.yscale);
  const float dy = __fsub_rn((float)c.y0 + 0.5f, k.yt);
  float v = wr_repeat_add(__fadd_rn(top, __fmul_rn(dy, sl)), sl, r0);
  float* t = a.row_tab + k.row_off + e;
  for (int r = r0; r < r1; r++) {
    t[(size_t)r * E] = v;
    v = __fadd_rn(v, sl);
  }
}
// short commands: one lane walks one edge sum of one command from its first row (plain additions,
// the reference's own sequence); 32 / 2N commands are filled at once
WRD_SHARED void wr_fill_row_edge(const SetupArgs& a, int cidx, int e) {
  const CmdHot c = a.hot[cidx];
  const CmdCold& k = a.cold[cidx];
  const int E = 2 * k.row_n, rows = c.y1 - c.y0;
  const int i = e >> 1;
  const float top = (e & 1) ? k.i_rt[i] : k.i_lt[i], bot = (e & 1) ? k.i_rb[i] : k.i_lb[i];
  const float sl = __fmul_rn(__fsub_rn(bot, top), k.yscale);
  const float dy = __fsub_rn((float)c.y0 + 0.5f, k.yt);
  float v = __fadd_rn(top, __fmul_rn(dy, sl));
  float* t = a.row_tab + k.row_off + e;
  for (int r = 0; r < rows; r++) {
    t[(size_t)r * E] = v;
    v = __fadd_rn(v, sl);
  }
}
#define WR_ROW_TAB_TALL 512
#ifdef WRCU_HOSTEMU
#define WR_SETUP_KERNEL(name)                                     \
  static void name##_block(const SetupArgs& a, int) {             \
    if (a.info_next) wr_reset_batch_info(a.info_next);            \
    for (int i = 0; i < a.n; i++) {                               \
      name##_one(a, i);                                           \
      if (a.cold[i].row_off >= 0 && a.cold[i].row_n > 0)          \
        for (int e = 0; e < 2 * a.cold[i].row_n; e++) wr_fill_row_edge(a, i, e); \
    }                                                             \
  }
#else
WRD void wr_fill_row_tables_warp(const SetupArgs& a, int idx) {
  const int lane = threadIdx.x & 31, wbase = idx - lane;
  const bool has = idx < a.n && a.cold[idx].row_off >= 0 && a.cold[idx].row_n > 0;
  unsigned m = __ballot_sync(0xFFFFFFFFu, has);
  if (!m) return;
  const int myE = has ? 2 * a.cold[idx].row_n : 0;
  const int myRows = has ? (int)a.hot[idx].y1 - (int)a.hot[idx].y0 : 0;
  const int E0 = __shfl_sync(0xFFFFFFFFu, myE, __ffs((int)m) - 1);
  unsigned mshort = __ballot_sync(0xFFFFFFFFu, has && myE == E0 && myRows <= WR_ROW_TAB_TALL);
  unsigned mlong = m & ~mshort;
  const int G = 32 / E0, slot = lane / E0, e = lane % E0;
  while (mshort) {
    const unsigned src = __fns(mshort, 0, slot + 1);  // lane of the slot-th pending command
    if (slot < G && src < 32u) wr_fill_row_edge(a, wbase + (int)src, e);
    for (int i = 0; i < G && mshort; i++) mshort &= mshort - 1;
  }
  while (mlong) {
    const int src = __ffs((int)mlong) - 1;
    mlong &= mlong - 1;
    wr_fill_row_table(a, wbase + src, lane);
  }
}
// One command's row table by a whole warp: the 2N edge sums x blocks of >= 16 rows spread over the lanes.
WRD_SHARED void wr_fill_row_table_spread(const SetupArgs& a, int cidx, int lane) {
  const CmdHot c = a.hot[cidx];
  const CmdCold& k = a.cold[cidx];
  const int E = 2 * k.row_n, rows = c.y1 - c.y0;
  if (E <= 0 || E > 32) return;
  const int nblk = max(1, min(32 / E, rows / 16));
  const int e = lane % E, blk = lane / E;
  if (blk >= nblk) return;
  const int per = (rows + nblk - 1) / nblk;
  const int r0 = blk * per, r1 = min(rows, r0 + per);
  if (r0 >= r1) return;
  const int i = e >> 1;
  const float top = (e & 1) ? k.i_rt[i] : k.i_lt[i], bot = (e & 1) ? k.i_rb[i] : k.i_lb[i];
  const float sl = __fmul_rn(__fsub_rn(bot, top), k.yscale);
  const float dy = __fsub_rn((float)c.y0 + 0.5f, k.yt);
  float v = wr_repeat_add(__fadd_rn(top, __fmul_rn(dy, sl)), sl, r0);
  float* t = a.row_tab + k.row_off + e;
  for (int r = r0; r < r1; r++) {
    t[(size_t)r * E] = v;
    v = __fadd_rn(v, sl);
  }
}
// Small batches (SetupArgs::warp_per_inst: what a page is mostly made of — a few instances per batch) are
// latency, not throughput: one warp per instance, so the instances' dependent table fetches overlap and
// each row table is filled by 32 lanes instead of one.
// name##_block: the kernel body for the batch's thread `idx` (CTA-relative to the batch's first block), so that
// one launch can run the set-up of MANY batches (wr_setup_multi, wrcu_api.cu): a page is ~150 batches of a few
// instances, and a launch per batch made its set-up latency (~10 us: a chain of table fetches) the frame time.
#define WR_SETUP_KERNEL(name)                                                  \
  __device__ __noinline__ void name##_block(const SetupArgs& a, int idx) {     \
    if (idx == 0 && a.info_next) wr_reset_batch_info(a.info_next);             \
    if (a.warp_per_inst) {                                                     \
      const int lane = threadIdx.x & 31;                                       \
      idx >>= 5;                                                               \
      if (idx >= a.n) return;                                                  \
      if (lane == 0) name##_one(a, idx);                                       \
      __syncwarp();                                                            \
      if (a.cold[idx].row_off >= 0 && a.cold[idx].row_n > 0) wr_fill_row_table_spread(a, idx, lane); \
      return;                                                                  \
    }                                                                          \
    if (idx < a.n) name##_one(a, idx);                                         \
    __syncwarp();                                                              \
    wr_fill_row_tables_warp(a, idx);                                           \
  }
#endif

WRD float4 wr_fetch(const float4* t, int n, int addr) {
  if (n <= 0) return make_float4(0, 0, 0, 0);
  addr = min(max(addr, 0), n - 1);
  return __ldg(t + addr);
}
WRD int4 wr_fetchi(const int4* t, int n, int addr) {
  if (n <= 0) return make_int4(0, 0, 0, 0);
  addr = min(max(addr, 0), n - 1);
  return __ldg(t + addr);
}

struct DevTransform {
  float m[16], inv_m[16];
  bool is_axis_aligned;
};

WRD DevTransform wr_fetch_transform(const FrameTablesDev& t, int id) {
  DevTransform r;
  r.is_axis_aligned = (id >> 23) == 0;
  int index = id & 0x007fffff;
  for (int i = 0; i < 4; i++) {
    float4 a = wr_fetch(t.transforms, t.n_transforms, index * 8 + i);
    float4 b = wr_fetch(t.transforms, t.n_transforms, index * 8 + 4 + i);
    r.m[4 * i + 0] = a.x; r.m[4 * i + 1] = a.y; r.m[4 * i + 2] = a.z; r.m[4 * i + 3] = a.w;
    r.inv_m[4 * i + 0] = b.x; r.inv_m[4 * i + 1] = b.y; r.inv_m[4 * i + 2] = b.z; r.inv_m[4 * i + 3] = b.w;
  }
  return r;
}

// mat4 * vec4 with glsl.h's evaluation order (glsl.h:2581-2588)
WRD float4 wr_mat_mul(const float* m, float4 v) {
  float4 u;
  u.x = m[0] * v.x + m[4] * v.y + m[8] * v.z + m[12] * v.w;
  u.y = m[1] * v.x + m[5] * v.y + m[9] * v.z + m[13] * v.w;
  u.z = m[2] * v.x + m[6] * v.y + m[10] * v.z + m[14] * v.w;
  u.w = m[3] * v.x + m[7] * v.y + m[11] * v.z + m[15] * v.w;
  return u;
}

struct DevPictureTask {
  float tx0, ty0, tx1, ty1;  // task_rect
  float device_pixel_scale;
  float ox, oy;  // content_origin
};
WRD DevPictureTask wr_fetch_picture_task(const FrameTablesDev& t, int address) {
  float4 a = wr_fetch(t.render_tasks, t.n_render_tasks, address * 2);
  float4 b = wr_fetch(t.render_tasks, t.n_render_tasks, address * 2 + 1);
  return DevPictureTask{a.x, a.y, a.z, a.w, b.x, b.y, b.z};
}

WRD int wr_round_i(float v) { return (int)floorf(v + 0.5f); }

// Output of a kind's vertex stage for one instance.
struct QuadOut {
  float4 pos[4];        // gl_Position per lane (lanes = unit quad corners 0,1,3,2)
  float interp[4][WR_NI];  // up to WR_NI interpolated floats per lane
  int n_interp;
  uint32_t flags;       // CMD_* set by the vertex stage
  int aa_edge_mask;     // swgl_antiAlias edges (lane-index bits)
  // swgl_clipMask(offset, bb_origin, bb_size)
  int cm_off[2], cm_bb[4];
  uint16_t col[4];
};

// ---- draw_perspective (rasterize.h:1422-1545): frustum clipping, projection, edge walk ----------------
#ifdef WRCU_HOSTEMU
#define WRD_NOINLINE static
#else
#define WRD_NOINLINE __device__ __noinline__
#endif
// clip_side<AXIS> (rasterize.h:1288-1420): clip the convex polygon against both planes -w <= c <= w of
// one axis; intersection points get interpolated attributes, the AA edge mask follows the new edges.
WRD_NOINLINE int wr_clip_side(int axis, int nump, const float (*p)[4], const float (*ip)[WR_NI], float (*op)[4],
                              float (*oip)[WR_NI], int* edge_mask_io) {
  enum { POSITIVE = 1, NEGATIVE = 2 };
  int numClip = 0;
  int edgeMask = *edge_mask_io, outEdgeMask = 0;
  float prev[4] = {p[nump - 1][0], p[nump - 1][1], p[nump - 1][2], p[nump - 1][3]};
  float prevI[WR_NI];
  for (int i = 0; i < WR_NI; i++) prevI[i] = ip[nump - 1][i];
  float prevCoord = prev[axis];
  int prevMask = (prevCoord < -prev[3] ? NEGATIVE : 0) | (prevCoord > prev[3] ? POSITIVE : 0);
  for (int i = 0; i < nump; i++, edgeMask >>= 1) {
    float cur[4] = {p[i][0], p[i][1], p[i][2], p[i][3]};
    float curI[WR_NI];
    for (int j = 0; j < WR_NI; j++) curI[j] = ip[i][j];
    const float curCoord = cur[axis];
    const int curMask = (curCoord < -cur[3] ? NEGATIVE : 0) | (curCoord > cur[3] ? POSITIVE : 0);
    if (!(curMask & prevMask)) {
      if (prevMask) {  // an edge that was outside crosses inside
        if (numClip >= nump + 2) return 0;
        const float prevSide = (prevMask & NEGATIVE) && (!(prevMask & POSITIVE) ||
                                                         prevCoord * (cur[3] - prev[3]) < prev[3] * (curCoord - prevCoord))
                                   ? -1.0f : 1.0f;
        const float prevDist = prevCoord - prevSide * prev[3];
        const float curDist = curCoord - prevSide * cur[3];
        float kk = prevDist / (prevDist - curDist);
        float cl[4];
        for (int j = 0; j < 4; j++) cl[j] = prev[j] + (cur[j] - prev[j]) * kk;
        if (prevSide * cl[axis] > cl[3]) {
          kk = nextafterf(kk, 1.0f);
          for (int j = 0; j < 4; j++) cl[j] = prev[j] + (cur[j] - prev[j]) * kk;
        }
        for (int j = 0; j < 4; j++) op[numClip][j] = cl[j];
        for (int j = 0; j < WR_NI; j++) oip[numClip][j] = prevI[j] + (curI[j] - prevI[j]) * kk;
        numClip++;
      }
      if (curMask) {  // an edge that was inside crosses outside
        if (numClip >= nump + 2) return 0;
        const float curSide = (curMask & POSITIVE) && (!(curMask & NEGATIVE) ||
                                                       prevCoord * (cur[3] - prev[3]) < prev[3] * (curCoord - prevCoord))
                                  ? 1.0f : -1.0f;
        const float prevDist = prevCoord - curSide * prev[3];
        const float curDist = curCoord - curSide * cur[3];
        float kk = prevDist / (prevDist - curDist);
        float cl[4];
        for (int j = 0; j < 4; j++) cl[j] = prev[j] + (cur[j] - prev[j]) * kk;
        if (curSide * cl[axis] > cl[3]) {
          kk = nextafterf(kk, 0.0f);
          for (int j = 0; j < 4; j++) cl[j] = prev[j] + (cur[j] - prev[j]) * kk;
        }
        for (int j = 0; j < 4; j++) op[numClip][j] = cl[j];
        for (int j = 0; j < WR_NI; j++) oip[numClip][j] = prevI[j] + (curI[j] - prevI[j]) * kk;
        outEdgeMask |= (edgeMask & 1) << numClip;
        numClip++;
      }
    }
    if (!curMask) {
      if (numClip >= nump + 2) return 0;
      for (int j = 0; j < 4; j++) op[numClip][j] = cur[j];
      for (int j = 0; j < WR_NI; j++) oip[numClip][j] = curI[j];
      outEdgeMask |= (edgeMask & 1) << numClip;
      numClip++;
    }
    for (int j = 0; j < 4; j++) prev[j] = cur[j];
    for (int j = 0; j < WR_NI; j++) prevI[j] = curI[j];
    prevCoord = curCoord;
    prevMask = curMask;
  }
  *edge_mask_io = outEdgeMask;
  return numClip;
}

// draw_perspective + the set-up part of draw_perspective_spans for one instance whose vertices differ in w.
// Writes the polygon into the row-table pool; fills the hot rect (bounding box of the rows / columns the
// walk can touch) and k.row_off.  Returns 1 = drawn, 0 = nothing to draw, -1 = cannot (pool exhausted).
WRD_NOINLINE int wr_emit_persp(const SetupArgs& a, const QuadOut& q, uint32_t flags, float cx0, float cy0, float cx1,
                               float cy1, CmdHot& h, CmdCold& k) {
  float pc[WR_PP_MAXV][4], ic[WR_PP_MAXV][WR_NI];
  float pt[WR_PP_MAXV][4], it[WR_PP_MAXV][WR_NI];
  int nump = 4;
  int aa_mask = q.aa_edge_mask;
  for (int i = 0; i < 4; i++) {
    pc[i][0] = q.pos[i].x; pc[i][1] = q.pos[i].y; pc[i][2] = q.pos[i].z; pc[i][3] = q.pos[i].w;
    for (int j = 0; j < WR_NI; j++) ic[i][j] = q.interp[i][j];
  }
  const float scx = (float)a.tgt.vp[2] * 0.5f, scy = (float)a.tgt.vp[3] * 0.5f, scz = 1.0f * 0.5f;
  const float ofx = (float)a.tgt.vp[0] + scx, ofy = (float)a.tgt.vp[1] + scy, ofz = 0.0f + scz;
  bool inside = true;
  for (int i = 0; i < 4; i++) inside = inside && (pc[i][2] > -pc[i][3] && pc[i][2] < pc[i][3]);
  if (!inside) {
    for (int i = 0; i < 4; i++) {
      for (int j = 0; j < 4; j++) pt[i][j] = pc[i][j];
      for (int j = 0; j < WR_NI; j++) it[i][j] = ic[i][j];
    }
    nump = wr_clip_side(2, nump, pt, it, pc, ic, &aa_mask);
    if (nump < 3) return 0;
    for (int i = 0; i < nump; i++) {
      if (pc[i][3] <= 0.0f) {
        nump = wr_clip_side(0, nump, pc, ic, pt, it, &aa_mask);
        if (nump < 3) return 0;
        nump = wr_clip_side(1, nump, pt, it, pc, ic, &aa_mask);
        if (nump < 3) return 0;
        break;
      }
    }
  }
  for (int i = 0; i < nump; i++) {
    const float w = 1.0f / pc[i][3];
    if (isfinite(w)) {
      pc[i][0] = pc[i][0] * w * scx + ofx;
      pc[i][1] = pc[i][1] * w * scy + ofy;
      pc[i][2] = pc[i][2] * w * scz + ofz;
      pc[i][3] = w;
    } else {
      pc[i][0] = pc[i][1] = pc[i][2] = pc[i][3] = 0.0f;
    }
  }
  // ClipRect::overlaps
  int sides = 0;
  for (int i = 0; i < nump; i++) {
    sides |= pc[i][0] < cx1 ? (pc[i][0] > cx0 ? 1 | 2 : 1) : 2;
    sides |= pc[i][1] < cy1 ? (pc[i][1] > cy0 ? 4 | 8 : 4) : 8;
  }
  if (sides != 0xF) return 0;
  if (!a.row_tab) return -1;
  const int off = atomicAdd(a.pool_ctr, WR_PP_FLOATS);
  if (off < 0 || off + WR_PP_FLOATS > a.row_cap) return -1;
  PerspPoly& P = *(PerspPoly*)(a.row_tab + off);
  P.nump = nump;
  P.aa_mask = aa_mask;
  P.clip[0] = cx0; P.clip[1] = cy0; P.clip[2] = cx1; P.clip[3] = cy1;
  for (int i = 0; i < nump; i++) {
    P.px[i] = pc[i][0]; P.py[i] = pc[i][1]; P.pz[i] = pc[i][2]; P.pw[i] = pc[i][3];
    for (int j = 0; j < WR_NI; j++) P.interp[i][j] = ic[i][j];
  }
  // vertex selection (rasterize.h:1070-1110)
  int top = 0;
  for (int i = 1; i < nump; i++)
    if (P.py[i] < P.py[top]) top = i;
  int l0i = top;
  for (int i = top + 1; i < nump && P.py[i] == P.py[top]; i++) l0i = i;
  if (l0i == nump - 1)
    for (int i = 0; i <= top && P.py[i] == P.py[top]; i++) l0i = i;
  int r0i = top;
  for (int i = top - 1; i >= 0 && P.py[i] == P.py[top]; i--) r0i = i;
  if (r0i == 0)
    for (int i = nump - 1; i >= top && P.py[i] == P.py[top]; i--) r0i = i;
#define WR_PP_NEXT(i) ((i) + 1 < nump ? (i) + 1 : 0)
#define WR_PP_PREV(i) ((i) - 1 >= 0 ? (i) - 1 : nump - 1)
  int l1i = WR_PP_NEXT(l0i), r1i = WR_PP_PREV(r0i);
  const bool aa = (flags & CMD_AA) != 0;
  const float aaR = aa ? 0.0f : 0.5f;
  float gy = floorf(wr_max(wr_min(P.py[l0i], cy1), cy0) + aaR) + 0.5f;
  int row = (int)(gy - 0.5f);
  {
    const float perp = (P.px[l1i] - P.px[l0i]) * (P.py[r1i] - P.py[r0i]) - (P.py[l1i] - P.py[l0i]) * (P.px[r1i] - P.px[r0i]);
    P.flipped = (P.px[l0i] > P.px[r0i] || (P.px[l0i] == P.px[r0i] && perp > 0.0f)) ? 1 : 0;
  }
  int lrow = row, rrow = row, n_ev = 0, first_row = row, last_row = row - 1;
  bool overflow = false;
#define WR_PP_EVENT()                                                                              \
  do {                                                                                             \
    if (n_ev < WR_PP_MAXEV) {                                                                      \
      P.ev[n_ev].row = (short)row; P.ev[n_ev].lrow = (short)lrow; P.ev[n_ev].rrow = (short)rrow;   \
      P.ev[n_ev].l0 = (uint8_t)l0i; P.ev[n_ev].l1 = (uint8_t)l1i;                                  \
      P.ev[n_ev].r0 = (uint8_t)r0i; P.ev[n_ev].r1 = (uint8_t)r1i;                                  \
      n_ev++;                                                                                      \
    } else overflow = true;                                                                        \
  } while (0)
  WR_PP_EVENT();
  float checkY = wr_min(wr_min(P.py[l1i], P.py[r1i]), cy1);
  for (int guard = 0; guard < 40000; guard++) {
    if (gy > checkY) {
      if (gy > cy1) break;
      bool changed = false, done = false;
      if (gy > P.py[l1i]) {  // STEP_EDGE(y, l0i, l0, l1i, l1, NEXT_POINT, r1i)
        do {
          l0i = l1i;
          l1i = WR_PP_NEXT(l1i);
          if (l0i == r1i) { done = true; break; }
        } while (gy > P.py[l1i]);
        lrow = row;
        changed = true;
      }
      if (!done && gy > P.py[r1i]) {  // STEP_EDGE(y, r0i, r0, r1i, r1, PREV_POINT, l1i)
        do {
          r0i = r1i;
          r1i = WR_PP_PREV(r1i);
          if (r0i == l1i) { done = true; break; }
        } while (gy > P.py[r1i]);
        rrow = row;
        changed = true;
      }
      if (done) break;
      checkY = wr_min(ceilf(wr_min(P.py[l1i], P.py[r1i]) - aaR), cy1);
      if (changed) WR_PP_EVENT();
    }
    last_row = row;
    row++;
    gy = gy + 1.0f;
  }
#undef WR_PP_EVENT
#undef WR_PP_NEXT
#undef WR_PP_PREV
  if (overflow) return -1;
  if (last_row < first_row) return 0;
  P.n_ev = n_ev;
  float minx = P.px[0], maxx = P.px[0];
  for (int i = 1; i < nump; i++) { minx = wr_min(minx, P.px[i]); maxx = wr_max(maxx, P.px[i]); }
  const int gx0 = (int)floorf(wr_clamp(minx, cx0, cx1)), gx1 = (int)ceilf(wr_clamp(maxx, cx0, cx1));
  if (gx1 <= gx0) return 0;
  h.x0 = (short)gx0; h.x1 = (short)gx1; h.y0 = (short)first_row; h.y1 = (short)(last_row + 1);
  // no span shaders in the perspective path: every chunk is fragment_shader->run<true>() (rasterize.h:1262-1270)
  h.flags = (flags & ~CMD_SPAN_SOLID) | CMD_GENERAL | CMD_PERSP;
  h.z = 0x7FFFFFFFu;  // never an occluder candidate of the depth-run prepass; the depth test uses the per-sample z
  k.row_off = off;
  k.row_n = -1;
  return 1;
}

// draw_quad + the parts of draw_quad_spans that are per-instance constants for
// a quad whose screen edges are vertical/horizontal.  Writes hot/cold; returns
// false (and writes an empty command) when the instance draws nothing.
// Sets *unsupported when the quad needs the general edge walker (rotation or
// perspective), which this backend does not rasterise yet.
WRD_SHARED bool wr_emit_quad(const SetupArgs& a, int idx, const QuadOut& q, int* unsupported) {
  CmdHot h;
  h.x0 = h.y0 = h.x1 = h.y1 = 0;
  h.flags = 0;
  h.z = 0;
  h.col[0] = q.col[0]; h.col[1] = q.col[1]; h.col[2] = q.col[2]; h.col[3] = q.col[3];
  h.aa_left_end = h.aa_right_start = 0;
  h.cold = idx;
  CmdCold k;
  memset(&k, 0, sizeof k);
  k.row_off = -1;
  k.fail_off = -1;
  bool ok = false;
  do {
    const bool persp = q.pos[1].w != q.pos[0].w || q.pos[2].w != q.pos[0].w || q.pos[3].w != q.pos[0].w;
    float w = 1.0f / q.pos[0].w;
    if (!isfinite(w)) w = 0.0f;
    float px[4], py[4];
    for (int i = 0; i < 4; i++) {
      px[i] = (q.pos[i].x * w + 1) * 0.5f * (float)a.tgt.vp[2] + (float)a.tgt.vp[0];
      py[i] = (q.pos[i].y * w + 1) * 0.5f * (float)a.tgt.vp[3] + (float)a.tgt.vp[1];
    }
    uint32_t flags = a.blend_enabled ? q.flags : (q.flags & ~(CMD_MASK | CMD_AA | CMD_SPAN_SOLID));
    float cx0 = (float)a.tgt.cx0, cy0 = (float)a.tgt.cy0, cx1 = (float)a.tgt.cx1, cy1 = (float)a.tgt.cy1;
    if ((flags & CMD_MASK) && a.clip_mask.ptr == nullptr) {
      *unsupported = 1;  // clip task referenced but no sClipMask bound
      break;
    }
    if (flags & CMD_MASK) {
      int mx0 = max(q.cm_bb[0], 0), my0 = max(q.cm_bb[1], 0);
      int mx1 = min(q.cm_bb[0] + q.cm_bb[2], a.clip_mask.w);
      int my1 = min(q.cm_bb[1] + q.cm_bb[3], a.clip_mask.h);
      int cmx = q.cm_off[0] + a.tgt.vp[0], cmy = q.cm_off[1] + a.tgt.vp[1];
      mx0 += cmx; mx1 += cmx; my0 += cmy; my1 += cmy;
      cx0 = wr_max(cx0, (float)mx0); cy0 = wr_max(cy0, (float)my0);
      cx1 = wr_min(cx1, (float)mx1); cy1 = wr_min(cy1, (float)my1);
      k.mask_ptr = a.clip_mask.ptr;
      k.mask_pitch = a.clip_mask.pitch;
      k.cmx = (short)cmx;
      k.cmy = (short)cmy;
    }
    if (persp) {  // draw_perspective (rasterize.h:1422-1545)
      if (!a.persp_ok || (q.flags & CMD_CLIP_DIST) || a.tgt.fmt != WRCU_FMT_RGBA8) { *unsupported = 1; break; }
      const int r = wr_emit_persp(a, q, flags, cx0, cy0, cx1, cy1, h, k);
      if (r < 0) *unsupported = 1;
      ok = r > 0;
      break;
    }
    int sides = 0;
    for (int i = 0; i < 4; i++) {
      sides |= px[i] < cx1 ? (px[i] > cx0 ? 1 | 2 : 1) : 2;
      sides |= py[i] < cy1 ? (py[i] > cy0 ? 4 | 8 : 4) : 8;
    }
    if (sides != 0xF) break;
    float screenZ = (q.pos[0].z * w + 1) * 0.5f;
    if (screenZ < 0 || screenZ > 1) break;
    h.z = (uint32_t)(16777215.0f * screenZ);

    // vertex selection, rasterize.h:796-846
    int top = py[3] < py[2] ? (py[0] < py[1] ? (py[0] < py[3] ? 0 : 3) : (py[1] < py[3] ? 1 : 3))
                            : (py[0] < py[1] ? (py[0] < py[2] ? 0 : 2) : (py[1] < py[2] ? 1 : 2));
    int next = (top + 1) & 3, prev = (top + 3) & 3;
    int l0i, l1i, r0i, r1i;
    if (py[top] == py[next]) {
      l0i = next; l1i = (next + 1) & 3; r0i = top; r1i = prev;
    } else if (py[top] == py[prev]) {
      l0i = top; l1i = next; r0i = prev; r1i = (prev + 3) & 3;
    } else {
      l0i = r0i = top; l1i = next; r1i = prev;
    }
    // Screen-axis-aligned quads (both descending edges vertical, same y extent) get
    // a constant span; anything else keeps the full edge walk of draw_quad_spans.
    if (px[l0i] != px[l1i] || px[r0i] != px[r1i] || py[l0i] != py[r0i] || py[l1i] != py[r1i]) {
      const bool gaa = (flags & CMD_AA) != 0;
      const float aaR = gaa ? 0.0f : 0.5f;
      float gy = floorf(wr_max(wr_min(py[l0i], cy1), cy0) + aaR) + 0.5f;
      int row = (int)(gy - 0.5f);
      float gperp = (px[l1i] - px[l0i]) * (py[r1i] - py[r0i]) - (py[l1i] - py[l0i]) * (px[r1i] - px[r0i]);
      k.gflipped = (px[l0i] > px[r0i] || (px[l0i] == px[r0i] && gperp > 0.0f)) ? 1 : 0;
      k.gaa_mask = q.aa_edge_mask;
      for (int i = 0; i < 4; i++) { k.gpx[i] = px[i]; k.gpy[i] = py[i]; }
      k.gclip[0] = cx0; k.gclip[1] = cy0; k.gclip[2] = cx1; k.gclip[3] = cy1;
      int gl0 = l0i, gl1 = l1i, gr0 = r0i, gr1 = r1i, lrow = row, rrow = row;
      int n_ev = 0, first_row = row, last_row = row - 1;
      bool overflow = false;
#define WR_ADD_EVENT()                                                                             \
  do {                                                                                             \
    if (n_ev < 6) {                                                                                \
      k.gev[n_ev].row = (short)row; k.gev[n_ev].lrow = (short)lrow; k.gev[n_ev].rrow = (short)rrow; \
      k.gev[n_ev].l0 = (uint8_t)gl0; k.gev[n_ev].l1 = (uint8_t)gl1;                                \
      k.gev[n_ev].r0 = (uint8_t)gr0; k.gev[n_ev].r1 = (uint8_t)gr1;                                \
      n_ev++;                                                                                      \
    } else overflow = true;                                                                        \
  } while (0)
      WR_ADD_EVENT();
      float checkY = wr_min(wr_min(py[gl1], py[gr1]), cy1);
      for (int guard = 0; guard < 40000; guard++) {
        if (gy > checkY) {
          if (gy > cy1) break;
          bool changed = false, done = false;
          if (gy > py[gl1]) {  // STEP_EDGE(l.., NEXT_POINT, r1i)
            do {
              gl0 = gl1;
              gl1 = (gl1 + 1) & 3;
              if (gl0 == gr1) { done = true; break; }
            } while (gy > py[gl1]);
            lrow = row;
            changed = true;
          }
          if (!done && gy > py[gr1]) {  // STEP_EDGE(r.., PREV_POINT, l1i)
            do {
              gr0 = gr1;
              gr1 = (gr1 + 3) & 3;
              if (gr0 == gl1) { done = true; break; }
            } while (gy > py[gr1]);
            rrow = row;
            changed = true;
          }
          if (done) break;
          checkY = wr_min(ceilf(wr_min(py[gl1], py[gr1]) - aaR), cy1);
          if (changed) WR_ADD_EVENT();
        }
        last_row = row;
        row++;
        gy = gy + 1.0f;
      }
#undef WR_ADD_EVENT
      if (overflow) { *unsupported = 1; break; }
      if (last_row < first_row) break;
      k.gn_ev = n_ev;
      float minx = wr_min(wr_min(px[0], px[1]), wr_min(px[2], px[3]));
      float maxx = wr_max(wr_max(px[0], px[1]), wr_max(px[2], px[3]));
      int gx0 = (int)floorf(wr_clamp(minx, cx0, cx1)), gx1 = (int)ceilf(wr_clamp(maxx, cx0, cx1));
      if (gx1 <= gx0) break;
      h.x0 = (short)gx0; h.x1 = (short)gx1; h.y0 = (short)first_row; h.y1 = (short)(last_row + 1);
      h.flags = flags | CMD_GENERAL;
      for (int i = 0; i < WR_NI; i++) {
        k.i_lt[i] = q.interp[0][i]; k.i_lb[i] = q.interp[1][i];
        k.i_rt[i] = q.interp[2][i]; k.i_rb[i] = q.interp[3][i];
      }
      ok = true;
      break;
    }
    float perp = (px[l1i] - px[l0i]) * (py[r1i] - py[r0i]) - (py[l1i] - py[l0i]) * (px[r1i] - px[r0i]);
    bool flipped = px[l0i] > px[r0i] || (px[l0i] == px[r0i] && perp > 0.0f);
    int Lt = flipped ? r0i : l0i, Lb = flipped ? r1i : l1i;   // final left edge: top/bottom lanes
    int Rt = flipped ? l0i : r0i, Rb = flipped ? l1i : r1i;
    int left_edge_index = flipped ? r0i : l1i;   // Edge(...,edgeIndex): left=l1i, right=r0i
    int right_edge_index = flipped ? l1i : r0i;
    float yt = py[l0i], yb = py[l1i];
    float xl = px[Lt], xr = px[Rt];
    bool aa = (flags & CMD_AA) != 0;
    float aaRound = aa ? 0.0f : 0.5f;
    float ystart = floorf(wr_max(wr_min(yt, cy1), cy0) + aaRound) + 0.5f;
    // Edge ctor: x = p0.x + (y - p0.y) * xSlope with xSlope == 0 * yScale
    float yScale = 1.0f / wr_max(yb - yt, 1.0f / 256);
    float slopeL = (px[Lb] - px[Lt]) * yScale, slopeR = (px[Rb] - px[Rt]) * yScale;
    float lx = xl + (ystart - yt) * slopeL, rx = xr + (ystart - yt) * slopeR;
    // rows: centre y drawn while y <= min(yb, cy1)
    float ylim = wr_min(yb, cy1);
    int r0 = (int)(ystart - 0.5f);
    int r1 = (int)floorf(ylim - 0.5f) + 1;
    while ((float)r1 + 0.5f <= ylim) r1++;
    while (r1 > r0 && (float)(r1 - 1) + 0.5f > ylim) r1--;
    if (r1 <= r0) break;
    // clipSpan = clipRect.x_range().clip(x_range(l0,l1).merge(x_range(r0,r1)))
    float cs0 = wr_clamp(wr_min(xl, xr), cx0, cx1), cs1 = wr_clamp(wr_max(xl, xr), cx0, cx1);
    int sx0, sx1;
    if (!aa) {
      sx0 = wr_round_i(wr_clamp(lx, cs0, cs1));
      sx1 = wr_round_i(wr_clamp(rx, cs0, cs1));
    } else {
      int la0, la1, ra0, ra1;
      bool lmask = (q.aa_edge_mask >> left_edge_index) & 1;
      bool rmask = (q.aa_edge_mask >> right_edge_index) & 1;
      if (lmask) {
        float rad = 0.5f * fabsf(slopeL);
        la0 = (int)floorf(wr_clamp(lx - rad, cs0, cs1));
        la1 = (int)ceilf(wr_clamp(lx + rad, cs0, cs1));
        float dx = (-1.0f * 256.0f) * (1.0f / sqrtf(1.0f + slopeL * slopeL));
        k.aa_l0 = 128.0f + dx * (lx - 0.5f);
        k.aa_ls = -dx;
      } else {
        la0 = la1 = wr_round_i(wr_clamp(lx, cs0, cs1));
        k.aa_l0 = 256.0f;
        k.aa_ls = 0.0f;
      }
      if (rmask) {
        float rad = 0.5f * fabsf(slopeR);
        ra0 = (int)floorf(wr_clamp(rx - rad, cs0, cs1));
        ra1 = (int)ceilf(wr_clamp(rx + rad, cs0, cs1));
        float dx = (1.0f * 256.0f) * (1.0f / sqrtf(1.0f + slopeR * slopeR));
        k.aa_r0 = 128.0f + dx * (rx - 0.5f);
        k.aa_rs = -dx;
      } else {
        ra0 = ra1 = wr_round_i(wr_clamp(rx, cs0, cs1));
        k.aa_r0 = 256.0f;
        k.aa_rs = 0.0f;
      }
      h.aa_left_end = (short)la1;
      h.aa_right_start = (short)ra0;
      sx0 = la0;
      sx1 = ra1;
    }
    if (sx1 <= sx0) break;
    h.x0 = (short)sx0; h.x1 = (short)sx1; h.y0 = (short)r0; h.y1 = (short)r1;
    h.flags = flags;
    k.xl = lx; k.xr = rx; k.yt = yt; k.yscale = yScale;
    for (int i = 0; i < WR_NI; i++) {
      k.i_lt[i] = q.interp[Lt][i]; k.i_lb[i] = q.interp[Lb][i];
      k.i_rt[i] = q.interp[Rt][i]; k.i_rb[i] = q.interp[Rb][i];
    }
    ok = true;
  } while (0);
  a.hot[idx] = h;
  if (ok && a.row_tab && q.n_interp > 0 && !(h.flags & CMD_GENERAL) && (int)h.y1 - (int)h.y0 >= WR_ROW_TAB_MIN) {
    const int need = ((int)h.y1 - (int)h.y0) * 2 * q.n_interp;
    const int off = atomicAdd(a.pool_ctr, need);
    if (off >= 0 && off + need <= a.row_cap) {  // pool exhausted: the raster kernel walks the sums itself
      k.row_off = off;
      k.row_n = q.n_interp;
    }
  }
  if (ok && a.depth_runs && !(h.flags & CMD_PERSP) &&
      (!(h.flags & CMD_CONST_COLOR) || (h.flags & (CMD_AA | CMD_MASK | CMD_TEXTURED | CMD_OUT_RRRR)))) {
    // the shading of this command depends on where its passing depth runs start (chunk phase, span-shader
    // body vs fragment tail, interpolant sums): wr_depth_fail_rows records them row by row
    const int W = ((int)h.x1 - (int)h.x0 + 31) >> 5;
    const int need = ((int)h.y1 - (int)h.y0) * (W + 1);
    const int off = atomicAdd(a.pool_ctr + 1, need);
    if (off >= 0 && off + need <= a.fail_cap) {
      k.fail_off = off;
      k.fail_w = W;
      h.flags |= CMD_RUNS;
      a.hot[idx].flags = h.flags;
    }
  }
  if (ok) {
    bool simple = (h.flags & CMD_CONST_COLOR) && !(h.flags & (CMD_MASK | CMD_AA | CMD_TEXTURED | CMD_OUT_RRRR | CMD_GENERAL)) &&
                  h.col[0] <= 255 && h.col[1] <= 255 && h.col[2] <= 255 && h.col[3] <= 255;
    if (!simple) a.info->simple = 0;
    if (!(h.col[0] <= h.col[3] && h.col[1] <= h.col[3] && h.col[2] <= h.col[3])) a.info->premul_valid = 0;
    atomicMin(&a.info->bx0, (int)h.x0); atomicMin(&a.info->by0, (int)h.y0);
    atomicMax(&a.info->bx1, (int)h.x1); atomicMax(&a.info->by1, (int)h.y1);
    if (simple) {  // the common cover is read only while the whole batch is simple
      atomicMax(&a.info->cx0, (int)h.x0); atomicMax(&a.info->cy0, (int)h.y0);
      atomicMin(&a.info->cx1, (int)h.x1); atomicMin(&a.info->cy1, (int)h.y1);
    }
    if (a.tile_mask) {
      const int tx_a = max((int)h.x0, 0) / WRCU_TILE_W, tx_b = (min((int)h.x1, a.tgt.w) + WRCU_TILE_W - 1) / WRCU_TILE_W;
      const int ty_a = max((int)h.y0, 0) / WRCU_TILE_H, ty_b = (min((int)h.y1, a.tgt.h) + WRCU_TILE_H - 1) / WRCU_TILE_H;
      const uint32_t bit = 1u << (idx & 31);
      const int word = idx >> 5;
      if ((tx_b - tx_a) * (ty_b - ty_a) > WR_WIDE_TILES) {
        atomicOr(&a.wide_mask[word], bit);
        if (a.tile_any) atomicOr(&a.tile_any[a.any_words], 1u);
      } else {
        for (int ty = ty_a; ty < ty_b; ty++)
          for (int tx = tx_a; tx < tx_b; tx++) {
            const int tid = ty * a.bin_tiles_x + tx;
            atomicOr(&a.tile_mask[(size_t)tid * a.bin_words + word], bit);
            if (a.tile_any) atomicOr(&a.tile_any[tid >> 5], 1u << (tid & 31));
          }
      }
    }
  }
  // cold record is written by the caller after it fills the kind-specific part
  a.cold[idx] = k;
  return ok;
}

// swgl_validateGradient (swgl_ext.h:1336-1348): the 130-entry x 2-texel table must
// sit inside one 1024-texel row of gpu_buffer_f.  Also precomputes the span
// routines' can_merge test (stops[e].stepColor == stops[e+1].stepColor) as bit e.
WRD bool wr_grad_validate_merge(const FrameTablesDev& T, int address, uint32_t* merge) {
  for (int i = 0; i < 5; i++) merge[i] = 0;
  int ax = (int)((uint32_t)address % 1024U);
  bool valid = address >= 0 && ax + 260 <= 1024 && address + 260 <= T.n_gpu_buffer_f;
  if (!valid) return false;
  float4 prev = __ldg(T.gpu_buffer_f + address + 1);
  for (int e = 0; e < 129; e++) {
    float4 nx = __ldg(T.gpu_buffer_f + address + 2 * (e + 1) + 1);
    if (prev.x == nx.x && prev.y == nx.y && prev.z == nx.z && prev.w == nx.w) merge[e >> 5] |= 1u << (e & 31);
    prev = nx;
  }
  return true;
}
