// shader_composite.cuh — composite [FAST_PATH] (webrender/res/composite.glsl
// :73-234, RGB path): picture-cache tiles and external RGB surfaces into the
// framebuffer.  Span body: swgl_commitTexture[Color]RGBA8; tail: main().
#pragma once
#include "raster.cuh"
#include "setup_common.cuh"
#include "tma.cuh"

// CmdCold: f[0..3] uv bounds used by the span shader, g[0..3] vColor,
//          g[4] FAST_PATH, g[5..8] vUVBounds (fragment clamp),
//          g[12..19] the instance's sColor0 view (tile lists carry one texture per instance)
WRD const TexView& wr_composite_tex(const CmdCold& k) { return *(const TexView*)&k.g[12]; }
static_assert(sizeof(TexView) <= 32, "TexView must fit CmdCold::g[12..19]");
// The most commands the copy kernel (wr_composite_copy) stages; the host keeps longer tile lists on the tile kernel.
#define WR_COPY_MAX_CMDS 128
struct CompositeShader {
  struct Row {
    float o[2], step[2];
    TexRow tr;
  };
  WRD_MEMBER void row_setup(const RasterArgs& a, const CmdHot& c, int y, int tx0, bool rgba, Row& r) {
    const CmdCold& k = a.cold[c.cold];
    wr_row_interp<2>(a, k, c, y, r.o, r.step);
    int len = c.x1 - c.x0;
    int body_len = (rgba && len >= 4) ? (len & ~3) : 0;
    float u[4], v[4];
    for (int j = 0; j < 4; j++) {
      float uv[2];
      wr_interp_at<2>(a, r.o, r.step, j, uv);
      u[j] = uv[0];
      v[j] = uv[1];
    }
    wr_tex_row_setup(wr_composite_tex(k), k.f, true, body_len, u, v, max(tx0, (int)c.x0) - (int)c.x0, r.tr);
  }
  WRD_MEMBER Px source(const RasterArgs& a, const CmdHot& c, const Row& r, int x, int, bool) {
    const CmdCold& k = a.cold[c.cold];
    const TexView& t = wr_composite_tex(k);
    int rel = x - c.x0;
    if (rel < r.tr.body_len) {
      Px col{c.col[0], c.col[1], c.col[2], c.col[3]};
      return px_apply_color(wr_tex_body(t, r.tr, rel), col);
    }
    float uv[2];
    wr_interp_at<2>(a, r.o, r.step, rel, uv);
    bool fast = k.g[4] != 0.0f;
    float cu = uv[0], cv = uv[1];
    if (!fast) {
      cu = wr_clamp(cu, k.g[5], k.g[7]);
      cv = wr_clamp(cv, k.g[6], k.g[8]);
    }
    float texel[4], col[4];
    wr_tex_fragment(t, cu, cv, texel);
    for (int i = 0; i < 4; i++) col[i] = fast ? texel[i] : k.g[i] * texel[i];
    Px o;
    o.r = wr_round_pixel(col[0], 255.0f) & 0xFFFF;
    o.g = wr_round_pixel(col[1], 255.0f) & 0xFFFF;
    o.b = wr_round_pixel(col[2], 255.0f) & 0xFFFF;
    o.a = wr_round_pixel(col[3], 255.0f) & 0xFFFF;
    return o;
  }
};

// composite vertex stage (composite.glsl:73-159)
WRD void wr_setup_composite_one(const SetupArgs& a, int idx) {
  const float* f = (const float*)(a.instances + (size_t)idx * a.stride);
  const float* dr = f;
  const float* cr = f + 4;
  const float* uvr = f + 16;
  float flipx = f[28], flipy = f[29];
  QuadOut q;
  memset(&q, 0, sizeof q);
  float rect[4] = {(dr[2] - dr[0]) * flipx + dr[0], (dr[3] - dr[1]) * flipy + dr[1],
                   (dr[0] - dr[2]) * flipx + dr[2], (dr[1] - dr[3]) * flipy + dr[3]};
  bool fast = (a.features & WRCU_FEAT_FAST_PATH) != 0;
  float ub[4] = {wr_min(uvr[0], uvr[2]), wr_min(uvr[1], uvr[3]), wr_max(uvr[0], uvr[2]), wr_max(uvr[1], uvr[3])};
  bool unnorm = (int)f[13] == 1;
  const TexView tex0 = a.tex_list ? a.tex_list[idx] : a.color0;
  float tw = (float)tex0.w, th = (float)tex0.h;
  if (unnorm) {
    ub[0] += 0.5f; ub[1] += 0.5f; ub[2] += -0.5f; ub[3] += -0.5f;
    ub[0] /= tw; ub[1] /= th; ub[2] /= tw; ub[3] /= th;
  }
  const float ax[4] = {0.0f, 1.0f, 1.0f, 0.0f}, ay[4] = {0.0f, 0.0f, 1.0f, 1.0f};
  for (int k = 0; k < 4; k++) {
    float wx = (rect[2] - rect[0]) * ax[k] + rect[0], wy = (rect[3] - rect[1]) * ay[k] + rect[1];
    float cx = wr_clamp(wx, cr[0], cr[2]), cy = wr_clamp(wy, cr[1], cr[3]);
    float ux = (cx - rect[0]) / (rect[2] - rect[0]), uy = (cy - rect[1]) / (rect[3] - rect[1]);
    ux = (uvr[2] - uvr[0]) * ux + uvr[0];
    uy = (uvr[3] - uvr[1]) * uy + uvr[1];
    if (unnorm) { ux /= tw; uy /= th; }
    q.interp[k][0] = ux;
    q.interp[k][1] = uy;
    q.pos[k] = wr_mat_mul(a.tgt.proj, make_float4(cx, cy, 0.0f, 1.0f));
  }
  q.n_interp = 2;
  q.flags = CMD_TEXTURED;
  float white[4] = {1.0f, 1.0f, 1.0f, 1.0f};
  const float* color = fast ? white : f + 8;
  // swgl_drawSpanRGBA8: colour modulation only when color != vec4(1.0)
  bool is_white = color[0] == 1.0f && color[1] == 1.0f && color[2] == 1.0f && color[3] == 1.0f;
  if (is_white) { q.col[0] = q.col[1] = q.col[2] = q.col[3] = 255; }
  else {
    q.col[0] = (uint16_t)wr_round_pixel(color[2], 255.0f); q.col[1] = (uint16_t)wr_round_pixel(color[1], 255.0f);
    q.col[2] = (uint16_t)wr_round_pixel(color[0], 255.0f); q.col[3] = (uint16_t)wr_round_pixel(color[3], 255.0f);
  }
  int unsupported = 0;
  bool ok = wr_emit_quad(a, idx, q, &unsupported);
  if (ok) {
    CmdCold* k = &a.cold[idx];
    if (fast) { k->f[0] = 0.0f; k->f[1] = 0.0f; k->f[2] = 1.0f; k->f[3] = 1.0f; }
    else for (int i = 0; i < 4; i++) k->f[i] = ub[i];
    for (int i = 0; i < 4; i++) { k->g[i] = f[8 + i]; k->g[5 + i] = ub[i]; }
    k->g[4] = fast ? 1.0f : 0.0f;
    *(TexView*)&k->g[12] = tex0;
    // Copy class (tma.cuh): an untinted instance whose texels map 1:1 onto whole pixels is a rectangle copy
    // (opaque) or a premultiplied-over of a rectangle (alpha tiles).  Device-space edges carry the rounding
    // of the projection (x = 3072.00024), so "1:1" is judged the way the samplers do: a coordinate within
    // 1/1024 texel of a texel centre gives exactly that texel through both the nearest filter (floor) and
    // the 7-bit linear filter (fraction 0), and at unit step the span shaders step texels as integers
    // (blendTextureNearestFast / the FAST linear filter, swgl_ext.h:284-371, 476-541) — so the first and the
    // last pixel of the span decide u; v is walked row by row by the reference (Edge::nextRow) and is
    // checked on every row of the row table unless its step is exact.
    bool copyc = false;
    const CmdHot h = a.hot[idx];
    const int tiw = tex0.w, tih = tex0.h;
    k->i[2] = 0;
    if (a.copy_ok == 1 && a.tgt.fmt == WRCU_FMT_RGBA8 && a.tgt.tmap_id && tex0.fmt == WRCU_FMT_RGBA8 &&
        tex0.tmap_id && is_white && !(h.flags & (CMD_GENERAL | CMD_AA | CMD_MASK | CMD_CLIP_DIST)) &&
        (tiw & (tiw - 1)) == 0 && (tih & (tih - 1)) == 0 &&
        k->i_lt[0] == k->i_lb[0] && k->i_rt[0] == k->i_rb[0] && k->i_lt[1] == k->i_rt[1] && k->i_lb[1] == k->i_rb[1]) {
      const float tol = 1.0f / 1024.0f;
      const int wpx = (int)h.x1 - (int)h.x0, rows = (int)h.y1 - (int)h.y0;
      const float su = (k->i_rt[0] - k->i_lt[0]) / (k->xr - k->xl);
      const float u0 = k->i_lt[0] + ((float)h.x0 + 0.5f - k->xl) * su;
      const float u1 = k->i_lt[0] + ((float)((int)h.x1 - 1) + 0.5f - k->xl) * su;
      const float txf = floorf(u0 * tw);
      const float sl = (k->i_lb[1] - k->i_lt[1]) * k->yscale;
      const float v = k->i_lt[1] + ((float)h.y0 + 0.5f - k->yt) * sl;
      const float tyf = floorf(v * th);
      if (fabsf(u0 * tw - (txf + 0.5f)) <= tol && fabsf(u1 * tw - (txf + (float)(wpx - 1) + 0.5f)) <= tol && txf >= 0.0f &&
          txf + (float)wpx <= tw && tyf >= 0.0f && tyf + (float)rows <= th && fabsf(v * th - (tyf + 0.5f)) <= tol) {
        k->i[0] = (int)txf;
        k->i[1] = (int)tyf;
        if (sl * th == 1.0f) copyc = true;                                      // exact row step: nothing can drift
        else if (k->row_off >= 0 && k->row_n == 2) { k->i[2] = 1; copyc = true; }  // rows checked against the table
      }
    }
    // Fill class: a solid-colour or clear tile samples the 1x1 white dummy texture (renderer/mod.rs:3197-3230), so its
    // fragments are the instance colour on every pixel — body chunks (applyColor: muldiv255(c, 255) = c) and tail
    // pixels (round(color * 1.0 * 255)) alike — and the tile is a constant store / over / dest-out of its rect.
    if (!copyc && a.copy_ok && a.tgt.fmt == WRCU_FMT_RGBA8 && a.tgt.tmap_id && tex0.fmt == WRCU_FMT_RGBA8 && tiw == 1 && tih == 1 &&
        !(h.flags & (CMD_GENERAL | CMD_AA | CMD_MASK | CMD_CLIP_DIST)) && *(const uint32_t*)tex0.ptr == 0xFFFFFFFFu &&
        h.col[0] <= 255 && h.col[1] <= 255 && h.col[2] <= 255 && h.col[3] <= 255) {
      k->i[2] = 2;
      copyc = true;
    }
    if (a.copy_ok == 2 && k->i[2] != 2) copyc = false;  // dest-out: fills only
    if (copyc) a.hot[idx].flags |= CMD_COPY;
    else atomicAdd(&a.info->n_noncopy, 1);
  }
  if (unsupported) {
    atomicAdd(&a.info->unsupported, 1);
    atomicAdd(a.err_counter, 1);
  }
}
#ifdef WRCU_HOSTEMU
WR_SETUP_KERNEL(wr_setup_composite)
#else
// Copy-class candidates whose row step carries the rounding of yScale: every row's v (the left-edge sum
// of interpolant 1 in the row table the warp has just filled) must sit within 1/1024 texel of its texel
// centre.  The warp takes its candidates one at a time, rows strided over the lanes.
__device__ void wr_composite_check_rows(const SetupArgs& a, int idx) {
  const int lane = threadIdx.x & 31, wbase = idx - lane;
  unsigned m = __ballot_sync(0xFFFFFFFFu, idx < a.n && a.hot[idx].x1 > a.hot[idx].x0 && a.cold[idx].i[2] == 1);
  while (m) {
    const int ci = wbase + __ffs((int)m) - 1;
    m &= m - 1;
    const CmdHot h = a.hot[ci];
    const CmdCold& k = a.cold[ci];
    const float th = (float)wr_composite_tex(k).h;
    const float* t = a.row_tab + k.row_off;
    const int rows = (int)h.y1 - (int)h.y0;
    bool bad = false;
    for (int r = lane; r < rows; r += 32) bad = bad || fabsf(t[(size_t)r * 4 + 2] * th - ((float)(k.i[1] + r) + 0.5f)) > (1.0f / 1024.0f);
    if (__any_sync(0xFFFFFFFFu, bad) && lane == 0) {
      a.hot[ci].flags &= ~CMD_COPY;
      atomicAdd(&a.info->n_noncopy, 1);
    }
  }
}
__device__ __noinline__ void wr_setup_composite_block(const SetupArgs& a, int idx) {
  if (idx == 0 && a.info_next) wr_reset_batch_info(a.info_next);
  if (a.warp_per_inst) {
    const int lane = threadIdx.x & 31;
    idx >>= 5;
    if (idx >= a.n) return;
    if (lane == 0) wr_setup_composite_one(a, idx);
    __syncwarp();
    if (a.cold[idx].row_off >= 0) wr_fill_row_table_spread(a, idx, lane);
    __syncwarp();
    // copy-class candidate whose row step is inexact: check its rows against the table just filled
    const CmdHot h = a.hot[idx];
    const CmdCold& k = a.cold[idx];
    if (h.x1 > h.x0 && k.i[2] == 1) {
      const float th = (float)wr_composite_tex(k).h;
      const float* t = a.row_tab + k.row_off;
      const int rows = (int)h.y1 - (int)h.y0;
      bool bad = false;
      for (int r = lane; r < rows; r += 32) bad = bad || fabsf(t[(size_t)r * 4 + 2] * th - ((float)(k.i[1] + r) + 0.5f)) > (1.0f / 1024.0f);
      if (__any_sync(0xFFFFFFFFu, bad) && lane == 0) {
        a.hot[idx].flags &= ~CMD_COPY;
        atomicAdd(&a.info->n_noncopy, 1);
      }
    }
    return;
  }
  if (idx < a.n) wr_setup_composite_one(a, idx);
  __syncwarp();
  wr_fill_row_tables_warp(a, idx);
  __syncwarp();
  wr_composite_check_rows(a, idx);
}

// ---- copy-class composite: the tile list as 2-D bulk-tensor copies (see tma.cuh) ----------------
// Work items = 256x16-pixel boxes of every instance's rect, dealt round-robin to the persistent CTAs.
// Boxes wholly inside their rect go through the copy engine; ragged-edge boxes are moved by the
// CTA's threads with plain accesses.
//   opaque (blend off):  thread 0 alone drives a ring of WR_TMA_STAGES shared-memory slots — bulk load
//     of the source box, bulk store of the same bytes into the framebuffer, loads two boxes ahead of
//     the stores — while warps 1..3 copy the ragged boxes.
//   premultiplied-alpha over (alpha tiles): each slot holds the source box AND the destination box
//     (one barrier, two bulk loads); the 128 threads blend in shared memory (blend.h:473-474), then
//     thread 0 bulk-stores the destination box and refills the slot that has just drained.
// The batch's copy commands, staged once per CTA into shared memory (index-preserving, so every CTA deals
// the boxes the same way): rect, source origin, the source's tensor map and plain view.
struct WrCopyCmd {
  short x0, y0;
  int w, h;        // 0 x 0: not a copy command
  int sx, sy;      // source origin (texels)
  int tmap, aligned;
  const uint8_t* sptr;
  int spitch;
  uint32_t fill;   // fill class (sptr == nullptr): the constant source pixel
};
struct WrBoxIter {
  int i = -1, b = 0, nb = 0, nbx = 1, g = 0;
  bool started = false;
  // next box of this CTA that is (full == want_full); false when the batch is exhausted
  __device__ bool next(const WrCopyCmd* cl, int n, bool want_full, int& bx, int& by) {
    const int G = (int)gridDim.x;
    for (;;) {
      if (started) b += G;
      started = true;
      while (i < 0 || b >= nb) {
        if (i >= 0) g += nb;
        i++;
        if (i >= n) return false;
        const WrCopyCmd& c = cl[i];
        if (c.w <= 0 || c.h <= 0) { nb = 0; b = 0; continue; }
        nbx = (c.w + WR_TMA_BOX_W - 1) / WR_TMA_BOX_W;
        nb = nbx * ((c.h + WR_TMA_BOX_H - 1) / WR_TMA_BOX_H);
        b = ((int)blockIdx.x - g % G + G) % G;
      }
      const WrCopyCmd& c = cl[i];
      bx = (b % nbx) * WR_TMA_BOX_W;
      by = (b / nbx) * WR_TMA_BOX_H;
      // the copy engine takes whole boxes whose source and destination start on 16-byte boundaries
      // (box origins off them fault: tools/probe/tma_probe.cu); everything else is moved by threads
      const bool full = c.aligned && c.sptr && bx + WR_TMA_BOX_W <= c.w && by + WR_TMA_BOX_H <= c.h;
      if (full == want_full) return true;
    }
  }
};

WRD uint32_t wr_over_px(uint32_t d, uint32_t s) {  // premultiplied-alpha over, one BGRA8 pixel
  const uint32_t cc = 255u - (s >> 24);
  const uint32_t rb = wr_premult_over_pair(d & 0x00FF00FFu, s & 0x00FF00FFu, cc);
  const uint32_t ga = wr_premult_over_pair((d >> 8) & 0x00FF00FFu, (s >> 8) & 0x00FF00FFu, cc);
  return rb | (ga << 8);
}

// BLEND: 0 store, 1 premultiplied-alpha over (blend.h:473-474), 2 premultiplied dest-out (d - muldiv255(d, src.a))
template <int BLEND>
WRD uint32_t wr_copy_px(uint32_t d, uint32_t s) {
  if (BLEND == 1) return wr_over_px(d, s);
  if (BLEND == 2) {
    const uint32_t sa = s >> 24;
    const uint32_t rb = d & 0x00FF00FFu, ga = (d >> 8) & 0x00FF00FFu;
    // per 16-bit lane: d - ((d * sa + d) >> 8), d <= 255 so the lanes never borrow or carry
    const uint32_t mrb = ((rb * sa + rb) >> 8) & 0x00FF00FFu, mga = ((ga * sa + ga) >> 8) & 0x00FF00FFu;
    return (rb - mrb) | ((ga - mga) << 8);
  }
  return s;
}
template <int BLEND>
WRD uint4 wr_copy_px4(uint4 d, uint4 s) {
  return make_uint4(wr_copy_px<BLEND>(d.x, s.x), wr_copy_px<BLEND>(d.y, s.y), wr_copy_px<BLEND>(d.z, s.z), wr_copy_px<BLEND>(d.w, s.w));
}
// Ragged-edge boxes and fills by plain accesses: `t` of `nt` threads (whole warps) share the rows of each box.
// A warp takes WR_RAG_ROWS rows at a time and issues every load of a step — source and, when blending,
// destination, of all its rows — before the first store, so a box costs two or three memory round trips
// instead of one per row.  The destination's pitch is a multiple of 16 bytes (it has a tensor map), so all rows of
// a box share the split into scalar head pixels up to the 16-byte boundary, 16-byte stores, scalar tail.
#define WR_RAG_ROWS 4
template <int BLEND>
__device__ void wr_copy_ragged(const RasterArgs& a, const WrCopyCmd* cl, int n, int t, int nt) {
  WrBoxIter it;
  int bx, by;
  const int lane = t & 31, w = t >> 5, nw = nt >> 5;
  while (it.next(cl, n, false, bx, by)) {
    const WrCopyCmd& c = cl[it.i];
    const int bw = min(WR_TMA_BOX_W, c.w - bx), bh = min(WR_TMA_BOX_H, c.h - by);
    const bool fill = c.sptr == nullptr;
    uint32_t* d0 = (uint32_t*)(a.tgt.color + (size_t)((int)c.y0 + by) * a.tgt.color_pitch) + (int)c.x0 + bx;
    const size_t dstride = (size_t)a.tgt.color_pitch >> 2;
    const uint32_t* s0 = fill ? nullptr : (const uint32_t*)(c.sptr + (size_t)(c.sy + by) * c.spitch) + c.sx + bx;
    const size_t sstride = (size_t)c.spitch >> 2;  // (RGBA8 sources: the pitch is a whole number of pixels)
    int head = (int)(((16u - (unsigned)((uintptr_t)d0 & 15u)) & 15u) >> 2);
    if (head > bw) head = bw;
    const int nv = (bw - head) >> 2, tail0 = head + (nv << 2);
    const bool in_phase = !fill && (((uintptr_t)(s0 + head) | (uintptr_t)c.spitch) & 15) == 0;
    for (int r0 = w * WR_RAG_ROWS; r0 < bh; r0 += nw * WR_RAG_ROWS) {
      const int nr = min(WR_RAG_ROWS, bh - r0);
      for (int q = lane; q < nv; q += 32) {
        uint4 sv[WR_RAG_ROWS], dv[WR_RAG_ROWS];
#pragma unroll
        for (int k = 0; k < WR_RAG_ROWS; k++) {
          if (k >= nr) break;
          if (fill) sv[k] = make_uint4(c.fill, c.fill, c.fill, c.fill);
          else {
            const uint32_t* sp = s0 + (size_t)(r0 + k) * sstride + head;
            if (in_phase) sv[k] = __ldg((const uint4*)sp + q);
            else sv[k] = make_uint4(__ldg(sp + 4 * q), __ldg(sp + 4 * q + 1), __ldg(sp + 4 * q + 2), __ldg(sp + 4 * q + 3));
          }
          if (BLEND) dv[k] = ((const uint4*)(d0 + (size_t)(r0 + k) * dstride + head))[q];
        }
#pragma unroll
        for (int k = 0; k < WR_RAG_ROWS; k++) {
          if (k >= nr) break;
          ((uint4*)(d0 + (size_t)(r0 + k) * dstride + head))[q] = BLEND ? wr_copy_px4<BLEND>(dv[k], sv[k]) : sv[k];
        }
      }
      // scalar pixels: the head and the tail of each row (at most 3 + 3), one (row, pixel) per lane
      const int ns = head + (bw - tail0);
      for (int e = lane; e < nr * ns; e += 32) {
        const int k = e / ns, j = e % ns, xq = j < head ? j : tail0 + (j - head);
        uint32_t* dp = d0 + (size_t)(r0 + k) * dstride + xq;
        const uint32_t sv = fill ? c.fill : __ldg(s0 + (size_t)(r0 + k) * sstride + xq);
        *dp = BLEND ? wr_copy_px<BLEND>(*dp, sv) : sv;
      }
    }
  }
}

#define WR_TMA_BLEND_STAGES 3
template <int BLEND>
__global__ void __launch_bounds__(WR_TMA_THREADS) wr_composite_copy(RasterArgs a) {
  extern __shared__ __align__(128) uint8_t wr_copy_smem[];
  __shared__ __align__(8) uint64_t full[WR_TMA_STAGES];
  __shared__ WrCopyCmd cl[WR_COPY_MAX_CMDS];
  wr_pdl_launch_dependents();
  wr_pdl_wait();
  const BatchInfo bi = *a.info;
  if (!bi.all_copy) return;  // the ordered tile kernel draws this batch
  const CUtensorMap* maps = (const CUtensorMap*)a.tmaps;
  const CUtensorMap* dst_map = maps + a.tgt.tmap_id;
  const int n0 = min(a.n, WR_COPY_MAX_CMDS);
  // A tile whose clip starts off a 16-byte boundary (a dirty rect cut anywhere) is split: a strip of 1-3 pixel
  // columns up to the boundary, copied by threads, and the rest — source and destination in phase for a 1:1
  // tile — through the copy engine.  Entry i = the body (or all) of command i, entry n0 + i = its strip.
  const bool split = 2 * n0 <= WR_COPY_MAX_CMDS;
  const int n = split ? 2 * n0 : n0;
  // Start-up, spread over the CTA's threads (one thread walking the list pays two dependent DRAM
  // round trips per command): thread t stages command t.
  for (int i = threadIdx.x; i < n0; i += WR_TMA_THREADS) {
    const CmdHot c = a.hot[i];
    WrCopyCmd cc, cs;
    cc.x0 = c.x0; cc.y0 = c.y0;
    cc.w = cc.h = 0;
    cc.sx = cc.sy = cc.tmap = cc.aligned = 0; cc.sptr = nullptr; cc.spitch = 0; cc.fill = 0;
    cs = cc;
    if (c.x1 > c.x0 && c.y1 > c.y0 && (c.flags & CMD_COPY) && a.cold[c.cold].i[2] == 2) {
      // fill class: the command's colour (BGRA lanes of the hot record) on every pixel
      cc.w = (int)c.x1 - (int)c.x0;
      cc.h = (int)c.y1 - (int)c.y0;
      cc.fill = (uint32_t)c.col[0] | ((uint32_t)c.col[1] << 8) | ((uint32_t)c.col[2] << 16) | ((uint32_t)c.col[3] << 24);
    } else if (BLEND != 2 && c.x1 > c.x0 && c.y1 > c.y0 && (c.flags & CMD_COPY)) {
      const CmdCold& k = a.cold[c.cold];
      const TexView& tv = wr_composite_tex(k);
      cc.w = (int)c.x1 - (int)c.x0;
      cc.h = (int)c.y1 - (int)c.y0;
      cc.sx = k.i[0]; cc.sy = k.i[1];
      cc.tmap = tv.tmap_id;
      cc.aligned = (((int)c.x0 | k.i[0]) & 3) == 0;
      cc.sptr = tv.ptr;
      cc.spitch = tv.pitch;
      const int head = (4 - ((int)c.x0 & 3)) & 3;
      if (split && !cc.aligned && (((int)c.x0 ^ k.i[0]) & 3) == 0 && cc.w > head) {
        cs = cc;
        cs.w = head;          // the strip: never a full box
        cc.x0 = (short)((int)c.x0 + head);
        cc.sx += head;
        cc.w -= head;
        cc.aligned = 1;
      }
      // a table slot that held another texture's map before (RasterArgs::tmap_acquire, see wrcu_api.cu
      // make_tensor_map) must be re-read through the tensormap proxy
      if (a.tmap_acquire) wr_tma_acquire_map(maps + tv.tmap_id);
    }
    cl[i] = cc;
    if (split) cl[n0 + i] = cs;
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < WR_TMA_STAGES; s++) wr_mbar_init(&full[s], 1);
    wr_fence_mbar_init();
    if (a.tmap_acquire) wr_tma_acquire_map(dst_map);
  }
  __syncthreads();
  int bx, by;
  if (BLEND == 2) {  // dest-out: fills only (no box is "full")
    wr_copy_ragged<2>(a, cl, n, threadIdx.x, WR_TMA_THREADS);
    return;
  }
  if (!BLEND) {
    if (threadIdx.x == 0) {
      // ---- the copy engine's driver: every full box of this CTA, loads DEPTH boxes ahead of stores ----
      constexpr int DEPTH = WR_TMA_STAGES - 2;
      int ring_x[WR_TMA_STAGES] = {0}, ring_y[WR_TMA_STAGES] = {0};
      int issued = 0, stored = 0;
      auto store_one = [&]() {
        const int s = stored % WR_TMA_STAGES;
        wr_mbar_wait(&full[s], (uint32_t)((stored / WR_TMA_STAGES) & 1));
        wr_tma_store_2d(dst_map, ring_x[s], ring_y[s], wr_copy_smem + (size_t)s * WR_TMA_BOX_BYTES);
        wr_tma_commit();
        stored++;
      };
      WrBoxIter it;
      while (it.next(cl, n, true, bx, by)) {
        const WrCopyCmd& c = cl[it.i];
        const int s = issued % WR_TMA_STAGES;
        if (issued >= WR_TMA_STAGES) wr_tma_wait_read<1>();  // the store that last read slot s has drained
        ring_x[s] = (int)c.x0 + bx;
        ring_y[s] = (int)c.y0 + by;
        wr_mbar_expect_tx(&full[s], WR_TMA_BOX_BYTES);
        wr_tma_load_2d(wr_copy_smem + (size_t)s * WR_TMA_BOX_BYTES, maps + c.tmap, c.sx + bx, c.sy + by, &full[s]);
        issued++;
        if (issued - stored > DEPTH) store_one();
      }
      while (stored < issued) store_one();
      wr_tma_wait_all<0>();  // stores complete before the CTA's shared memory is released
    } else if (threadIdx.x >= 32) {
      wr_copy_ragged<0>(a, cl, n, threadIdx.x - 32, WR_TMA_THREADS - 32);
    }
    return;
  }
  // ---- blended: all threads walk the CTA's full boxes in step; thread 0 also feeds the ring ----
  constexpr int ST = WR_TMA_BLEND_STAGES, DEPTH = ST - 1;
  WrBoxIter prod, cons;
  auto issue = [&](int nn) {  // thread 0: source and destination box of the producer's current item → slot nn % ST
    const WrCopyCmd& c = cl[prod.i];
    uint8_t* slot = wr_copy_smem + (size_t)(nn % ST) * 2 * WR_TMA_BOX_BYTES;
    wr_mbar_expect_tx(&full[nn % ST], 2 * WR_TMA_BOX_BYTES);
    wr_tma_load_2d(slot, maps + c.tmap, c.sx + bx, c.sy + by, &full[nn % ST]);
    wr_tma_load_2d(slot + WR_TMA_BOX_BYTES, dst_map, (int)c.x0 + bx, (int)c.y0 + by, &full[nn % ST]);
  };
  int nload = 0;
  bool more = true;
  if (threadIdx.x == 0)
    for (int d = 0; d < DEPTH && more; d++) {
      more = prod.next(cl, n, true, bx, by);
      if (more) issue(nload++);
    }
  int j = 0;
  while (cons.next(cl, n, true, bx, by)) {
    const int s = j % ST;
    wr_mbar_wait(&full[s], (uint32_t)((j / ST) & 1));
    uint4* sp = (uint4*)(wr_copy_smem + (size_t)s * 2 * WR_TMA_BOX_BYTES);
    uint4* dp = sp + WR_TMA_BOX_BYTES / 16;
#pragma unroll 4
    for (int q = threadIdx.x; q < WR_TMA_BOX_BYTES / 16; q += WR_TMA_THREADS) {
      const uint4 sv = sp[q], dv = dp[q];
      dp[q] = make_uint4(wr_over_px(dv.x, sv.x), wr_over_px(dv.y, sv.y), wr_over_px(dv.z, sv.z), wr_over_px(dv.w, sv.w));
    }
    wr_fence_proxy_async();  // the blended box → visible to the copy engine
    __syncthreads();
    if (threadIdx.x == 0) {
      wr_tma_store_2d(dst_map, (int)cl[cons.i].x0 + bx, (int)cl[cons.i].y0 + by, dp);
      wr_tma_commit();
      if (more) {
        int pbx = bx, pby = by;  // (issue() reads bx/by of the producer's item)
        more = prod.next(cl, n, true, bx, by);
        if (more) {
          wr_tma_wait_read<1>();  // item j-1's store (slot (j + DEPTH) % ST) has finished reading shared memory
          issue(nload++);
        }
        bx = pbx; by = pby;
      }
    }
    j++;
  }
  if (threadIdx.x == 0) wr_tma_wait_all<0>();
  __syncthreads();
  wr_copy_ragged<1>(a, cl, n, threadIdx.x, WR_TMA_THREADS);
}
#endif

#ifndef WRCU_HOSTEMU
template <> struct WrMinCtas<CompositeShader> { enum { v = 3 }; };
#endif
