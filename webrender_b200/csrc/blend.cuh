// blend.cuh — the blend stage.  Bit-identical restatement of the reference's
// 8-bit fixed-point blend arithmetic (swgl/src/blend.h:416-735): 16-bit lanes
// in B,G,R,A memory order, muldiv255(x,y) = (x*y + x) >> 8, saturating pack.
//
// Two forms:
//  * packed-pair fast paths for the keys on the hot path (premultiplied over,
//    alpha, multiply, dest-out): a pixel is two 32-bit words holding two
//    16-bit lanes each (rb = B | R<<16, ga = G | A<<16) so one integer
//    multiply processes two channels; no lane can carry into its neighbour
//    because 255*256 < 65536.
//  * a generic per-lane path for every other key (advanced blend modes etc.).
#pragma once
#include <stdint.h>
#include "wrcu_internal.h"

// internal blend keys set per command by blend overrides (not part of the ABI)
#define WRCU_BLEND__DROP_SHADOW 100
#define WRCU_BLEND__SUBPIXEL_TEXT 101

struct Px {  // 16-bit lanes held in ints, memory order B,G,R,A
  int b, g, r, a;
};

// 16-bit lanes: products wrap mod 2^16 before the logical shift, as in the
// reference's uint16_t vectors.
WRD int wr_muldiv255(int x, int y) { return ((x * y + x) & 0xFFFF) >> 8; }
WRD int wr_muldiv256(int x, int y) { return ((x * y) & 0xFFFF) >> 8; }
// 16-bit lane wrap + signed-saturating pack (texture.h:13-21)
WRD uint32_t wr_pack16(int v) {
  uint32_t u = (uint32_t)v & 0xFFFFu;
  return (u & 0x8000u) ? 0u : (u > 255u ? 255u : u);
}
WRD int wr_addlow(int x, int y) {  // blend.h:202-205
  return (((x & 0xFF) + (y & 0xFF)) & 0xFF) |
         (((((x >> 8) & 0xFF) + ((y >> 8) & 0xFF)) & 0xFF) << 8);
}
WRD Px px_unpack(uint32_t p) {
  return Px{(int)(p & 0xFF), (int)((p >> 8) & 0xFF), (int)((p >> 16) & 0xFF), (int)(p >> 24)};
}
WRD uint32_t px_pack(Px v) {
  return wr_pack16(v.b) | (wr_pack16(v.g) << 8) | (wr_pack16(v.r) << 16) | (wr_pack16(v.a) << 24);
}
WRD Px px_scale256(Px s, int aa) {
  return Px{wr_muldiv256(s.b, aa), wr_muldiv256(s.g, aa), wr_muldiv256(s.r, aa), wr_muldiv256(s.a, aa)};
}
WRD Px px_scale255(Px s, int m) {
  return Px{wr_muldiv255(s.b, m), wr_muldiv255(s.g, m), wr_muldiv255(s.r, m), wr_muldiv255(s.a, m)};
}
// applyColor(src, color) = muldiv255(color, src)  (blend.h:156-163)
WRD Px px_apply_color(Px src, Px color) {
  return Px{wr_muldiv255(color.b, src.b), wr_muldiv255(color.g, src.g),
            wr_muldiv255(color.r, src.r), wr_muldiv255(color.a, src.a)};
}

WRD int wr_round_pixel(float v, float scale) {
  // roundfast for the non-SSE build: int(v*scale + 0.5f) (glsl.h:732-737)
  return (int)(__fadd_rn(__fmul_rn(v, scale), 0.5f));
}
WRD float wr_recip_or(float v, float f) {
  return v != 0.0f ? __fdiv_rn(1.0f, v) : f;
}
WRD float wr_min(float a, float b) { return a < b ? a : b; }
WRD float wr_max(float a, float b) { return a > b ? a : b; }
WRD float wr_clamp(float a, float lo, float hi) {
  return wr_min(wr_max(a, lo), hi);
}

// ---- HSL helpers (blend.h:312-343) -------------------------------------------
WRD float wr_lum(const float* v) {
  return __fadd_rn(__fadd_rn(__fmul_rn(v[0], 0.30f), __fmul_rn(v[1], 0.59f)), __fmul_rn(v[2], 0.11f));
}
WRD float wr_min3(const float* v) { return wr_min(wr_min(v[0], v[1]), v[2]); }
WRD float wr_max3(const float* v) { return wr_max(wr_max(v[0], v[1]), v[2]); }
WRD void wr_clip_color(float* out, const float* v, float lum, float alpha) {
  float mincol = wr_max(-wr_min3(v), lum);
  float maxcol = wr_max(wr_max3(v), __fsub_rn(alpha, lum));
  float k = __fmul_rn(__fmul_rn(lum, __fsub_rn(alpha, lum)),
                      wr_recip_or(__fmul_rn(mincol, maxcol), 0.0f));
  for (int i = 0; i < 3; i++) out[i] = __fadd_rn(lum, __fmul_rn(v[i], k));
}
WRD void wr_set_lum(float* out, const float* base, const float* ref, float alpha) {
  float lb = wr_lum(base);
  float t[3] = {__fsub_rn(base[0], lb), __fsub_rn(base[1], lb), __fsub_rn(base[2], lb)};
  wr_clip_color(out, t, wr_lum(ref), alpha);
}
WRD void wr_set_lum_sat(float* out, const float* base, const float* sref,
                                      const float* lref, float alpha) {
  float mb = wr_min3(base);
  float diff[3] = {__fsub_rn(base[0], mb), __fsub_rn(base[1], mb), __fsub_rn(base[2], mb)};
  float sbase = wr_max3(diff);
  float ssat = __fsub_rn(wr_max3(sref), wr_min3(sref));
  float k = wr_recip_or(sbase, 0.0f);
  float t[3] = {__fmul_rn(__fmul_rn(diff[0], ssat), k), __fmul_rn(__fmul_rn(diff[1], ssat), k),
                __fmul_rn(__fmul_rn(diff[2], ssat), k)};
  wr_set_lum(out, t, lref, alpha);
}

#define WR_LANES4(o, expr)                                       \
  do {                                                           \
    int s, d;                                                    \
    s = src.b; d = dst.b; (o).b = (expr) & 0xFFFF;               \
    s = src.g; d = dst.g; (o).g = (expr) & 0xFFFF;               \
    s = src.r; d = dst.r; (o).r = (expr) & 0xFFFF;               \
    s = src.a; d = dst.a; (o).a = (expr) & 0xFFFF;               \
    (void)s; (void)d;                                            \
  } while (0)

// Generic blend of one RGBA8 pixel (all keys), blend.h:462-700.  `kc` is
// ctx->blendcolor in B,G,R,A lane order.
WRD_SHARED Px wr_blend_rgba8(int key, Px src, Px dst, Px kc) {
  Px o = src;
  switch (key) {
    case WRCU_BLEND_NONE:
      return src;
    case WRCU_BLEND_ALPHA: {
      int sa = src.a;
      Px s1 = src;
      s1.a = src.a | 255;
      o.b = wr_addlow(dst.b, wr_muldiv255(sa, (s1.b - dst.b) & 0xFFFF) & 0xFFFF);
      o.g = wr_addlow(dst.g, wr_muldiv255(sa, (s1.g - dst.g) & 0xFFFF) & 0xFFFF);
      o.r = wr_addlow(dst.r, wr_muldiv255(sa, (s1.r - dst.r) & 0xFFFF) & 0xFFFF);
      o.a = wr_addlow(dst.a, wr_muldiv255(sa, (s1.a - dst.a) & 0xFFFF) & 0xFFFF);
      return o;
    }
    case WRCU_BLEND_PREMULTIPLIED_ALPHA: {
      int sa = src.a;
      WR_LANES4(o, s + d - wr_muldiv255(d, sa));
      return o;
    }
    case WRCU_BLEND_SUBPIXEL_PASS0:
      WR_LANES4(o, d - wr_muldiv255(d, s));
      return o;
    case WRCU_BLEND_SUBPIXEL_PASS0_KEEP_A:
      WR_LANES4(o, d - wr_muldiv255(d, s));
      o.a = dst.a;
      return o;
    case WRCU_BLEND_PREMULTIPLIED_DEST_OUT: {
      int sa = src.a;
      WR_LANES4(o, d - wr_muldiv255(d, sa));
      return o;
    }
    case WRCU_BLEND_MULTIPLY:
      WR_LANES4(o, wr_muldiv255(s, d));
      return o;
    case WRCU_BLEND_PLUS_LIGHTER:
      WR_LANES4(o, s + d);
      return o;
    case WRCU_BLEND_ADD_KEEP_ALPHA_OVER: {
      int a = src.a + dst.a - wr_muldiv255(dst.a, src.a);
      WR_LANES4(o, s + d);
      o.a = a & 0xFFFF;
      return o;
    }
    case WRCU_BLEND_DST_ALPHA_ADD: {
      int da = dst.a;
      WR_LANES4(o, d + ((s - wr_muldiv255(s, da)) & 0xFFFF));
      o.a = dst.a;
      return o;
    }
    case WRCU_BLEND_CONSTANT_COLOR:
      o.b = wr_addlow(dst.b, wr_muldiv255(src.b, (kc.b - dst.b) & 0xFFFF) & 0xFFFF);
      o.g = wr_addlow(dst.g, wr_muldiv255(src.g, (kc.g - dst.g) & 0xFFFF) & 0xFFFF);
      o.r = wr_addlow(dst.r, wr_muldiv255(src.r, (kc.r - dst.r) & 0xFFFF) & 0xFFFF);
      o.a = wr_addlow(dst.a, wr_muldiv255(src.a, (kc.a - dst.a) & 0xFFFF) & 0xFFFF);
      return o;
    case WRCU_BLEND_MIN:
      WR_LANES4(o, s < d ? s : d);
      return o;
    case WRCU_BLEND_MAX:
      WR_LANES4(o, s > d ? s : d);
      return o;
    case WRCU_BLEND_ADV_MULTIPLY: {
      int sa = src.a, da = dst.a;
      int db = wr_muldiv255(sa - src.b, da - dst.b) & 0xFFFF;
      int dg = wr_muldiv255(sa - src.g, da - dst.g) & 0xFFFF;
      int dr = wr_muldiv255(sa - src.r, da - dst.r) & 0xFFFF;
      int dA = wr_muldiv255(sa, da) & 0xFFFF;
      o.b = (src.b + dst.b + db - dA) & 0xFFFF;
      o.g = (src.g + dst.g + dg - dA) & 0xFFFF;
      o.r = (src.r + dst.r + dr - dA) & 0xFFFF;
      o.a = (src.a + dst.a - dA) & 0xFFFF;
      return o;
    }
    case WRCU_BLEND_ADV_SCREEN:
      WR_LANES4(o, s + d - wr_muldiv255(s, d));
      return o;
    case WRCU_BLEND_ADV_OVERLAY:
    case WRCU_BLEND_ADV_HARD_LIGHT: {
      int sa = src.a, da = dst.a;
      int sv[4] = {src.b, src.g, src.r, src.a}, dv[4] = {dst.b, dst.g, dst.r, dst.a}, ov[4], diff[4];
      for (int i = 0; i < 4; i++)
        diff[i] = (wr_muldiv255(sv[i], dv[i]) +
                   wr_muldiv255((sa - sv[i]) & 0xFFFF, (da - dv[i]) & 0xFFFF)) & 0xFFFF;
      for (int i = 0; i < 4; i++) {
        bool cond = key == WRCU_BLEND_ADV_OVERLAY
                        ? (((dv[i] * 2) & 0xFFFF) <= (da & 0xFFFF))
                        : (((sv[i] * 2) & 0xFFFF) <= (sa & 0xFFFF));
        int t = cond ? (((i < 3 ? diff[i] : 0) - diff[3]) & 0xFFFF) : ((-diff[i]) & 0xFFFF);
        ov[i] = (sv[i] + dv[i] + t) & 0xFFFF;
      }
      return Px{ov[0], ov[1], ov[2], ov[3]};
    }
    case WRCU_BLEND_ADV_DARKEN: {
      int sa = src.a, da = dst.a;
      WR_LANES4(o, s + d - max(wr_muldiv255(s, da), wr_muldiv255(d, sa)));
      return o;
    }
    case WRCU_BLEND_ADV_LIGHTEN: {
      int sa = src.a, da = dst.a;
      WR_LANES4(o, s + d - min(wr_muldiv255(s, da), wr_muldiv255(d, sa)));
      return o;
    }
    case WRCU_BLEND_ADV_COLOR_DODGE:
    case WRCU_BLEND_ADV_COLOR_BURN:
    case WRCU_BLEND_ADV_SOFT_LIGHT: {
      float sv[4] = {(float)src.b, (float)src.g, (float)src.r, (float)src.a};
      float dv[4] = {(float)dst.b, (float)dst.g, (float)dst.r, (float)dst.a};
      float sa = sv[3], da = dv[3];
      int ov[4];
      float dua = wr_recip_or(da, 0.0f);
      for (int i = 0; i < 4; i++) {
        float v;
        if (key == WRCU_BLEND_ADV_COLOR_DODGE) {
          float t = i < 3 ? wr_min(da, __fmul_rn(__fmul_rn(dv[i], sa),
                                                 wr_recip_or(__fsub_rn(sa, sv[i]), 255.0f)))
                          : dv[i];
          v = __fadd_rn(__fadd_rn(__fmul_rn(sa, t), __fmul_rn(sv[i], __fsub_rn(255.0f, da))),
                        __fmul_rn(dv[i], __fsub_rn(255.0f, sa)));
        } else if (key == WRCU_BLEND_ADV_COLOR_BURN) {
          float t = i < 3 ? __fsub_rn(da, wr_min(da, __fmul_rn(__fmul_rn(__fsub_rn(da, dv[i]), sa),
                                                               wr_recip_or(sv[i], 255.0f))))
                          : dv[i];
          v = __fadd_rn(__fadd_rn(__fmul_rn(sa, t), __fmul_rn(sv[i], __fsub_rn(255.0f, da))),
                        __fmul_rn(dv[i], __fsub_rn(255.0f, sa)));
        } else {
          float dstU = __fmul_rn(dv[i], dua);
          float scale = __fsub_rn(__fadd_rn(sv[i], sv[i]), sa);
          float t = 0.0f;
          if (i < 3) {
            float alt = wr_min(
                __fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(16.0f, dstU), 12.0f), dstU), 3.0f),
                __fsub_rn(__fdiv_rn(1.0f, __fsqrt_rn(dstU)), 1.0f));
            t = __fmul_rn(scale, scale < 0.0f ? __fsub_rn(1.0f, dstU) : alt);
          }
          v = __fadd_rn(__fmul_rn(dv[i], __fadd_rn(255.0f, t)),
                        __fmul_rn(sv[i], __fsub_rn(255.0f, da)));
        }
        ov[i] = wr_round_pixel(v, 1.0f / 255.0f) & 0xFFFF;
      }
      return Px{ov[0], ov[1], ov[2], ov[3]};
    }
    case WRCU_BLEND_ADV_DIFFERENCE: {
      int sa = src.a, da = dst.a;
      int sv[4] = {src.b, src.g, src.r, src.a}, dv[4] = {dst.b, dst.g, dst.r, dst.a}, ov[4];
      for (int i = 0; i < 4; i++) {
        int diff = min(wr_muldiv255(dv[i], sa), wr_muldiv255(sv[i], da));
        ov[i] = (sv[i] + dv[i] - diff - (i < 3 ? diff : 0)) & 0xFFFF;
      }
      return Px{ov[0], ov[1], ov[2], ov[3]};
    }
    case WRCU_BLEND_ADV_EXCLUSION: {
      int sv[4] = {src.b, src.g, src.r, src.a}, dv[4] = {dst.b, dst.g, dst.r, dst.a}, ov[4];
      for (int i = 0; i < 4; i++) {
        int diff = wr_muldiv255(sv[i], dv[i]);
        ov[i] = (sv[i] + dv[i] - diff - (i < 3 ? diff : 0)) & 0xFFFF;
      }
      return Px{ov[0], ov[1], ov[2], ov[3]};
    }
    case WRCU_BLEND_ADV_HUE:
    case WRCU_BLEND_ADV_SATURATION:
    case WRCU_BLEND_ADV_COLOR:
    case WRCU_BLEND_ADV_LUMINOSITY: {
      float srcV[4] = {(float)src.r, (float)src.g, (float)src.b, (float)src.a};
      float dstV[4] = {(float)dst.r, (float)dst.g, (float)dst.b, (float)dst.a};
      float srcA = __fmul_rn(srcV[3], 1.0f / 255.0f);
      float dstA = __fmul_rn(dstV[3], 1.0f / 255.0f);
      float srcDstA = __fmul_rn(srcV[3], dstA);
      float srcC[3] = {__fmul_rn(srcV[0], dstA), __fmul_rn(srcV[1], dstA), __fmul_rn(srcV[2], dstA)};
      float dstC[3] = {__fmul_rn(dstV[0], srcA), __fmul_rn(dstV[1], srcA), __fmul_rn(dstV[2], srcA)};
      float rgb[3];
      if (key == WRCU_BLEND_ADV_HUE) wr_set_lum_sat(rgb, srcC, dstC, dstC, srcDstA);
      else if (key == WRCU_BLEND_ADV_SATURATION) wr_set_lum_sat(rgb, dstC, srcC, dstC, srcDstA);
      else if (key == WRCU_BLEND_ADV_COLOR) wr_set_lum(rgb, srcC, dstC, srcDstA);
      else wr_set_lum(rgb, dstC, srcC, srcDstA);
      float out[4];
      for (int i = 0; i < 3; i++)
        out[i] = __fsub_rn(__fadd_rn(__fsub_rn(__fadd_rn(rgb[i], srcV[i]), srcC[i]), dstV[i]), dstC[i]);
      out[3] = __fsub_rn(__fadd_rn(srcV[3], dstV[3]), srcDstA);
      o.r = wr_round_pixel(out[0], 1.0f) & 0xFFFF;
      o.g = wr_round_pixel(out[1], 1.0f) & 0xFFFF;
      o.b = wr_round_pixel(out[2], 1.0f) & 0xFFFF;
      o.a = wr_round_pixel(out[3], 1.0f) & 0xFFFF;
      return o;
    }
    case WRCU_BLEND__DROP_SHADOW: {  // SWGL_BLEND_DROP_SHADOW, blend.h:680-686
      Px color{wr_muldiv255(kc.b, src.a), wr_muldiv255(kc.g, src.a), wr_muldiv255(kc.r, src.a), wr_muldiv255(kc.a, src.a)};
      int ca = color.a;
      o.b = (color.b + dst.b - wr_muldiv255(dst.b, ca)) & 0xFFFF;
      o.g = (color.g + dst.g - wr_muldiv255(dst.g, ca)) & 0xFFFF;
      o.r = (color.r + dst.r - wr_muldiv255(dst.r, ca)) & 0xFFFF;
      o.a = (color.a + dst.a - wr_muldiv255(dst.a, ca)) & 0xFFFF;
      return o;
    }
    case WRCU_BLEND__SUBPIXEL_TEXT: {  // SWGL_BLEND_SUBPIXEL_TEXT, blend.h:688-692
      int ka = kc.a;
      o.b = (wr_muldiv255(kc.b, src.b) + dst.b - wr_muldiv255(dst.b, wr_muldiv255(ka, src.b))) & 0xFFFF;
      o.g = (wr_muldiv255(kc.g, src.g) + dst.g - wr_muldiv255(dst.g, wr_muldiv255(ka, src.g))) & 0xFFFF;
      o.r = (wr_muldiv255(kc.r, src.r) + dst.r - wr_muldiv255(dst.r, wr_muldiv255(ka, src.r))) & 0xFFFF;
      o.a = (wr_muldiv255(kc.a, src.a) + dst.a - wr_muldiv255(dst.a, wr_muldiv255(ka, src.a))) & 0xFFFF;
      return o;
    }
    default:
      return src;
  }
}

// R8 blend stage (blend.h:703-735)
WRD int wr_blend_r8(int key, int src, int dst) {
  switch (key) {
    case WRCU_BLEND_MULTIPLY: return wr_muldiv255(src, dst) & 0xFFFF;
    case WRCU_BLEND_PLUS_LIGHTER: return (src + dst) & 0xFFFF;
    default: return src;
  }
}

// ---- packed-pair fast paths ----------------------------------------------------
// dst, src as (rb, ga) pairs of 16-bit lanes, all lanes in [0,255].
// Premultiplied over: out = sat(src + dst - muldiv255(dst, sa)).
// With c = 255 - sa:  dst - ((dst*(sa+1))>>8) == (dst*c + 255) >> 8   (exact:
// dst - floor(t/256) = ceil((256*dst - t)/256) with t = dst*(sa+1)), so one
// multiply-add per lane pair.  Requires 0 <= sa <= 255.
WRD uint32_t wr_premult_over_pair(uint32_t dst_pair, uint32_t src_pair,
                                                         uint32_t c /*255-sa*/) {
  uint32_t t = dst_pair * c + 0x00FF00FFu;     // each lane <= 255*255+255 < 65536
  uint32_t m = __byte_perm(t, 0, 0x4341);      // (t >> 8) & 0x00FF00FF
  uint32_t s = m + src_pair;                   // lanes <= 510
  return __vminu2(s, 0x00FF00FFu);             // saturating pack
}

// Premultiplied over with `+ src` folded into the addend k = 255 + 256*src: exact when every source lane
// is <= src.a (the sum then cannot exceed 255).  See wr_fast_blend8.
WRD uint32_t wr_over_folded(uint32_t dst_pair, uint32_t c, uint32_t k) {
  return __byte_perm(dst_pair * c + k, 0, 0x4341);  // (t >> 8) & 0x00FF00FF
}

// One solid premultiplied-over layer on 8 pixels held as (B,R) / (G,A) pairs, with the layer's constants
// from wr_solid_consts.  VALID: every source lane <= src.a (BatchInfo::premul_valid), no saturation needed.
template <bool VALID>
WRD void wr_fast_blend8(uint32_t* rb, uint32_t* ga, uint32_t c, uint32_t krb, uint32_t kga) {
  if (VALID) {
#pragma unroll
    for (int p = 0; p < 8; p++) {
      rb[p] = wr_over_folded(rb[p], c, krb);
      ga[p] = wr_over_folded(ga[p], c, kga);
    }
  } else {
    const uint32_t srb = (krb - 0x00FF00FFu) >> 8, sga = (kga - 0x00FF00FFu) >> 8;
#pragma unroll
    for (int p = 0; p < 8; p++) {
      rb[p] = wr_premult_over_pair(rb[p], srb, c);
      ga[p] = wr_premult_over_pair(ga[p], sga, c);
    }
  }
}
