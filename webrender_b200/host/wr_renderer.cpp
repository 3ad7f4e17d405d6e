// wr_renderer.cpp — see wr_renderer.h.  Each method follows the control flow of
// its namesake in webrender/src/renderer/mod.rs and issues the wrcu calls that
// replace the GL calls there (INTEGRATION.md §2).
#include "wr_renderer.h"

#include <math.h>
#include <string.h>

#include <algorithm>

namespace wr {

// set_blend_mode_* (device/gl.rs:3901-4017) followed by SWGL's hash_blend_key
// (swgl/src/gl.cc:1240-1335) collapse to one key per mode.
int blend_key(BlendMode mode, MixBlendMode advanced) {
  switch (mode) {
    case BlendMode::None: return WRCU_BLEND_NONE;
    case BlendMode::Alpha: return WRCU_BLEND_ALPHA;
    case BlendMode::PremultipliedAlpha: return WRCU_BLEND_PREMULTIPLIED_ALPHA;
    case BlendMode::PremultipliedDestOut: return WRCU_BLEND_PREMULTIPLIED_DEST_OUT;
    case BlendMode::SubpixelDualSource: return WRCU_BLEND_SUBPIXEL_DUAL_SOURCE;
    case BlendMode::MultiplyDualSource: return WRCU_BLEND_SUBPIXEL_DUAL_SOURCE;
    // set_blend_mode_screen / _exclusion (ONE,1-SRC_COLOR / 1-DST_COLOR,1-SRC_COLOR) are not
    // among SWGL's blend keys (gl.cc:614-645): an is_software host advertises
    // KHR_blend_equation_advanced, so these modes arrive as BlendMode::Advanced instead
    // (BlendMode::from_mix_blend_mode, internal_types.rs).  -1 makes the draw fail loudly.
    case BlendMode::Screen: return -1;
    case BlendMode::Exclusion: return -1;
    case BlendMode::PlusLighter: return WRCU_BLEND_PLUS_LIGHTER;
    case BlendMode::Advanced:
      switch (advanced) {
        case MixBlendMode::Multiply: return WRCU_BLEND_ADV_MULTIPLY;
        case MixBlendMode::Screen: return WRCU_BLEND_ADV_SCREEN;
        case MixBlendMode::Overlay: return WRCU_BLEND_ADV_OVERLAY;
        case MixBlendMode::Darken: return WRCU_BLEND_ADV_DARKEN;
        case MixBlendMode::Lighten: return WRCU_BLEND_ADV_LIGHTEN;
        case MixBlendMode::ColorDodge: return WRCU_BLEND_ADV_COLOR_DODGE;
        case MixBlendMode::ColorBurn: return WRCU_BLEND_ADV_COLOR_BURN;
        case MixBlendMode::HardLight: return WRCU_BLEND_ADV_HARD_LIGHT;
        case MixBlendMode::SoftLight: return WRCU_BLEND_ADV_SOFT_LIGHT;
        case MixBlendMode::Difference: return WRCU_BLEND_ADV_DIFFERENCE;
        case MixBlendMode::Exclusion: return WRCU_BLEND_ADV_EXCLUSION;
        case MixBlendMode::Hue: return WRCU_BLEND_ADV_HUE;
        case MixBlendMode::Saturation: return WRCU_BLEND_ADV_SATURATION;
        case MixBlendMode::Color: return WRCU_BLEND_ADV_COLOR;
        case MixBlendMode::Luminosity: return WRCU_BLEND_ADV_LUMINOSITY;
        default: return WRCU_BLEND_PREMULTIPLIED_ALPHA;
      }
  }
  return WRCU_BLEND_NONE;
}

int batch_kind_to_wrcu(BatchKind kind) {
  switch (kind) {
    case BatchKind::QuadColorOrTexture: return WRCU_KIND_QUAD_TEXTURED;
    case BatchKind::QuadMask: return WRCU_KIND_QUAD_MASK;
    case BatchKind::BrushSolid: return WRCU_KIND_BRUSH_SOLID;
    case BatchKind::BrushImage: return WRCU_KIND_BRUSH_IMAGE;
    case BatchKind::BrushBlend: return WRCU_KIND_BRUSH_BLEND;
    case BatchKind::BrushMixBlend: return WRCU_KIND_BRUSH_MIX_BLEND;
    case BatchKind::BrushLinearGradient: return WRCU_KIND_BRUSH_LINEAR_GRADIENT;
    case BatchKind::BrushOpacity: return WRCU_KIND_BRUSH_OPACITY;
    case BatchKind::TextRun: return WRCU_KIND_TEXT_RUN;
    case BatchKind::QuadRadialGradient: return WRCU_KIND_QUAD_RADIAL_GRADIENT;
    case BatchKind::QuadConicGradient: return WRCU_KIND_QUAD_CONIC_GRADIENT;
    case BatchKind::BrushYuvImage: return WRCU_KIND_BRUSH_YUV_IMAGE;
    case BatchKind::SplitComposite: return WRCU_KIND_SPLIT_COMPOSITE;
  }
  return 0;
}

// Transform3D::ortho(0, w, 0, h, ORTHO_NEAR, ORTHO_FAR) (mod.rs:4705-4712; euclid), column major
static void ortho(float w, float h, float* m) {
  const float n = -100000.0f, f = 100000.0f;
  memset(m, 0, 16 * sizeof(float));
  m[0] = 2.0f / w;
  m[5] = 2.0f / h;
  m[10] = -2.0f / (f - n);
  m[12] = -1.0f;
  m[13] = -1.0f;
  m[14] = -(f + n) / (f - n);
  m[15] = 1.0f;
}

void Renderer::bind_draw_target(wrcu_tex color, wrcu_tex depth, int w, int h) {
  float proj[16];
  ortho((float)w, (float)h, proj);
  int32_t vp[4] = {0, 0, w, h};
  if (wrcu_target_bind(device, color, depth, proj, vp) != WRCU_OK) failed++;
}

void Renderer::draw_instanced_batch(int kind, uint32_t features, const void* instances, size_t stride, size_t n,
                                    const BatchTextures& textures, RendererStats& stats) {
  if (n == 0) return;
  for (int i = 0; i < 3; i++) state.color[i] = textures.colors[i];  // bind_textures (mod.rs:2030-2040)
  state.clip_mask = textures.clip_mask;
  if (wrcu_draw_batch(device, kind, features, &state, instances, stride, (int)n) != WRCU_OK) failed++;
  stats.total_draw_calls++;
}

void Renderer::draw_alpha_batch_container(const AlphaBatchContainer& c, bool has_depth, RendererStats& stats) {
  const bool uses_scissor = c.task_scissor_rect.has_value();
  state.scissor_enabled = uses_scissor ? 1 : 0;
  if (uses_scissor) {
    const DeviceIntRect& r = *c.task_scissor_rect;
    state.scissor[0] = r.x0; state.scissor[1] = r.y0; state.scissor[2] = r.x1 - r.x0; state.scissor[3] = r.y1 - r.y0;
  }
  if (!c.opaque_batches.empty()) {
    // set_blend(false); enable_depth(LessEqual); enable_depth_write
    state.blend = WRCU_BLEND_NONE;
    state.depth = has_depth ? WRCU_DEPTH_TEST_WRITE : WRCU_DEPTH_OFF;
    for (auto it = c.opaque_batches.rbegin(); it != c.opaque_batches.rend(); ++it)  // front to back
      draw_instanced_batch(batch_kind_to_wrcu(it->key.kind), it->features, it->instances.data(), it->instance_stride,
                           it->instances.size() / it->instance_stride, it->key.textures, stats);
    state.depth = has_depth ? WRCU_DEPTH_TEST : WRCU_DEPTH_OFF;  // disable_depth_write
  } else {
    state.depth = WRCU_DEPTH_OFF;  // disable_depth
  }
  if (!c.alpha_batches.empty()) {
    for (const PrimitiveBatch& b : c.alpha_batches) {
      if (b.key.blend_mode == BlendMode::None) {  // unreachable!("bug: opaque blend in alpha pass")
        renderer_errors.push_back("bug: opaque blend in alpha pass");
        failed++;
        continue;
      }
      state.blend = blend_key(b.key.blend_mode, b.key.advanced_mode);
      draw_instanced_batch(batch_kind_to_wrcu(b.key.kind), b.features | ALPHA_PASS, b.instances.data(),
                           b.instance_stride, b.instances.size() / b.instance_stride, b.key.textures, stats);
    }
    state.blend = WRCU_BLEND_NONE;
  }
  state.depth = WRCU_DEPTH_OFF;
  state.scissor_enabled = 0;
}

void Renderer::draw_picture_cache_target(const PictureCacheTarget& t, RendererStats& stats) {
  bind_draw_target(t.surface, t.depth, t.width, t.height);
  // clear_target(clear_color, Some(1.0), dirty rect) (mod.rs:2745-2750)
  int32_t rect[4] = {t.dirty_rect.x0, t.dirty_rect.y0, t.dirty_rect.x1 - t.dirty_rect.x0, t.dirty_rect.y1 - t.dirty_rect.y0};
  const bool whole = rect[2] <= 0 || rect[3] <= 0;
  float one = 1.0f;
  if (wrcu_clear(device, whole ? nullptr : rect, t.has_clear_color ? t.clear_color : nullptr,
                 t.depth ? &one : nullptr) != WRCU_OK) failed++;
  draw_alpha_batch_container(t.alpha_batch_container, t.depth != 0, stats);
}

void Renderer::draw_color_target(const ColorRenderTarget& t, RendererStats& stats) {
  stats.color_target_count++;
  bind_draw_target(t.texture, t.depth, t.width, t.height);
  state.blend = WRCU_BLEND_NONE;
  state.depth = WRCU_DEPTH_OFF;
  state.scissor_enabled = 0;
  // clear to transparent black (mod.rs:3560-3600): whole target, or the listed task rects
  const float zero[4] = {0, 0, 0, 0};
  float one = 1.0f;
  if (t.clears.empty()) {
    if (wrcu_clear(device, nullptr, zero, t.depth ? &one : nullptr) != WRCU_OK) failed++;
  } else {
    for (const DeviceIntRect& r : t.clears) {
      int32_t rect[4] = {r.x0, r.y0, r.x1 - r.x0, r.y1 - r.y0};
      if (wrcu_clear(device, rect, zero, t.depth ? &one : nullptr) != WRCU_OK) failed++;
    }
  }
  // blurs and scalings of this target (mod.rs:3607-3640)
  draw_blurs(t.vertical_blurs, true, stats);
  draw_blurs(t.horizontal_blurs, true, stats);
  handle_scaling(t.scalings, stats);
  // handle_prims (mod.rs:2199-2276): quad primitives of off-screen tasks, blending off
  for (const PrimitiveBatch& b : t.prim_batches)
    draw_instanced_batch(batch_kind_to_wrcu(b.key.kind), b.features, b.instances.data(), b.instance_stride,
                         b.instances.size() / b.instance_stride, b.key.textures, stats);
  // handle_clips (mod.rs:2278-2340): masks multiplied in
  if (!t.mask_batches.empty()) {
    state.blend = WRCU_BLEND_MULTIPLY;
    for (const PrimitiveBatch& b : t.mask_batches)
      draw_instanced_batch(batch_kind_to_wrcu(b.key.kind), b.features, b.instances.data(), b.instance_stride,
                           b.instances.size() / b.instance_stride, b.key.textures, stats);
    state.blend = WRCU_BLEND_NONE;
  }
  for (const AlphaBatchContainer& c : t.alpha_batch_containers) draw_alpha_batch_container(c, t.depth != 0, stats);
}

void Renderer::draw_clip_batch_list(const ClipBatchList& list, int blend, RendererStats& stats) {
  state.blend = blend;
  BatchTextures none = BatchTextures::empty();
  // draw rounded cornered rectangles (mod.rs:3703-3733)
  draw_instanced_batch(WRCU_KIND_CLIP_RECTANGLE, 0, list.slow_rectangles.data(), 200, list.slow_rectangles.size() / 200,
                       none, stats);
  draw_instanced_batch(WRCU_KIND_CLIP_RECTANGLE, FAST_PATH, list.fast_rectangles.data(), 200,
                       list.fast_rectangles.size() / 200, none, stats);
  // draw box-shadow clips (mod.rs:3735-3750)
  for (const auto& kv : list.box_shadows) {
    BatchTextures tex;
    tex.colors[0] = kv.first;
    draw_instanced_batch(WRCU_KIND_CLIP_BOX_SHADOW, TEXTURE_2D, kv.second.data(), 84, kv.second.size() / 84, tex, stats);
  }
}

void Renderer::draw_blurs(const BlurMap& blurs, bool color_target, RendererStats& stats) {
  for (const auto& kv : blurs) {
    BatchTextures tex;
    tex.colors[0] = kv.first;  // BatchTextures::composite_rgb(texture)
    draw_instanced_batch(WRCU_KIND_BLUR, color_target ? WRCU_FEAT_COLOR_TARGET : WRCU_FEAT_ALPHA_TARGET,
                         kv.second.data(), sizeof(BlurInstance), kv.second.size(), tex, stats);
  }
}

void Renderer::handle_scaling(const ScalingMap& scalings, RendererStats& stats) {
  for (const auto& kv : scalings) {
    BatchTextures tex;
    tex.colors[0] = kv.first;
    draw_instanced_batch(WRCU_KIND_SCALE, TEXTURE_2D, kv.second.data(), sizeof(ScalingInstance), kv.second.size(), tex,
                         stats);
  }
}

void Renderer::draw_alpha_target(const AlphaRenderTarget& t, RendererStats& stats) {
  stats.alpha_target_count++;
  bind_draw_target(t.texture, 0, t.width, t.height);
  state.depth = WRCU_DEPTH_OFF;
  state.scissor_enabled = 0;
  state.blend = WRCU_BLEND_NONE;
  const float zero[4] = {0, 0, 0, 0}, one[4] = {1, 1, 1, 1};
  for (const DeviceIntRect& r : t.zero_clears) {
    int32_t rect[4] = {r.x0, r.y0, r.x1 - r.x0, r.y1 - r.y0};
    if (wrcu_clear(device, rect, zero, nullptr) != WRCU_OK) failed++;
  }
  for (const DeviceIntRect& r : t.one_clears) {
    int32_t rect[4] = {r.x0, r.y0, r.x1 - r.x0, r.y1 - r.y0};
    if (wrcu_clear(device, rect, one, nullptr) != WRCU_OK) failed++;
  }
  // blurs: a standard two-pass separable implementation (mod.rs:3860-3884), then scalings
  draw_blurs(t.vertical_blurs, false, stats);
  draw_blurs(t.horizontal_blurs, false, stats);
  handle_scaling(t.scalings, stats);
  // primary clips overwrite (blend off), secondary clips multiply (mod.rs:3903-3918)
  draw_clip_batch_list(t.clip_batcher.primary_clips, WRCU_BLEND_NONE, stats);
  draw_clip_batch_list(t.clip_batcher.secondary_clips, WRCU_BLEND_MULTIPLY, stats);
  state.blend = WRCU_BLEND_NONE;
}

// draw_texture_cache_target (mod.rs:3931-4200): cached render tasks — clears, borders and line
// decorations (premultiplied-alpha blending on), gradients (blending off), horizontal blurs.
void Renderer::draw_texture_cache_target(const TextureCacheRenderTarget& t, RendererStats& stats) {
  bind_draw_target(t.texture, 0, t.width, t.height);
  state.depth = WRCU_DEPTH_OFF;
  state.scissor_enabled = 0;
  state.blend = WRCU_BLEND_NONE;
  const float zero[4] = {0, 0, 0, 0};
  for (const DeviceIntRect& r : t.clears) {
    int32_t rect[4] = {r.x0, r.y0, r.x1 - r.x0, r.y1 - r.y0};
    if (wrcu_clear(device, rect, zero, nullptr) != WRCU_OK) failed++;
  }
  const BatchTextures none;
  if (!t.border_segments_solid.empty() || !t.border_segments_complex.empty()) {
    state.blend = WRCU_BLEND_PREMULTIPLIED_ALPHA;
    if (!t.border_segments_solid.empty())
      draw_instanced_batch(WRCU_KIND_BORDER_SOLID, 0, t.border_segments_solid.data(), sizeof(BorderInstance),
                           t.border_segments_solid.size(), none, stats);
    if (!t.border_segments_complex.empty())
      draw_instanced_batch(WRCU_KIND_BORDER_SEGMENT, 0, t.border_segments_complex.data(), sizeof(BorderInstance),
                           t.border_segments_complex.size(), none, stats);
    state.blend = WRCU_BLEND_NONE;
  }
  if (!t.line_decorations.empty()) {
    state.blend = WRCU_BLEND_PREMULTIPLIED_ALPHA;
    draw_instanced_batch(WRCU_KIND_LINE_DECORATION, 0, t.line_decorations.data(), sizeof(LineDecorationJob),
                         t.line_decorations.size(), none, stats);
    state.blend = WRCU_BLEND_NONE;
  }
  if (!t.fast_linear_gradients.empty())
    draw_instanced_batch(WRCU_KIND_FAST_LINEAR_GRADIENT, 0, t.fast_linear_gradients.data(),
                         sizeof(FastLinearGradientInstance), t.fast_linear_gradients.size(), none, stats);
  if (!t.linear_gradients.empty())
    draw_instanced_batch(WRCU_KIND_LINEAR_GRADIENT, 0, t.linear_gradients.data(), sizeof(LinearGradientInstance),
                         t.linear_gradients.size(), none, stats);
  if (!t.radial_gradients.empty())
    draw_instanced_batch(WRCU_KIND_RADIAL_GRADIENT, 0, t.radial_gradients.data(), sizeof(RadialGradientInstance),
                         t.radial_gradients.size(), none, stats);
  if (!t.conic_gradients.empty())
    draw_instanced_batch(WRCU_KIND_CONIC_GRADIENT, 0, t.conic_gradients.data(), sizeof(ConicGradientInstance),
                         t.conic_gradients.size(), none, stats);
  draw_blurs(t.horizontal_blurs, true, stats);
}

void Renderer::draw_tile_list(const std::vector<CompositeTile>& tiles, const std::vector<occlusion::Item>& items,
                              int blend, RendererStats& stats) {
  // The reference breaks the instance list whenever the texture or the shader parameters change
  // (mod.rs:3289-3316) — a GL draw binds one sColor0.  wrcu_draw_composite_tiles carries the texture
  // per instance, so a run of tiles only breaks on the shader parameters (FAST_PATH; RGBA vs YUV).
  // Pieces of one tile never overlap, so a run of them stays a copy-engine batch (BatchInfo::all_copy).
  state.blend = blend;
  std::vector<CompositeInstance> instances;
  std::vector<wrcu_tex> textures;
  const CompositeTile* cur = nullptr;
  auto flush = [&]() {
    if (instances.empty()) return;
    if (cur->yuv) {  // get_composite_shader(CompositeSurfaceFormat::Yuv, ..) (shade.rs); planes in sColor0..2
      BatchTextures tex;
      tex.colors[0] = cur->texture;
      tex.colors[1] = cur->planes[0];
      tex.colors[2] = cur->planes[1];
      draw_instanced_batch(WRCU_KIND_COMPOSITE, TEXTURE_2D | WRCU_FEAT_YUV, instances.data(), sizeof(CompositeInstance),
                           instances.size(), tex, stats);
    } else {
      state.clip_mask = 0;
      if (wrcu_draw_composite_tiles(device, TEXTURE_2D | (cur->fast_path ? FAST_PATH : 0u), &state, instances.data(),
                                    sizeof(CompositeInstance), (int)instances.size(), textures.data()) != WRCU_OK)
        failed++;
      stats.total_draw_calls++;
    }
    instances.clear();
    textures.clear();
  };
  for (const occlusion::Item& item : items) {
    const CompositeTile* t = &tiles[item.key];
    bool brk = cur && (cur->fast_path != t->fast_path || cur->yuv != t->yuv);
    if (cur && t->yuv && !brk)
      brk = cur->texture != t->texture || cur->planes[0] != t->planes[0] || cur->planes[1] != t->planes[1];
    if (brk) flush();
    cur = t;
    CompositeInstance inst = t->instance;  // CompositeInstance::new(tile_rect, clip_rect = item.rectangle, ..)
    inst.v[4] = item.rectangle.x0; inst.v[5] = item.rectangle.y0;
    inst.v[6] = item.rectangle.x1; inst.v[7] = item.rectangle.y1;
    instances.push_back(inst);
    textures.push_back(t->texture);
  }
  flush();
}

static bool whole_pixels(const DeviceBox2D& r) {
  return floorf(r.x0) == r.x0 && floorf(r.y0) == r.y0 && floorf(r.x1) == r.x1 && floorf(r.y1) == r.y1;
}

void Renderer::composite_simple(const Frame& frame, const std::optional<PartialPresentMode>& partial_present_mode,
                                RendererStats& stats) {
  bind_draw_target(frame.framebuffer, 0, frame.fb_width, frame.fb_height);
  state.depth = WRCU_DEPTH_OFF;
  state.scissor_enabled = 0;
  const CompositeState& cs = frame.composite_state;
  // front to back (CompositeState::end_frame, composite.rs:1021), or as listed
  std::vector<size_t> order(cs.tiles.size());
  for (size_t i = 0; i < order.size(); i++) order[i] = i;
  if (!cs.listed)
    std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return cs.tiles[a].z_id < cs.tiles[b].z_id; });

  occlusion::FrontToBackBuilder occlusion;
  std::vector<occlusion::Item> opaque, clear_tiles, alpha;  // in draw order
  for (size_t idx : order) {
    const CompositeTile& tile = cs.tiles[idx];
    const DeviceBox2D device_tile_box = tile.device_box();
    const DeviceBox2D partial_clip_rect = partial_present_mode ? partial_present_mode->dirty_rect : device_tile_box;
    const DeviceBox2D rect = device_tile_box.intersection_unchecked(tile.clip_rect())
                                 .intersection_unchecked(partial_clip_rect)
                                 .intersection_unchecked(tile.valid_rect);
    if (rect.is_empty()) continue;
    // Clear tiles overwrite what is under them, but with their own blend state: drawn after the opaque
    // tiles and before the alpha ones, outside the occlusion lists.
    if (tile.kind == CompositeTileKind::Clear) clear_tiles.push_back(occlusion::Item{rect, idx});
    else if (cs.listed) (tile.kind == CompositeTileKind::Opaque ? opaque : alpha).push_back(occlusion::Item{rect, idx});
    else occlusion.add(rect, tile.kind == CompositeTileKind::Opaque, idx);
  }
  if (!cs.listed) {
    opaque = occlusion.opaque_items();
    alpha.assign(occlusion.alpha_items().rbegin(), occlusion.alpha_items().rend());  // back to front
  }

  // The reference clears the framebuffer, or the dirty rect unless it is fully hidden (mod.rs:3420-3445).
  // Of that region only what no opaque item covers is cleared: an opaque item with whole-pixel edges
  // writes every pixel of its rect with blending off, so clearing those pixels first changes nothing.
  // A fractional item may leave its edge pixels untouched, so its rect stays in the clear.
  if (cs.has_clear_color) {
    std::vector<DeviceBox2D> region;
    const DeviceBox2D fb{0.0f, 0.0f, (float)frame.fb_width, (float)frame.fb_height};
    if (!partial_present_mode) {
      region.push_back(fb);
    } else {
      const DeviceBox2D& d = partial_present_mode->dirty_rect;
      if (!d.is_empty() && (cs.listed || occlusion.test(d))) {  // DeviceRect::to_i32 truncates
        const DeviceBox2D di{(float)(int32_t)d.x0, (float)(int32_t)d.y0, (float)(int32_t)d.x1, (float)(int32_t)d.y1};
        const DeviceBox2D r = di.intersection_unchecked(fb);
        if (!r.is_empty()) region.push_back(r);
      }
    }
    for (const occlusion::Item& it : opaque) {
      if (region.empty()) break;
      if (whole_pixels(it.rectangle)) occlusion::apply_occluder(it.rectangle, region);
    }
    if (!region.empty()) {
      std::vector<int32_t> rects;
      for (const DeviceBox2D& r : region)
        rects.insert(rects.end(), {(int32_t)r.x0, (int32_t)r.y0, (int32_t)(r.x1 - r.x0), (int32_t)(r.y1 - r.y0)});
      if (wrcu_clear_rects(device, rects.data(), (int)region.size(), cs.clear_color) != WRCU_OK) failed++;
    }
  }

  // opaque items front to back with blending off, then clear tiles (dest-out), then alpha items back to
  // front (mod.rs:3447-3483)
  if (!opaque.empty()) draw_tile_list(cs.tiles, opaque, WRCU_BLEND_NONE, stats);
  if (!clear_tiles.empty()) draw_tile_list(cs.tiles, clear_tiles, WRCU_BLEND_PREMULTIPLIED_DEST_OUT, stats);
  if (!alpha.empty()) draw_tile_list(cs.tiles, alpha, WRCU_BLEND_PREMULTIPLIED_ALPHA, stats);
  state.blend = WRCU_BLEND_NONE;
}

void BufferDamageTracker::push_dirty_rect(const DeviceBox2D& rect) {
  damage_rects[current_offset] = rect;
  current_offset = current_offset == 0 ? 3 : current_offset - 1;
}

std::optional<DeviceBox2D> BufferDamageTracker::get_damage_rect(size_t buffer_age) const {
  if (buffer_age == 0) return std::nullopt;           // a new buffer: nothing in it is valid
  if (buffer_age == 1) return DeviceBox2D{};          // last frame's back buffer: all valid
  if (buffer_age > 5) return std::nullopt;            // older than the frames tracked
  DeviceBox2D r;                                      // the frames drawn since it was the back buffer
  for (size_t k = 0; k < buffer_age - 1; k++) r = r.union_with(damage_rects[(current_offset + 1 + k) % 4]);
  return r;
}

static DeviceBox2D round_box(const DeviceBox2D& r) {  // euclid Box2D::round
  return DeviceBox2D{floorf(r.x0 + 0.5f), floorf(r.y0 + 0.5f), floorf(r.x1 + 0.5f), floorf(r.y1 + 0.5f)};
}

// calculate_dirty_rects (mod.rs:4311-4416) for the Draw compositor with a partial-present interface
std::optional<PartialPresentMode> Renderer::calculate_dirty_rects(size_t buffer_age, const CompositeState& cs,
                                                                  int fb_width, int fb_height, RenderResults& results) {
  std::optional<PartialPresentMode> mode;
  if (partial_present.max_partial_present_rects <= 0) return mode;
  const bool draw_previous = partial_present.draw_previous_partial_present_regions;
  const DeviceBox2D fb_rect{0.0f, 0.0f, (float)fb_width, (float)fb_height};
  const DeviceBox2D prev_frames_damage_rect = buffer_damage_tracker.get_damage_rect(buffer_age).value_or(fb_rect);
  if (cs.dirty_rects_are_valid && !force_redraw) {
    DeviceBox2D combined;
    for (const CompositeTile& tile : cs.tiles) {
      if (tile.kind == CompositeTileKind::Clear) continue;
      const DeviceBox2D d = tile.dirty_rect.intersection_unchecked(fb_rect);
      if (!d.is_empty()) combined = combined.union_with(d);
    }
    combined = round_box(combined);
    if (!combined.is_empty())
      results.dirty_rects.push_back(DeviceIntRect{(int32_t)combined.x0, (int32_t)combined.y0, (int32_t)combined.x1,
                                                  (int32_t)combined.y1});
    if (draw_previous) buffer_damage_tracker.push_dirty_rect(combined);
    mode = PartialPresentMode{draw_previous ? combined.union_with(prev_frames_damage_rect) : combined};
  } else {
    results.dirty_rects.push_back(DeviceIntRect{0, 0, fb_width, fb_height});
    if (draw_previous) buffer_damage_tracker.push_dirty_rect(fb_rect);
  }
  force_redraw = false;
  return mode;
}

void Renderer::draw_frame(const Frame& frame, size_t buffer_age, RenderResults& results) {
  // bind_frame_data + gpu buffers + gpu cache (mod.rs:4418, 4551-4558) in one call
  if (wrcu_frame_begin(device, &frame.tables) != WRCU_OK) { failed++; return; }
  std::optional<PartialPresentMode> present_mode;
  if (frame.present)
    present_mode = calculate_dirty_rects(buffer_age, frame.composite_state, frame.fb_width, frame.fb_height, results);
  for (const RenderPass& pass : frame.passes) {
    for (const TextureCacheRenderTarget& t : pass.texture_cache) draw_texture_cache_target(t, results.stats);
    for (const PictureCacheTarget& t : pass.picture_cache) draw_picture_cache_target(t, results.stats);
    for (const AlphaRenderTarget& t : pass.alpha) draw_alpha_target(t, results.stats);
    for (const ColorRenderTarget& t : pass.color) draw_color_target(t, results.stats);
  }
  if (frame.present) composite_simple(frame, present_mode, results.stats);
  else force_redraw = true;  // a frame drawn but not presented leaves the partial-present state unknown (mod.rs:4914)
  if (wrcu_frame_end(device) != WRCU_OK) failed++;
}

// update_gpu_cache (mod.rs:1498-1535): every pending list goes to the device in order; the cache
// persists there (wrcu_gpu_cache_update), so a frame carries only the blocks that changed.
void Renderer::update_gpu_cache() {
  for (const GpuCacheUpdateList& list : pending_gpu_cache_updates) {
    static_assert(sizeof(GpuCacheUpdate) == sizeof(wrcu_gpu_cache_copy), "GpuCacheUpdate layout");
    bool clear = list.clear || pending_gpu_cache_clear;
    pending_gpu_cache_clear = false;
    if (wrcu_gpu_cache_update(device, list.height, clear ? 1 : 0, (const wrcu_gpu_cache_copy*)list.updates.data(),
                              list.updates.size(), list.blocks.empty() ? nullptr : list.blocks[0].data,
                              list.blocks.size()) != WRCU_OK)
      failed++;
  }
  pending_gpu_cache_updates.clear();
}

// update_texture_cache (mod.rs:1795-1990): copies between cache textures first (defragmentation),
// then each texture's updates as ONE batched upload — the rows are packed into a staging blob the
// way upload_to_texture_cache packs them into PBO staging buffers (renderer/upload.rs:67-330).
void Renderer::update_texture_cache() {
  for (const TextureUpdateList& list : pending_texture_updates) {
    for (const auto& kv : list.copies)
      for (const TextureCacheCopy& cp : kv.second) {
        int32_t r[4] = {cp.src_rect.x0, cp.src_rect.y0, cp.src_rect.x1 - cp.src_rect.x0, cp.src_rect.y1 - cp.src_rect.y0};
        if (wrcu_texture_copy(device, kv.first.first, kv.first.second, r, cp.dst_rect.x0, cp.dst_rect.y0) != WRCU_OK) failed++;
      }
    for (const auto& kv : list.updates) {
      std::vector<wrcu_upload_rect> rects;
      std::vector<uint8_t> staging;
      for (const TextureCacheUpdate& u : kv.second) {
        const int w = u.rect.x1 - u.rect.x0, h = u.rect.y1 - u.rect.y0;
        if (w <= 0 || h <= 0 || !u.data) continue;
        // rows are repacked at a 16-byte aligned offset and pitch (only the rect's bytes are read)
        const size_t row = (size_t)w * u.bytes_per_pixel, pitch = (row + 15) & ~(size_t)15;
        size_t off = (staging.size() + 15) & ~(size_t)15;
        staging.resize(off + pitch * (size_t)h);
        for (int y = 0; y < h; y++) memcpy(staging.data() + off + pitch * (size_t)y, u.data + u.stride * (size_t)y, row);
        rects.push_back(wrcu_upload_rect{u.rect.x0, u.rect.y0, w, h, (uint64_t)off, (uint64_t)pitch});
      }
      if (!rects.empty() &&
          wrcu_texture_upload_batch(device, kv.first, rects.data(), rects.size(), staging.data(), staging.size()) != WRCU_OK)
        failed++;
    }
  }
  pending_texture_updates.clear();
}

RendererError Renderer::check_gl_errors() {
  int e = wrcu_get_error(device);
  if (e == WRCU_ERR_OOM) return RendererError::OutOfMemory;
  if (e != WRCU_OK || failed) {
    const char* msg = wrcu_last_error_string(device);
    renderer_errors.push_back(msg ? msg : "wrcu error");
    failed = 0;
    return RendererError::SoftwareRasterizer;
  }
  return RendererError::None;
}

RendererError Renderer::render(const Frame& frame, size_t buffer_age, RenderResults* results) {
  RenderResults local;
  // render_impl (mod.rs:1441-1560): resource updates first, then the frame
  update_texture_cache();
  update_gpu_cache();
  draw_frame(frame, buffer_age, results ? *results : local);
  return check_gl_errors();
}

RendererError Renderer::render(const Frame& frame, RendererStats* stats) {
  RenderResults results;
  RendererError e = render(frame, 0, &results);
  if (stats) *stats = results.stats;
  return e;
}

}  // namespace wr

// ---- flat C binding so a harness (tests, a Rust shim) can build a wr::Frame ---------------------
using namespace wr;
extern "C" {
Renderer* wrh_renderer_create(wrcu_ctx* device) { return new Renderer(device); }
void wrh_renderer_destroy(Renderer* r) { delete r; }
Frame* wrh_frame_create(const wrcu_frame_tables* tables) {
  Frame* f = new Frame();
  f->tables = *tables;
  return f;
}
void wrh_frame_destroy(Frame* f) { delete f; }
int wrh_frame_add_pass(Frame* f) { f->passes.emplace_back(); return (int)f->passes.size() - 1; }

// targets: returns the index within its list
int wrh_pass_add_picture_cache_target(Frame* f, int pass, wrcu_tex surface, wrcu_tex depth, int w, int h,
                                      const float* clear_color, const int32_t* dirty_rect) {
  PictureCacheTarget t;
  t.surface = surface; t.depth = depth; t.width = w; t.height = h;
  if (clear_color) { t.has_clear_color = true; memcpy(t.clear_color, clear_color, 16); }
  if (dirty_rect) t.dirty_rect = DeviceIntRect{dirty_rect[0], dirty_rect[1], dirty_rect[2], dirty_rect[3]};
  f->passes[pass].picture_cache.push_back(t);
  return (int)f->passes[pass].picture_cache.size() - 1;
}
int wrh_pass_add_color_target(Frame* f, int pass, wrcu_tex texture, wrcu_tex depth, int w, int h) {
  ColorRenderTarget t;
  t.texture = texture; t.depth = depth; t.width = w; t.height = h;
  f->passes[pass].color.push_back(t);
  return (int)f->passes[pass].color.size() - 1;
}
int wrh_pass_add_alpha_target(Frame* f, int pass, wrcu_tex texture, int w, int h) {
  AlphaRenderTarget t;
  t.texture = texture; t.width = w; t.height = h;
  f->passes[pass].alpha.push_back(t);
  return (int)f->passes[pass].alpha.size() - 1;
}
int wrh_pass_add_texture_cache_target(Frame* f, int pass, wrcu_tex texture, int w, int h) {
  TextureCacheRenderTarget t;
  t.texture = texture; t.width = w; t.height = h;
  f->passes[pass].texture_cache.push_back(t);
  return (int)f->passes[pass].texture_cache.size() - 1;
}
void wrh_texture_cache_target_add_clear(Frame* f, int pass, int target, const int32_t* rect) {
  f->passes[pass].texture_cache[target].clears.push_back(DeviceIntRect{rect[0], rect[1], rect[2], rect[3]});
}
// kind: the WRCU_KIND_* of the task list the instances go to
int wrh_texture_cache_target_add_tasks(Frame* f, int pass, int target, int kind, const void* instances, int n) {
  TextureCacheRenderTarget& t = f->passes[pass].texture_cache[target];
#define WRH_APPEND(vec, T) { const T* p = (const T*)instances; (vec).insert((vec).end(), p, p + n); return 0; }
  switch (kind) {
    case WRCU_KIND_BORDER_SOLID: WRH_APPEND(t.border_segments_solid, BorderInstance)
    case WRCU_KIND_BORDER_SEGMENT: WRH_APPEND(t.border_segments_complex, BorderInstance)
    case WRCU_KIND_LINE_DECORATION: WRH_APPEND(t.line_decorations, LineDecorationJob)
    case WRCU_KIND_FAST_LINEAR_GRADIENT: WRH_APPEND(t.fast_linear_gradients, FastLinearGradientInstance)
    case WRCU_KIND_LINEAR_GRADIENT: WRH_APPEND(t.linear_gradients, LinearGradientInstance)
    case WRCU_KIND_RADIAL_GRADIENT: WRH_APPEND(t.radial_gradients, RadialGradientInstance)
    case WRCU_KIND_CONIC_GRADIENT: WRH_APPEND(t.conic_gradients, ConicGradientInstance)
    default: return -1;
  }
#undef WRH_APPEND
}
static PrimitiveBatch make_batch(int kind, int blend_mode, int advanced, uint32_t features, const uint32_t* textures,
                                 const void* instances, size_t stride, int n) {
  PrimitiveBatch b;
  b.key.kind = (BatchKind)kind;
  b.key.blend_mode = (BlendMode)blend_mode;
  b.key.advanced_mode = (MixBlendMode)advanced;
  for (int i = 0; i < 3; i++) b.key.textures.colors[i] = textures[i];
  b.key.textures.clip_mask = textures[3];
  b.features = features;
  b.instance_stride = stride;
  b.instances.assign((const uint8_t*)instances, (const uint8_t*)instances + stride * (size_t)n);
  return b;
}
// list: 0 = opaque_batches, 1 = alpha_batches of a picture-cache target's container
void wrh_picture_target_add_batch(Frame* f, int pass, int target, int list, int kind, int blend_mode, int advanced,
                                  uint32_t features, const uint32_t* textures4, const void* instances, size_t stride,
                                  int n) {
  AlphaBatchContainer& c = f->passes[pass].picture_cache[target].alpha_batch_container;
  (list == 0 ? c.opaque_batches : c.alpha_batches)
      .push_back(make_batch(kind, blend_mode, advanced, features, textures4, instances, stride, n));
}
// list: 0 = prim_batches (blend off), 1 = mask_batches (multiply), 2 = alpha batches of container 0
void wrh_color_target_add_batch(Frame* f, int pass, int target, int list, int kind, int blend_mode, int advanced,
                                uint32_t features, const uint32_t* textures4, const void* instances, size_t stride,
                                int n) {
  ColorRenderTarget& t = f->passes[pass].color[target];
  PrimitiveBatch b = make_batch(kind, blend_mode, advanced, features, textures4, instances, stride, n);
  if (list == 0) t.prim_batches.push_back(b);
  else if (list == 1) t.mask_batches.push_back(b);
  else {
    if (t.alpha_batch_containers.empty()) t.alpha_batch_containers.emplace_back();
    t.alpha_batch_containers[0].alpha_batches.push_back(b);
  }
}
void wrh_alpha_target_add_clear(Frame* f, int pass, int target, int one, const int32_t* rect) {
  AlphaRenderTarget& t = f->passes[pass].alpha[target];
  (one ? t.one_clears : t.zero_clears).push_back(DeviceIntRect{rect[0], rect[1], rect[2], rect[3]});
}
// which: 0 = primary, 1 = secondary; shape: 0 = slow rects, 1 = fast rects, 2 = box shadows (texture)
void wrh_alpha_target_add_clips(Frame* f, int pass, int target, int which, int shape, wrcu_tex texture,
                                const void* instances, size_t stride, int n) {
  ClipBatcher& cb = f->passes[pass].alpha[target].clip_batcher;
  ClipBatchList& l = which == 0 ? cb.primary_clips : cb.secondary_clips;
  std::vector<uint8_t>& v = shape == 0 ? l.slow_rectangles : shape == 1 ? l.fast_rectangles : l.box_shadows[texture];
  v.insert(v.end(), (const uint8_t*)instances, (const uint8_t*)instances + stride * (size_t)n);
}
// target_kind: 0 = alpha target, 1 = colour target; which: 0 = vertical_blurs, 1 = horizontal_blurs, 2 = scalings
void wrh_target_add_blur_or_scale(Frame* f, int pass, int target_kind, int target, int which, wrcu_tex source,
                                  const void* instances, int n) {
  BlurMap* vb; BlurMap* hb; ScalingMap* sc;
  if (target_kind == 0) {
    AlphaRenderTarget& t = f->passes[pass].alpha[target];
    vb = &t.vertical_blurs; hb = &t.horizontal_blurs; sc = &t.scalings;
  } else {
    ColorRenderTarget& t = f->passes[pass].color[target];
    vb = &t.vertical_blurs; hb = &t.horizontal_blurs; sc = &t.scalings;
  }
  if (which == 2) {
    const ScalingInstance* p = (const ScalingInstance*)instances;
    (*sc)[source].insert((*sc)[source].end(), p, p + n);
  } else {
    const BlurInstance* p = (const BlurInstance*)instances;
    BlurMap& m = which == 0 ? *vb : *hb;
    m[source].insert(m[source].end(), p, p + n);
  }
}
void wrh_frame_set_framebuffer(Frame* f, wrcu_tex fb, int w, int h, const float* clear_color) {
  f->framebuffer = fb; f->fb_width = w; f->fb_height = h; f->present = true;
  f->composite_state.has_clear_color = clear_color != nullptr;
  if (clear_color) memcpy(f->composite_state.clear_color, clear_color, 16);
}
// Tiles added by these two are drawn as listed, unsplit: opaque tiles in the order added, then clear
// tiles, then alpha tiles, each in the order added (a flat frame's painter's order).  Their valid and
// dirty rects are the instance's rect clipped to its clip rect.
static void add_listed_tile(Frame* f, CompositeTile& t) {
  t.valid_rect = t.dirty_rect = t.device_box().intersection_unchecked(t.clip_rect());
  f->composite_state.listed = true;
  f->composite_state.tiles.push_back(t);
}
void wrh_frame_add_composite_tile(Frame* f, int kind, wrcu_tex texture, int fast_path, const float* instance30) {
  CompositeTile t;
  t.kind = (CompositeTileKind)kind;
  t.texture = texture;
  t.fast_path = fast_path != 0;
  memcpy(t.instance.v, instance30, sizeof t.instance.v);
  add_listed_tile(f, t);
}
void wrh_frame_add_composite_yuv_tile(Frame* f, int kind, const wrcu_tex* planes3, const float* instance30) {
  CompositeTile t;
  t.kind = (CompositeTileKind)kind;
  t.texture = planes3[0];
  t.yuv = true;
  t.planes[0] = planes3[1];
  t.planes[1] = planes3[2];
  memcpy(t.instance.v, instance30, sizeof t.instance.v);
  add_listed_tile(f, t);
}
// A tile of the composite state with its place and rects given (CompositeTile, composite.rs):
//   kind: 0 opaque, 1 clear, 2 alpha; yuv = 0: planes3[0] is the RGBA texture (fast_path as above),
//   yuv = 1: planes3 are the three planes; instance30: the CompositeInstance, whose rect is the device
//   tile box and whose clip rect the tile's device clip rect; z_id: tiles are drawn in ascending z_id,
//   front to back (ties keep the order of addition); valid_rect4 / dirty_rect4: x0, y0, x1, y1 in
//   device pixels, NULL = the instance's rect clipped to its clip rect.
void wrh_composite_state_add_tile(Frame* f, int kind, const wrcu_tex* planes3, int yuv, int fast_path,
                                  const float* instance30, int32_t z_id, const float* valid_rect4,
                                  const float* dirty_rect4) {
  CompositeTile t;
  t.kind = (CompositeTileKind)kind;
  t.texture = planes3[0];
  t.yuv = yuv != 0;
  if (t.yuv) { t.planes[0] = planes3[1]; t.planes[1] = planes3[2]; }
  t.fast_path = !t.yuv && fast_path != 0;
  memcpy(t.instance.v, instance30, sizeof t.instance.v);
  t.z_id = z_id;
  const DeviceBox2D drawn = t.device_box().intersection_unchecked(t.clip_rect());
  t.valid_rect = valid_rect4 ? DeviceBox2D{valid_rect4[0], valid_rect4[1], valid_rect4[2], valid_rect4[3]} : drawn;
  t.dirty_rect = dirty_rect4 ? DeviceBox2D{dirty_rect4[0], dirty_rect4[1], dirty_rect4[2], dirty_rect4[3]} : drawn;
  f->composite_state.tiles.push_back(t);
}
void wrh_composite_state_set_dirty_rects_are_valid(Frame* f, int valid) {
  f->composite_state.dirty_rects_are_valid = valid != 0;
}
// CompositorConfig::Draw's max_partial_present_rects / draw_previous_partial_present_regions
void wrh_renderer_set_partial_present(Renderer* r, int max_partial_present_rects,
                                      int draw_previous_partial_present_regions) {
  r->partial_present.max_partial_present_rects = max_partial_present_rects;
  r->partial_present.draw_previous_partial_present_regions = draw_previous_partial_present_regions != 0;
}
// Renderer::render with the back buffer's age.  Up to `cap` dirty rects (x0, y0, x1, y1) go to
// dirty_rects4; *n_dirty receives how many the frame has.  Returns RendererError as int.
int wrh_renderer_render_with_age(Renderer* r, const Frame* f, uint64_t buffer_age, uint64_t* draw_calls,
                                 int32_t* dirty_rects4, int cap, int* n_dirty) {
  RenderResults results;
  RendererError e = r->render(*f, (size_t)buffer_age, &results);
  if (draw_calls) *draw_calls = results.stats.total_draw_calls;
  if (n_dirty) *n_dirty = (int)results.dirty_rects.size();
  for (int i = 0; i < cap && i < (int)results.dirty_rects.size(); i++) {
    const DeviceIntRect& d = results.dirty_rects[(size_t)i];
    dirty_rects4[4 * i] = d.x0; dirty_rects4[4 * i + 1] = d.y0; dirty_rects4[4 * i + 2] = d.x1; dirty_rects4[4 * i + 3] = d.y1;
  }
  return (int)e;
}
// Test hook: FrontToBackBuilder over n rects (x0, y0, x1, y1) added front to back, rect i opaque when
// opaque[i].  visible[i] receives test(rect i) just before add(rect i), visible[n + i] what add returned.
// The opaque items, then the alpha items, go to keys / items4 (at most cap); returns how many items there
// are in all, with the opaque count in *n_opaque.
int wrh_occlusion_build(const float* rects4, const int32_t* opaque, int n, int32_t* visible, int32_t* keys,
                        float* items4, int cap, int* n_opaque) {
  occlusion::FrontToBackBuilder b;
  for (int i = 0; i < n; i++) {
    const DeviceBox2D r{rects4[4 * i], rects4[4 * i + 1], rects4[4 * i + 2], rects4[4 * i + 3]};
    visible[i] = b.test(r) ? 1 : 0;
    visible[n + i] = b.add(r, opaque[i] != 0, (size_t)i) ? 1 : 0;
  }
  std::vector<occlusion::Item> all(b.opaque_items());
  all.insert(all.end(), b.alpha_items().begin(), b.alpha_items().end());
  *n_opaque = (int)b.opaque_items().size();
  for (int i = 0; i < cap && i < (int)all.size(); i++) {
    keys[i] = (int32_t)all[(size_t)i].key;
    const DeviceBox2D& r = all[(size_t)i].rectangle;
    items4[4 * i] = r.x0; items4[4 * i + 1] = r.y0; items4[4 * i + 2] = r.x1; items4[4 * i + 3] = r.y1;
  }
  return (int)all.size();
}
// returns RendererError as int; *draw_calls receives RendererStats.total_draw_calls
// update path: queue a GpuCacheUpdateList / texture updates for the next render
void wrh_renderer_queue_gpu_cache_updates(Renderer* r, int height, int clear, const wrcu_gpu_cache_copy* updates, int n_updates,
                                          const float* blocks, int n_blocks) {
  GpuCacheUpdateList l;
  l.clear = clear != 0;
  l.height = height;
  for (int i = 0; i < n_updates; i++)
    l.updates.push_back(GpuCacheUpdate{updates[i].block_index, updates[i].block_count, GpuCacheAddress{updates[i].u, updates[i].v}});
  l.blocks.resize((size_t)n_blocks);
  if (n_blocks) memcpy(l.blocks.data(), blocks, (size_t)n_blocks * 16);
  r->pending_gpu_cache_updates.push_back(std::move(l));
}
// `data` must stay valid until the next wrh_renderer_render
void wrh_renderer_queue_texture_update(Renderer* r, wrcu_tex texture, const int32_t* rect, const void* data, size_t stride,
                                       int bytes_per_pixel) {
  if (r->pending_texture_updates.empty()) r->pending_texture_updates.emplace_back();
  TextureCacheUpdate u;
  u.rect = DeviceIntRect{rect[0], rect[1], rect[2], rect[3]};
  u.data = (const uint8_t*)data;
  u.stride = stride;
  u.bytes_per_pixel = (uint32_t)bytes_per_pixel;
  r->pending_texture_updates.back().updates[texture].push_back(u);
}
void wrh_renderer_queue_texture_copy(Renderer* r, wrcu_tex src, wrcu_tex dst, const int32_t* src_rect, const int32_t* dst_rect) {
  if (r->pending_texture_updates.empty()) r->pending_texture_updates.emplace_back();
  TextureCacheCopy c;
  c.src_rect = DeviceIntRect{src_rect[0], src_rect[1], src_rect[2], src_rect[3]};
  c.dst_rect = DeviceIntRect{dst_rect[0], dst_rect[1], dst_rect[2], dst_rect[3]};
  r->pending_texture_updates.back().copies[std::make_pair(src, dst)].push_back(c);
}
int wrh_renderer_render(Renderer* r, const Frame* f, uint64_t* draw_calls) {
  RendererStats stats;
  RendererError e = r->render(*f, &stats);
  if (draw_calls) *draw_calls = stats.total_draw_calls;
  return (int)e;
}
const char* wrh_renderer_last_error(Renderer* r) {
  return r->renderer_errors.empty() ? "" : r->renderer_errors.back().c_str();
}
}
