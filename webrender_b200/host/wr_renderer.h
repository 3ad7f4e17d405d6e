// wr_renderer.h — host-side mirror of the reference's frame-draw driver
// (webrender/src/renderer/mod.rs) above the wrcu C ABI.
//
// The reference's `Renderer` is Rust; there is no Rust toolchain in this image,
// so the same operator interface is restated in C++: same type and method names,
// same argument meaning, same error behaviour (sticky GL-style errors polled by
// check_gl_errors, mod.rs:1992).  Only the members the draw path reads are
// mirrored; everything is plain data so a binding can fill it directly.
#pragma once
#include <stdint.h>

#include <map>
#include <utility>
#include <optional>
#include <string>
#include <vector>

#include "../../include/wrcu.h"
#include "occlusion.h"

namespace wr {

struct DeviceIntRect { int32_t x0, y0, x1, y1; };  // min/max corners (units.rs)

// internal_types.rs BlendMode → the GL state set by set_blend_mode_* (device/gl.rs:3901-4017)
enum class BlendMode {
  None, Alpha, PremultipliedAlpha, PremultipliedDestOut, SubpixelDualSource, Advanced, MultiplyDualSource,
  Screen, Exclusion, PlusLighter,
};
enum class MixBlendMode {  // api/src/display_item.rs:1251-1270 (only used with BlendMode::Advanced)
  Normal, Multiply, Screen, Overlay, Darken, Lighten, ColorDodge, ColorBurn, HardLight, SoftLight, Difference,
  Exclusion, Hue, Saturation, Color, Luminosity, PlusLighter,
};

// batch.rs:56-130
enum class BatchKind {
  QuadColorOrTexture, QuadMask, BrushSolid, BrushImage, BrushBlend, BrushMixBlend, BrushLinearGradient,
  BrushOpacity, TextRun,
  QuadRadialGradient, QuadConicGradient,  // BatchKind::Quad(PatternKind::RadialGradient / ConicGradient), pattern.rs
  BrushYuvImage,                          // BatchKind::Brush(BrushBatchKind::YuvImage(..)), batch.rs:60-86
  SplitComposite,                         // BatchKind::SplitComposite (batch.rs:74): plane-split preserve-3d polygons
};
// batch.rs BatchFeatures / shade.rs feature strings
enum BatchFeatures : uint32_t {
  ALPHA_PASS = WRCU_FEAT_ALPHA_PASS, ANTIALIASING = WRCU_FEAT_ANTIALIASING, REPETITION = WRCU_FEAT_REPETITION,
  DUAL_SOURCE_BLENDING = WRCU_FEAT_DUAL_SOURCE_BLENDING, ADVANCED_BLEND = WRCU_FEAT_ADVANCED_BLEND,
  FAST_PATH = WRCU_FEAT_FAST_PATH, TEXTURE_2D = WRCU_FEAT_TEXTURE_2D,
};

struct BatchTextures {  // batch.rs:150-230: input colours + clip mask
  wrcu_tex colors[3] = {0, 0, 0};
  wrcu_tex clip_mask = 0;
  static BatchTextures empty() { return BatchTextures(); }
};
struct BatchKey {  // batch.rs:233-237
  BatchKind kind = BatchKind::BrushSolid;
  BlendMode blend_mode = BlendMode::None;
  MixBlendMode advanced_mode = MixBlendMode::Normal;
  BatchTextures textures;
};
struct PrimitiveInstanceData { int32_t data[4]; };  // gpu_types.rs:254-256
struct MaskInstance { int32_t prim[4]; int32_t clip[4]; };  // gpu_types.rs:614-624
struct PrimitiveBatch {  // batch.rs:504-508
  BatchKey key;
  std::vector<uint8_t> instances;  // PrimitiveInstanceData (16 B) or MaskInstance (32 B) records
  size_t instance_stride = 16;
  uint32_t features = 0;
};
struct AlphaBatchContainer {  // batch.rs:549-558
  std::vector<PrimitiveBatch> opaque_batches;  // in batch order; drawn reversed (front to back)
  std::vector<PrimitiveBatch> alpha_batches;
  std::optional<DeviceIntRect> task_scissor_rect;
};

// batch.rs:3596-3606
struct ClipBatchList {
  std::vector<uint8_t> slow_rectangles, fast_rectangles;  // ClipMaskInstanceRect, 200 B each
  std::map<wrcu_tex, std::vector<uint8_t>> box_shadows;    // ClipMaskInstanceBoxShadow, 84 B each, per source texture
};
struct ClipBatcher { ClipBatchList primary_clips, secondary_clips; };

struct PictureCacheTarget {  // render_target.rs:707-713
  wrcu_tex surface = 0, depth = 0;
  int32_t width = 0, height = 0;
  AlphaBatchContainer alpha_batch_container;
  std::optional<float> clear_depth;
  bool has_clear_color = false;
  float clear_color[4] = {0, 0, 0, 0};
  DeviceIntRect dirty_rect = {0, 0, 0, 0};
};
struct BlurInstance { int32_t task_address, src_task_address, blur_direction; float blur_std_deviation, blur_region[2]; };  // gpu_types.rs:112-118
struct ScalingInstance { float target_rect[4], source_rect[4], source_rect_type; };  // gpu_types.rs:124-128
typedef std::map<wrcu_tex, std::vector<BlurInstance>> BlurMap;      // keyed by source texture
typedef std::map<wrcu_tex, std::vector<ScalingInstance>> ScalingMap;

struct ColorRenderTarget {  // render_target.rs:215-238 (members the path reads)
  wrcu_tex texture = 0, depth = 0;
  int32_t width = 0, height = 0;
  BlurMap vertical_blurs, horizontal_blurs;
  ScalingMap scalings;
  std::vector<AlphaBatchContainer> alpha_batch_containers;
  std::vector<PrimitiveBatch> prim_batches;  // quad prims into off-screen tasks (handle_prims, mod.rs:2199), blend off
  std::vector<PrimitiveBatch> mask_batches;  // ps_quad_mask multiplied in (handle_clips, mod.rs:2278)
  std::vector<DeviceIntRect> clears;         // cleared to transparent black
};
struct AlphaRenderTarget {  // render_target.rs:522-532
  wrcu_tex texture = 0;
  int32_t width = 0, height = 0;
  ClipBatcher clip_batcher;
  std::vector<DeviceIntRect> zero_clears, one_clears;
  BlurMap vertical_blurs, horizontal_blurs;
  ScalingMap scalings;
};
// Instances of the render tasks drawn into texture-cache targets (the records travel as raw bytes:
// BorderInstance 108 B gpu_types.rs:193-202, LineDecorationJob 36 B render_target.rs:1184-1190,
// Fast/Linear/Radial/ConicGradientInstance 52/48/52/52 B prim_store/gradient/*.rs)
struct BorderInstance { float task_origin[2], local_rect[4], color0[4], color1[4]; int32_t flags; float widths[2], radius[2], clip_params[8]; };
struct LineDecorationJob { float task_rect[4], local_size[2], wavy_line_thickness; int32_t style; float axis_select; };
struct FastLinearGradientInstance { float task_rect[4], color0[4], color1[4], axis_select; };
struct LinearGradientInstance { float task_rect[4], start[2], end[2], scale[2]; int32_t extend_mode, gradient_stops_address; };
struct RadialGradientInstance { float task_rect[4], center[2], scale[2], start_radius, end_radius, ratio_xy; int32_t extend_mode, gradient_stops_address; };
struct ConicGradientInstance { float task_rect[4], center[2], scale[2], start_offset, end_offset, angle; int32_t extend_mode, gradient_stops_address; };
struct TextureCacheRenderTarget {  // render_target.rs:717-729
  wrcu_tex texture = 0;
  int32_t width = 0, height = 0;
  BlurMap horizontal_blurs;
  std::vector<BorderInstance> border_segments_complex, border_segments_solid;
  std::vector<DeviceIntRect> clears;
  std::vector<LineDecorationJob> line_decorations;
  std::vector<FastLinearGradientInstance> fast_linear_gradients;
  std::vector<LinearGradientInstance> linear_gradients;
  std::vector<RadialGradientInstance> radial_gradients;
  std::vector<ConicGradientInstance> conic_gradients;
};
struct RenderPass {  // render_task_graph.rs:854-861
  std::vector<TextureCacheRenderTarget> texture_cache;
  std::vector<AlphaRenderTarget> alpha;
  std::vector<ColorRenderTarget> color;
  std::vector<PictureCacheTarget> picture_cache;
};

// composite.rs: the tiles composite_simple draws
struct CompositeInstance { float v[30]; };  // gpu_types.rs:288-310, 120 B
enum class CompositeTileKind { Opaque, Clear, Alpha };
struct CompositeTile {
  CompositeTileKind kind = CompositeTileKind::Opaque;
  wrcu_tex texture = 0;   // picture-cache texture, external surface, or the 1x1 dummy
  CompositeInstance instance;  // v[0..3] the device tile box, v[4..7] its device clip rect
  bool fast_path = false; // NO_UV_CLAMP | NO_COLOR_MODULATION (composite.rs get_rgb_features)
  // ResolvedExternalSurfaceColorData::Yuv (composite.rs): CompositeSurfaceFormat::Yuv, planes in
  // sColor0..2 (BatchTextures::composite_yuv); `texture` is plane 0
  bool yuv = false;
  wrcu_tex planes[2] = {0, 0};  // planes 1 and 2
  // CompositeTile::z_id: tiles are culled and drawn in ascending z_id, i.e. front to back (composite.rs:1021
  // sorts them so); equal ids keep the order they were added in
  int32_t z_id = 0;
  DeviceBox2D valid_rect, dirty_rect;  // local_valid_rect / local_dirty_rect mapped to device space
  DeviceBox2D device_box() const { return DeviceBox2D{instance.v[0], instance.v[1], instance.v[2], instance.v[3]}; }
  DeviceBox2D clip_rect() const { return DeviceBox2D{instance.v[4], instance.v[5], instance.v[6], instance.v[7]}; }
};
struct CompositeState {
  std::vector<CompositeTile> tiles;
  bool has_clear_color = true;
  float clear_color[4] = {0, 0, 0, 0};
  bool dirty_rects_are_valid = true;  // false: the tiles' dirty rects say nothing; present everything
  // Tiles given in draw order (wrh_frame_add_composite_tile): drawn unsplit as listed, no occlusion
  // culling.  Splitting a tile that is scaled, filtered or placed off the pixel grid changes where its
  // rows start sampling, and so its bytes, against a frame that draws the tiles whole.
  bool listed = false;
};

// PartialPresentMode::Single (mod.rs:440-452): only `dirty_rect` of the framebuffer is redrawn
struct PartialPresentMode { DeviceBox2D dirty_rect; };

// The Draw compositor's partial-present settings (CompositorConfig::Draw, composite.rs)
struct PartialPresentConfig {
  int max_partial_present_rects = 0;                  // 0 = no partial present: every frame is redrawn whole
  bool draw_previous_partial_present_regions = false; // the host keeps no copy: redraw what older frames changed
};

// BufferDamageTracker (mod.rs:720-762): the dirty rects of the last four frames, so that a back buffer
// `buffer_age` frames old can be brought up to date
struct BufferDamageTracker {
  DeviceBox2D damage_rects[4];
  size_t current_offset = 0;
  void push_dirty_rect(const DeviceBox2D& rect);
  // empty = the buffer is up to date; nullopt = every pixel of it is stale
  std::optional<DeviceBox2D> get_damage_rect(size_t buffer_age) const;
};

struct Frame {  // frame_builder.rs:1129 (members the path reads)
  wrcu_frame_tables tables = {};
  std::vector<RenderPass> passes;
  CompositeState composite_state;
  wrcu_tex framebuffer = 0;  // DrawTarget::Default stand-in
  int32_t fb_width = 0, fb_height = 0;
  bool present = false;      // run composite_simple
};

// ---- update path: what the backend thread hands the renderer before a frame (mod.rs:1441-1560) ----
struct GpuCacheAddress { uint16_t u, v; };                                          // gpu_cache.rs:88-92
struct GpuCacheUpdate { uint32_t block_index, block_count; GpuCacheAddress address; };  // GpuCacheUpdate::Copy, gpu_cache.rs:299-305
struct GpuBlockData { float data[4]; };
struct GpuCacheUpdateList {  // gpu_cache.rs:327-345
  uint64_t frame_id = 0;
  bool clear = false;
  int32_t height = 0;
  std::vector<GpuCacheUpdate> updates;
  std::vector<GpuBlockData> blocks;
};
struct TextureCacheUpdate {  // texture_cache.rs TextureCacheUpdate with TextureUpdateSource::Bytes
  DeviceIntRect rect;
  const uint8_t* data = nullptr;  // first row of the rect
  size_t stride = 0;              // bytes between rows
  uint32_t bytes_per_pixel = 4;   // from the cache texture's ImageFormat
};
struct TextureCacheCopy { DeviceIntRect src_rect, dst_rect; };  // texture_cache.rs TextureCacheCopy
struct TextureUpdateList {  // texture_cache.rs:  per-texture updates + (src, dst) copies
  std::map<wrcu_tex, std::vector<TextureCacheUpdate>> updates;
  std::map<std::pair<wrcu_tex, wrcu_tex>, std::vector<TextureCacheCopy>> copies;
};

enum class RendererError { None, Shader, Thread, MaxTextureSize, SoftwareRasterizer, OutOfMemory };  // mod.rs:5700-5720

struct RendererStats {  // mod.rs RendererStats
  size_t total_draw_calls = 0, alpha_target_count = 0, color_target_count = 0;
};
struct RenderResults {  // mod.rs RenderResults (members the path fills)
  RendererStats stats;
  std::vector<DeviceIntRect> dirty_rects;  // what changed on screen this frame; none = nothing to present
};

class Renderer {
 public:
  explicit Renderer(wrcu_ctx* device) : device(device) {}
  // Renderer::render → render_impl → draw_frame (mod.rs:1241, 1441, 4525)
  RendererError render(const Frame& frame, RendererStats* stats);
  // The same with the back buffer's age (frames since it was last the back buffer; 0 = new) for
  // partial present: results->dirty_rects receives the frame's dirty rects.
  RendererError render(const Frame& frame, size_t buffer_age, RenderResults* results);

  void draw_frame(const Frame& frame, size_t buffer_age, RenderResults& results);
  void draw_picture_cache_target(const PictureCacheTarget& target, RendererStats& stats);         // mod.rs:2669
  void draw_color_target(const ColorRenderTarget& target, RendererStats& stats);                  // mod.rs:3486
  void draw_alpha_target(const AlphaRenderTarget& target, RendererStats& stats);                  // mod.rs:3754
  void draw_texture_cache_target(const TextureCacheRenderTarget& target, RendererStats& stats);   // mod.rs:3931
  void draw_alpha_batch_container(const AlphaBatchContainer& c, bool has_depth, RendererStats& stats);  // mod.rs:2804
  void draw_clip_batch_list(const ClipBatchList& list, int blend, RendererStats& stats);          // mod.rs:3695
  void draw_blurs(const BlurMap& blurs, bool color_target, RendererStats& stats);                 // mod.rs:3675
  void handle_scaling(const ScalingMap& scalings, RendererStats& stats);                          // mod.rs:2472
  void composite_simple(const Frame& frame, const std::optional<PartialPresentMode>& partial_present_mode,
                        RendererStats& stats);                                                    // mod.rs:3340
  // mod.rs:3126; each item is drawn with its tile's instance, clipped to the item's rectangle
  void draw_tile_list(const std::vector<CompositeTile>& tiles, const std::vector<occlusion::Item>& items, int blend,
                      RendererStats& stats);
  std::optional<PartialPresentMode> calculate_dirty_rects(size_t buffer_age, const CompositeState& cs, int fb_width,
                                                          int fb_height, RenderResults& results);  // mod.rs:4311
  PartialPresentConfig partial_present;
  BufferDamageTracker buffer_damage_tracker;
  bool force_redraw = true;  // the next frame is presented whole (init.rs:782)
  // draw_instanced_batch<T> (mod.rs:2022-2065)
  void draw_instanced_batch(int kind, uint32_t features, const void* instances, size_t stride, size_t n,
                            const BatchTextures& textures, RendererStats& stats);
  // update path (SURVEY.md §8f rank 3): lists queued by update_document, applied at the top of render_impl
  void update_gpu_cache();      // mod.rs:1498-1535 → GpuCacheTexture::update / flush (renderer/gpu_cache.rs:218-380)
  void update_texture_cache();  // mod.rs:1795-1990 → upload_to_texture_cache (renderer/upload.rs)
  std::vector<GpuCacheUpdateList> pending_gpu_cache_updates;
  std::vector<TextureUpdateList> pending_texture_updates;
  bool pending_gpu_cache_clear = false;
  RendererError check_gl_errors();  // mod.rs:1992
  std::vector<std::string> renderer_errors;

 private:
  void bind_draw_target(wrcu_tex color, wrcu_tex depth, int w, int h);
  wrcu_ctx* device;
  wrcu_draw_state state = {};
  int failed = 0;
};

int blend_key(BlendMode mode, MixBlendMode advanced);  // set_blend_mode_* → SWGL blend key
int batch_kind_to_wrcu(BatchKind kind);                // Shaders::get (shade.rs:1206-1305)

}  // namespace wr
