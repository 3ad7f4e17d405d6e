"""ctypes binding of libwrhost.so — the C++ mirror of the reference's `Renderer`
(webrender_b200/host/wr_renderer.h) — plus a converter from this package's flat
`Frame` (frame.py) to the reference-shaped `wr::Frame` (passes → picture-cache /
colour / alpha targets → batch containers, composite state).

The converter classifies ops the way the frame builder would have placed them:
  * R8 target                               → AlphaRenderTarget (clip batcher; blend NONE = primary, MULTIPLY = secondary)
  * RGBA8 target, quad prims + ps_quad_mask → ColorRenderTarget (prim_batches / mask_batches)
  * RGBA8 target, brush / text batches      → PictureCacheTarget (opaque batches = blend NONE + depth write,
                                              stored in batch order: the renderer draws them reversed)
  * RGBA8 target with only composite ops    → composite_simple (CompositeState tiles)

A composite state can also be handed over directly (build_composite): tiles with their z order, valid and
dirty rects, drawn with occlusion culling and, once set_partial_present enables it, partial present.
"""
import ctypes as C
import os

import numpy as np

from . import abi
from .device import WrcuError
from .frame import Batch, Clear, Frame

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libwrhost.so")

# wr::BatchKind / wr::BlendMode enumerators (wr_renderer.h)
BATCH_KIND = {abi.KIND_QUAD_TEXTURED: 0, abi.KIND_QUAD_MASK: 1, abi.KIND_BRUSH_SOLID: 2, abi.KIND_BRUSH_IMAGE: 3,
              abi.KIND_BRUSH_BLEND: 4, abi.KIND_BRUSH_MIX_BLEND: 5, abi.KIND_BRUSH_LINEAR_GRADIENT: 6,
              abi.KIND_BRUSH_OPACITY: 7, abi.KIND_TEXT_RUN: 8, abi.KIND_QUAD_RADIAL_GRADIENT: 9,
              abi.KIND_QUAD_CONIC_GRADIENT: 10, abi.KIND_BRUSH_YUV_IMAGE: 11, abi.KIND_SPLIT_COMPOSITE: 12}
CACHE_TASK_KINDS = {abi.KIND_BORDER_SOLID, abi.KIND_BORDER_SEGMENT, abi.KIND_LINE_DECORATION,
                    abi.KIND_FAST_LINEAR_GRADIENT, abi.KIND_LINEAR_GRADIENT, abi.KIND_RADIAL_GRADIENT,
                    abi.KIND_CONIC_GRADIENT}
BM_NONE, BM_ALPHA, BM_PREMULT, BM_DEST_OUT, BM_SUBPX_DUAL, BM_ADVANCED, BM_MULT_DUAL, BM_SCREEN, BM_EXCL, BM_PLUS = range(10)


def _blend_mode(key):
    """wrcu blend key → (wr::BlendMode, wr::MixBlendMode)."""
    if key == abi.BLEND_NONE:
        return BM_NONE, 0
    if key == abi.BLEND_ALPHA:
        return BM_ALPHA, 0
    if key == abi.BLEND_PREMULTIPLIED_ALPHA:
        return BM_PREMULT, 0
    if key == abi.BLEND_PREMULTIPLIED_DEST_OUT:
        return BM_DEST_OUT, 0
    if key == abi.BLEND_PLUS_LIGHTER:
        return BM_PLUS, 0
    if abi.BLEND_ADV_MULTIPLY <= key <= abi.BLEND_ADV_LUMINOSITY:
        return BM_ADVANCED, 1 + key - abi.BLEND_ADV_MULTIPLY
    raise ValueError(f"blend key {key} has no BlendMode equivalent")


TILE_OPAQUE, TILE_CLEAR, TILE_ALPHA = 0, 1, 2   # wr::CompositeTileKind


class CompositeTile:
    """One tile of a composite state (composite.rs CompositeTile).

    kind: TILE_OPAQUE / TILE_CLEAR / TILE_ALPHA.  textures: one RGBA texture handle, or three YUV plane
    handles (then `instance` is a composite_yuv_instance).  instance: the 120-byte CompositeInstance;
    its rect is the device tile box, its clip rect the tile's device clip rect.  z_id: tiles are drawn in
    ascending z_id, i.e. front to back.  valid_rect / dirty_rect: (x0, y0, x1, y1) in device pixels,
    None = the instance's rect clipped to its clip rect."""

    def __init__(self, kind, textures, instance, z_id, valid_rect=None, dirty_rect=None, fast_path=False):
        self.kind, self.instance, self.z_id = kind, instance, z_id
        self.textures = tuple(textures) if isinstance(textures, (tuple, list)) else (textures,)
        self.valid_rect, self.dirty_rect, self.fast_path = valid_rect, dirty_rect, fast_path


class NativeFrame:
    """A wr::Frame built by HostRenderer.build (owns the arrays its pointers refer to)."""

    def __init__(self, hr, ptr, handles, keep):
        self.hr, self.ptr, self.handles, self.keep = hr, ptr, handles, keep

    def destroy(self):
        if self.ptr:
            self.hr.lib.wrh_frame_destroy(self.ptr)
            self.ptr = None


def occlusion_build(lib, rects, opaque):
    """wrh_occlusion_build through `lib` (libwrhost.so; needs no device).  See HostRenderer.occlusion_build."""
    rects = np.ascontiguousarray(np.asarray(rects, dtype=np.float32).reshape(-1, 4))
    op = np.ascontiguousarray(np.asarray(opaque, dtype=np.int32))
    n = len(rects)
    vis = np.zeros(max(1, 2 * n), np.int32)
    n_opaque = C.c_int(0)
    vp = C.c_void_p
    lib.wrh_occlusion_build.argtypes = [vp, vp, C.c_int, vp, vp, vp, C.c_int, C.POINTER(C.c_int)]
    total = 0
    for cap in (0, None):   # count the items, then fetch them
        cap = total if cap is None else cap
        keys, items = np.zeros(max(1, cap), np.int32), np.zeros((max(1, cap), 4), np.float32)
        total = lib.wrh_occlusion_build(rects.ctypes.data, op.ctypes.data, n, vis.ctypes.data, keys.ctypes.data,
                                        items.ctypes.data, cap, C.byref(n_opaque))
    out = [(int(keys[i]), tuple(float(v) for v in items[i])) for i in range(total)]
    return out[:n_opaque.value], out[n_opaque.value:], vis[:n].astype(bool), vis[n:].astype(bool)


class HostRenderer:
    """wr::Renderer over a CudaDevice's context."""

    def __init__(self, dev, lib_path=LIB_PATH):
        if not os.path.exists(lib_path):
            raise WrcuError(abi.ERR_NO_DEVICE, f"{lib_path} not built — run __graft_entry__.build()")
        self.dev = dev
        self._pending_keep = []
        L = self.lib = C.CDLL(lib_path)
        vp, i32, u32, sz = C.c_void_p, C.c_int32, C.c_uint32, C.c_size_t
        L.wrh_renderer_create.restype = vp
        L.wrh_renderer_create.argtypes = [vp]
        L.wrh_renderer_destroy.argtypes = [vp]
        L.wrh_frame_create.restype = vp
        L.wrh_frame_create.argtypes = [C.POINTER(abi.FrameTables)]
        L.wrh_frame_destroy.argtypes = [vp]
        L.wrh_frame_add_pass.argtypes = [vp]
        L.wrh_pass_add_picture_cache_target.argtypes = [vp, i32, u32, u32, i32, i32, C.POINTER(C.c_float), C.POINTER(i32)]
        L.wrh_pass_add_color_target.argtypes = [vp, i32, u32, u32, i32, i32]
        L.wrh_pass_add_alpha_target.argtypes = [vp, i32, u32, i32, i32]
        L.wrh_renderer_queue_gpu_cache_updates.argtypes = [vp, i32, i32, vp, i32, vp, i32]
        L.wrh_renderer_queue_texture_update.argtypes = [vp, u32, C.POINTER(i32), vp, sz, i32]
        L.wrh_renderer_queue_texture_copy.argtypes = [vp, u32, u32, C.POINTER(i32), C.POINTER(i32)]
        L.wrh_pass_add_texture_cache_target.argtypes = [vp, i32, u32, i32, i32]
        L.wrh_texture_cache_target_add_clear.argtypes = [vp, i32, i32, C.POINTER(i32)]
        L.wrh_texture_cache_target_add_tasks.argtypes = [vp, i32, i32, i32, vp, i32]
        batch_args = [vp, i32, i32, i32, i32, i32, i32, u32, C.POINTER(u32), vp, sz, i32]
        L.wrh_picture_target_add_batch.argtypes = batch_args
        L.wrh_color_target_add_batch.argtypes = batch_args
        L.wrh_alpha_target_add_clear.argtypes = [vp, i32, i32, i32, C.POINTER(i32)]
        L.wrh_alpha_target_add_clips.argtypes = [vp, i32, i32, i32, i32, u32, vp, sz, i32]
        L.wrh_target_add_blur_or_scale.argtypes = [vp, i32, i32, i32, i32, u32, vp, i32]
        L.wrh_frame_set_framebuffer.argtypes = [vp, u32, i32, i32, C.POINTER(C.c_float)]
        L.wrh_frame_add_composite_tile.argtypes = [vp, i32, u32, i32, C.POINTER(C.c_float)]
        L.wrh_frame_add_composite_yuv_tile.argtypes = [vp, i32, C.POINTER(u32), C.POINTER(C.c_float)]
        L.wrh_renderer_render.argtypes = [vp, vp, C.POINTER(C.c_uint64)]
        f4 = C.POINTER(C.c_float)
        L.wrh_composite_state_add_tile.argtypes = [vp, i32, C.POINTER(u32), i32, i32, f4, i32, f4, f4]
        L.wrh_composite_state_set_dirty_rects_are_valid.argtypes = [vp, i32]
        L.wrh_renderer_set_partial_present.argtypes = [vp, i32, i32]
        L.wrh_renderer_render_with_age.argtypes = [vp, vp, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(i32), i32,
                                                   C.POINTER(C.c_int)]
        L.wrh_renderer_last_error.restype = C.c_char_p
        L.wrh_renderer_last_error.argtypes = [vp]
        self.r = L.wrh_renderer_create(dev.ctx)

    def close(self):
        if self.r:
            self.lib.wrh_renderer_destroy(self.r)
            self.r = None

    # -- update path: queued like the backend thread's update lists, applied by the next render() ----
    def queue_gpu_cache_updates(self, height, clear, updates, blocks):
        blocks = np.ascontiguousarray(blocks, dtype=np.float32).reshape(-1, 4)
        arr = (abi.GpuCacheCopy * max(1, len(updates)))(*[abi.GpuCacheCopy(*[int(v) for v in u]) for u in updates])
        self.lib.wrh_renderer_queue_gpu_cache_updates(self.r, height, 1 if clear else 0, arr, len(updates),
                                                      blocks.ctypes.data if len(blocks) else None, len(blocks))

    def queue_texture_update(self, tex, rect, rows, bpp):
        """rect = (x0, y0, x1, y1); rows: 2-D uint8 array (h, >= w * bpp), kept alive until render()."""
        rows = np.ascontiguousarray(rows)
        self._pending_keep.append(rows)
        self.lib.wrh_renderer_queue_texture_update(self.r, tex, (C.c_int32 * 4)(*rect), rows.ctypes.data,
                                                   rows.strides[0], bpp)

    def queue_texture_copy(self, src, dst, src_rect, dst_rect):
        self.lib.wrh_renderer_queue_texture_copy(self.r, src, dst, (C.c_int32 * 4)(*src_rect), (C.c_int32 * 4)(*dst_rect))

    def build(self, frame: Frame, handles=None):
        """Build the native wr::Frame for `frame` (the frame builder's job upstream).  Returns a
        NativeFrame to pass to render_native() any number of times; free it with destroy()."""
        dev, L = self.dev, self.lib
        handles = {} if handles is None else handles
        for name, t in frame.textures.items():
            if name not in handles:
                handles[name] = dev.texture_create(t.fmt, t.width, t.height)
                dev.texture_set_filter(handles[name], t.filter)
                if t.data is not None:
                    dev.texture_upload(handles[name], 0, 0, t.width, t.height, t.data)
        tabs = abi.FrameTables()
        keep = []
        for name in ("prim_headers_f", "prim_headers_i", "transforms", "render_tasks", "gpu_cache", "gpu_buffer_f",
                     "gpu_buffer_i"):
            if frame.tables[name] is None:   # persistent GPU cache
                continue
            arr = np.ascontiguousarray(frame.tables[name])
            keep.append(arr)
            setattr(tabs, name, arr.ctypes.data if arr.size else None)
            setattr(tabs, name + "_texels", arr.size // 4)
        f = L.wrh_frame_create(C.byref(tabs))
        try:
            for rpass in frame.passes:
                p = L.wrh_frame_add_pass(f)
                for tgt in rpass:
                    self._add_target(f, p, frame, tgt, handles, keep)
        except Exception:
            L.wrh_frame_destroy(f)
            raise
        return NativeFrame(self, f, handles, keep)

    def render_native(self, nf):
        """Renderer::render on a built frame: C++ only from here down to the kernels."""
        calls = C.c_uint64(0)
        err = self.lib.wrh_renderer_render(self.r, nf.ptr, C.byref(calls))
        self._pending_keep = []
        if err != 0:
            raise WrcuError(err, "RendererError: " + self.lib.wrh_renderer_last_error(self.r).decode())
        return calls.value

    # -- composite state handed over directly ---------------------------------------------------------
    def build_composite(self, fb, width, height, clear_color, tiles, dirty_rects_are_valid=True):
        """A wr::Frame that only composites `tiles` (CompositeTile list) into the framebuffer texture `fb`
        (clear_color None = no clear).  Render it with render_native or render_with_age."""
        L = self.lib
        f = L.wrh_frame_create(C.byref(abi.FrameTables()))
        L.wrh_frame_set_framebuffer(f, fb, width, height, (C.c_float * 4)(*clear_color) if clear_color else None)
        for t in tiles:
            yuv = len(t.textures) == 3
            planes = (C.c_uint32 * 3)(*(t.textures if yuv else (t.textures[0], 0, 0)))
            inst = np.ascontiguousarray(t.instance).view(np.float32)
            r4 = lambda r: (C.c_float * 4)(*r) if r is not None else None
            L.wrh_composite_state_add_tile(f, t.kind, planes, 1 if yuv else 0, 1 if t.fast_path else 0,
                                           (C.c_float * 30)(*inst), int(t.z_id), r4(t.valid_rect), r4(t.dirty_rect))
        L.wrh_composite_state_set_dirty_rects_are_valid(f, 1 if dirty_rects_are_valid else 0)
        return NativeFrame(self, f, {}, [])

    def set_partial_present(self, max_partial_present_rects, draw_previous_partial_present_regions=False):
        """The Draw compositor's partial-present settings (0 rects = redraw every frame whole)."""
        self.lib.wrh_renderer_set_partial_present(self.r, max_partial_present_rects,
                                                  1 if draw_previous_partial_present_regions else 0)

    def render_with_age(self, nf, buffer_age):
        """Renderer::render of a built frame into a back buffer `buffer_age` frames old (0 = new).
        Returns (draw_calls, dirty_rects) with the rects as (x0, y0, x1, y1)."""
        calls, n = C.c_uint64(0), C.c_int(0)
        out = (C.c_int32 * 64)()
        err = self.lib.wrh_renderer_render_with_age(self.r, nf.ptr, buffer_age, C.byref(calls), out, 16, C.byref(n))
        self._pending_keep = []
        if err != 0:
            raise WrcuError(err, "RendererError: " + self.lib.wrh_renderer_last_error(self.r).decode())
        return calls.value, [tuple(out[4 * i:4 * i + 4]) for i in range(min(n.value, 16))]

    def render(self, frame: Frame, handles=None):
        """Build the wr::Frame for `frame`, render it, return (handles, draw_calls)."""
        nf = self.build(frame, handles)
        try:
            calls = self.render_native(nf)
        finally:
            nf.destroy()
        return nf.handles, calls

    def occlusion_build(self, rects, opaque):
        """The compositor's occlusion builder on `rects` (x0, y0, x1, y1 floats, front to back).  Returns
        (opaque_items, alpha_items, tested, added): items as (key, rect) in the builder's order, `tested`
        and `added` the per-rect results of test() just before add() and of add()."""
        return occlusion_build(self.lib, rects, opaque)

    def _add_blur_scale(self, f, p, target_kind, t, b, handles, ptr, n):
        if b.kind == abi.KIND_SCALE:
            which = 2
        else:
            direction = int(np.ascontiguousarray(b.instance_bytes()[0]).view(np.int32)[2])
            which = 0 if direction == 1 else 1   # DIR_VERTICAL = 1 → vertical_blurs
        self.lib.wrh_target_add_blur_or_scale(f, p, target_kind, t, which, handles[b.color[0]], ptr, n)

    def _add_target(self, f, p, frame, tgt, handles, keep):
        L = self.lib
        desc = frame.textures[tgt.texture]
        tex = handles[tgt.texture]
        depth = handles.get(tgt.depth, 0) if tgt.depth else 0
        batches = [op for op in tgt.ops if isinstance(op, Batch)]
        clears = [op for op in tgt.ops if isinstance(op, Clear)]
        kinds = {b.kind for b in batches}

        def tex4(b):
            arr = (C.c_uint32 * 4)(*[handles.get(n, 0) if n else 0 for n in b.color],
                                   handles.get(b.clip_mask, 0) if b.clip_mask else 0)
            return arr

        def inst(b):
            a = b.instance_bytes()
            keep.append(a)
            return a.ctypes.data, a.shape[1], a.shape[0]

        if kinds and kinds <= CACHE_TASK_KINDS:
            # texture-cache target (draw_texture_cache_target, mod.rs:3931)
            t = L.wrh_pass_add_texture_cache_target(f, p, tex, desc.width, desc.height)
            for c in clears:
                r = c.rect if c.rect else (0, 0, desc.width, desc.height)
                L.wrh_texture_cache_target_add_clear(f, p, t, (C.c_int32 * 4)(r[0], r[1], r[0] + r[2], r[1] + r[3]))
            for b in batches:
                ptr, stride, n = inst(b)
                if L.wrh_texture_cache_target_add_tasks(f, p, t, b.kind, ptr, n) != 0:
                    raise ValueError("texture-cache target: unexpected task kind")
            return
        if desc.fmt == abi.FMT_R8:
            t = L.wrh_pass_add_alpha_target(f, p, tex, desc.width, desc.height)
            for c in clears:
                rect = (C.c_int32 * 4)(*(c.rect if c.rect else (0, 0, desc.width, desc.height)))
                if c.rect:
                    rect = (C.c_int32 * 4)(c.rect[0], c.rect[1], c.rect[0] + c.rect[2], c.rect[1] + c.rect[3])
                L.wrh_alpha_target_add_clear(f, p, t, 1 if c.color[0] >= 0.5 else 0, rect)
            for b in batches:
                which = 0 if b.blend == abi.BLEND_NONE else 1
                ptr, stride, n = inst(b)
                if b.kind in (abi.KIND_BLUR, abi.KIND_SCALE):
                    self._add_blur_scale(f, p, 0, t, b, handles, ptr, n)
                    continue
                if b.kind == abi.KIND_CLIP_RECTANGLE:
                    L.wrh_alpha_target_add_clips(f, p, t, which, 1 if b.features & abi.FEAT_FAST_PATH else 0, 0, ptr, stride, n)
                elif b.kind == abi.KIND_CLIP_BOX_SHADOW:
                    L.wrh_alpha_target_add_clips(f, p, t, which, 2, handles[b.color[0]], ptr, stride, n)
                else:
                    raise ValueError("alpha target: unexpected batch kind")
            return
        if kinds and kinds <= {abi.KIND_COMPOSITE}:
            cc = clears[0].color if clears else None
            L.wrh_frame_set_framebuffer(f, tex, desc.width, desc.height, (C.c_float * 4)(*cc) if cc else None)
            # listed in the flat frame's draw order: composite_simple draws them so, unsplit
            opaque = [b for b in batches if b.blend == abi.BLEND_NONE]
            rest = [b for b in batches if b.blend != abi.BLEND_NONE]
            for b in opaque + rest:
                kind = 0 if b.blend == abi.BLEND_NONE else (1 if b.blend == abi.BLEND_PREMULTIPLIED_DEST_OUT else 2)
                for row in b.instance_bytes():
                    v = np.ascontiguousarray(row).view(np.float32)
                    if b.features & abi.FEAT_YUV:
                        planes = (C.c_uint32 * 3)(*[handles[nm] if nm else 0 for nm in b.color])
                        L.wrh_frame_add_composite_yuv_tile(f, kind, planes, (C.c_float * 30)(*v))
                        continue
                    L.wrh_frame_add_composite_tile(f, kind, handles[b.color[0]], 1 if b.features & abi.FEAT_FAST_PATH else 0,
                                                   (C.c_float * 30)(*v))
            return
        if kinds & {abi.KIND_QUAD_MASK, abi.KIND_BLUR, abi.KIND_SCALE} or (
                kinds == {abi.KIND_QUAD_TEXTURED} and all(b.blend == abi.BLEND_NONE for b in batches)):
            t = L.wrh_pass_add_color_target(f, p, tex, depth, desc.width, desc.height)
            for b in batches:
                ptr, stride, n = inst(b)
                if b.kind in (abi.KIND_BLUR, abi.KIND_SCALE):
                    self._add_blur_scale(f, p, 1, t, b, handles, ptr, n)
                    continue
                lst = 1 if b.kind == abi.KIND_QUAD_MASK else (0 if b.blend == abi.BLEND_NONE else 2)
                bm, adv = _blend_mode(b.blend if lst == 2 else abi.BLEND_NONE)
                L.wrh_color_target_add_batch(f, p, t, lst, BATCH_KIND[b.kind], bm, adv, b.features, tex4(b), ptr, stride, n)
            return
        # picture-cache target
        cc = clears[0].color if clears and clears[0].color is not None else None
        t = L.wrh_pass_add_picture_cache_target(f, p, tex, depth, desc.width, desc.height,
                                                (C.c_float * 4)(*cc) if cc else None, None)
        opaque = [b for b in batches if b.blend == abi.BLEND_NONE]
        for b in opaque[::-1]:   # flat order is draw order (front to back); the container holds batch order
            ptr, stride, n = inst(b)
            a = np.ascontiguousarray(b.instance_bytes()[::-1])
            keep.append(a)
            L.wrh_picture_target_add_batch(f, p, t, 0, BATCH_KIND[b.kind], BM_NONE, 0, b.features, tex4(b), a.ctypes.data, stride, n)
        for b in batches:
            if b.blend == abi.BLEND_NONE:
                continue
            ptr, stride, n = inst(b)
            bm, adv = _blend_mode(b.blend)
            L.wrh_picture_target_add_batch(f, p, t, 1, BATCH_KIND[b.kind], bm, adv, b.features & ~abi.FEAT_ALPHA_PASS,
                                           tex4(b), ptr, stride, n)
