"""ctypes binding of libwrcu.so (include/wrcu.h): the product device.

Fails loudly when the CUDA library or a CUDA device is missing — there is no
CPU path in this package.
"""
import ctypes as C
import os

import numpy as np

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libwrcu.so")


class WrcuError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"wrcu error {code}: {msg}")
        self.code = code


def load_library(path=LIB_PATH):
    if not os.path.exists(path):
        raise WrcuError(abi.ERR_NO_DEVICE,
                        f"{path} not built — run `python -c 'import __graft_entry__ as g; g.build()'`")
    lib = C.CDLL(path)
    lib.wrcu_last_error_string.restype = C.c_char_p
    lib.wrcu_get_string.restype = C.c_char_p
    return lib


def bind_prefixed(lib, prefix):
    """Give `lib`'s `<prefix>_*` device entry points the shared argtypes."""
    def f(name):
        return getattr(lib, prefix + name)
    vp, i32, u32, sz = C.c_void_p, C.c_int32, C.c_uint32, C.c_size_t
    f("texture_create").argtypes = [vp, i32, i32, i32, C.POINTER(u32)]
    f("texture_set_filter").argtypes = [vp, u32, i32]
    f("texture_upload").argtypes = [vp, u32, i32, i32, i32, i32, vp, sz]
    f("texture_destroy").argtypes = [vp, u32]
    f("read_pixels").argtypes = [vp, u32, i32, i32, i32, i32, vp, sz]
    f("frame_begin").argtypes = [vp, C.POINTER(abi.FrameTables)]
    f("frame_end").argtypes = [vp]
    f("target_bind").argtypes = [vp, u32, u32, C.POINTER(C.c_float), C.POINTER(i32)]
    f("clear").argtypes = [vp, C.POINTER(i32), C.POINTER(C.c_float), C.POINTER(C.c_float)]
    f("draw_batch").argtypes = [vp, i32, u32, C.POINTER(abi.DrawState), vp, sz, i32]
    f("draw_composite_tiles").argtypes = [vp, u32, C.POINTER(abi.DrawState), vp, sz, i32, C.POINTER(C.c_uint32)]
    f("last_error_string").argtypes = [vp]
    f("last_error_string").restype = C.c_char_p
    f("texture_upload_batch").argtypes = [vp, u32, C.POINTER(abi.UploadRect), sz, vp, sz]
    f("texture_copy").argtypes = [vp, u32, u32, C.POINTER(i32), i32, i32]
    f("gpu_cache_update").argtypes = [vp, i32, i32, C.POINTER(abi.GpuCacheCopy), sz, vp, sz]


class DeviceBase:
    """Shared marshalling for any library exporting the wrcu device calls under
    a prefix (`wrcu_` for the CUDA backend)."""
    prefix = "wrcu_"

    def _f(self, name):
        return getattr(self.lib, self.prefix + name)

    def _check(self, rc):
        if rc != 0:
            raise WrcuError(rc, self._f("last_error_string")(self.ctx).decode())

    def texture_create(self, fmt, w, h):
        out = C.c_uint32(0)
        self._check(self._f("texture_create")(self.ctx, fmt, w, h, C.byref(out)))
        return out.value

    def texture_set_filter(self, tex, filt):
        self._check(self._f("texture_set_filter")(self.ctx, tex, filt))

    def texture_upload(self, tex, x, y, w, h, data):
        data = np.ascontiguousarray(data)
        rows = data.view(np.uint8).reshape(h, -1)
        self._check(self._f("texture_upload")(self.ctx, tex, x, y, w, h, rows.ctypes.data, rows.strides[0]))

    def texture_destroy(self, tex):
        self._check(self._f("texture_destroy")(self.ctx, tex))

    # -- update path (SURVEY.md §8f rank 3) ------------------------------------------
    def texture_upload_batch(self, tex, rects, staging):
        """rects: [(x, y, w, h, offset, stride)]; staging: one contiguous uint8 blob."""
        staging = np.ascontiguousarray(staging).view(np.uint8).reshape(-1)
        arr = rects if isinstance(rects, C.Array) else self.upload_rects(rects)
        self._check(self._f("texture_upload_batch")(self.ctx, tex, arr, len(arr), staging.ctypes.data, staging.size))

    @staticmethod
    def upload_rects(rects):
        """The #[repr(C)] rect array for texture_upload_batch (build once, reuse across frames)."""
        return (abi.UploadRect * len(rects))(*[abi.UploadRect(*[int(v) for v in r]) for r in rects])

    @staticmethod
    def gpu_cache_copies(updates):
        return (abi.GpuCacheCopy * max(1, len(updates)))(*[abi.GpuCacheCopy(*[int(v) for v in u]) for u in updates])

    def texture_copy(self, src, dst, src_rect, dst_x, dst_y):
        self._check(self._f("texture_copy")(self.ctx, src, dst, (C.c_int32 * 4)(*src_rect), dst_x, dst_y))

    def gpu_cache_update(self, height, clear, updates, blocks):
        """updates: [(block_index, block_count, u, v)] (GpuCacheUpdate::Copy); blocks: (n, 4) float32."""
        blocks = np.ascontiguousarray(blocks, dtype=np.float32).reshape(-1, 4)
        n = len(updates)
        arr = updates if isinstance(updates, C.Array) else self.gpu_cache_copies(updates)
        self._check(self._f("gpu_cache_update")(self.ctx, height, 1 if clear else 0, arr, n,
                                                blocks.ctypes.data if len(blocks) else None, len(blocks)))

    def read_pixels(self, tex, x, y, w, h, bpp):
        out = np.empty((h, w * bpp), dtype=np.uint8)
        self._check(self._f("read_pixels")(self.ctx, tex, x, y, w, h, out.ctypes.data, out.strides[0]))
        return out

    def frame_begin(self, tables):
        t = abi.FrameTables()
        self._keep = []
        for name in ("prim_headers_f", "prim_headers_i", "transforms", "render_tasks", "gpu_cache",
                     "gpu_buffer_f", "gpu_buffer_i"):
            if tables[name] is None:   # gpu_cache: bind the persistent cache (wrcu_gpu_cache_update)
                setattr(t, name, None)
                setattr(t, name + "_texels", 0)
                continue
            arr = np.ascontiguousarray(tables[name])
            self._keep.append(arr)
            setattr(t, name, arr.ctypes.data if arr.size else None)
            setattr(t, name + "_texels", arr.size // 4)
        self._check(self._f("frame_begin")(self.ctx, C.byref(t)))

    def frame_end(self):
        self._check(self._f("frame_end")(self.ctx))

    def target_bind(self, color, depth, projection, viewport):
        proj = (C.c_float * 16)(*[float(v) for v in projection])
        vp = (C.c_int32 * 4)(*viewport)
        self._check(self._f("target_bind")(self.ctx, color, depth, proj, vp))

    def clear(self, rect, color, depth):
        r = (C.c_int32 * 4)(*rect) if rect is not None else None
        col = (C.c_float * 4)(*color) if color is not None else None
        d = C.byref(C.c_float(depth)) if depth is not None else None
        self._check(self._f("clear")(self.ctx, r, col, C.cast(d, C.POINTER(C.c_float)) if d is not None else None))

    def clear_rects(self, rects, color):
        """wrcu_clear_rects: clear each (x, y, w, h) of `rects` to `color` (one launch per 64 rects)."""
        rects = np.ascontiguousarray(np.asarray(rects, dtype=np.int32).reshape(-1, 4))
        f = self._f("clear_rects")
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(C.c_float)]
        self._check(f(self.ctx, rects.ctypes.data if len(rects) else None, len(rects),
                      (C.c_float * 4)(*color)))

    def draw_batch(self, kind, features, blend, depth, colors, clip_mask, scissor, blend_color, inst):
        st = abi.DrawState()
        st.blend, st.depth = blend, depth
        for i in range(3):
            st.color[i] = colors[i]
        st.clip_mask = clip_mask
        st.scissor_enabled = 1 if scissor is not None else 0
        if scissor is not None:
            for i in range(4):
                st.scissor[i] = scissor[i]
        for i in range(4):
            st.blend_color[i] = blend_color[i]
        inst = np.ascontiguousarray(inst)
        n, stride = inst.shape
        self._check(self._f("draw_batch")(self.ctx, kind, features, C.byref(st), inst.ctypes.data, stride, n))

    def draw_composite_tiles(self, features, blend, scissor, blend_color, inst, textures):
        """wrcu_draw_composite_tiles: one CompositeInstance list, one texture per instance."""
        st = abi.DrawState()
        st.blend, st.depth = blend, abi.DEPTH_OFF
        st.scissor_enabled = 1 if scissor is not None else 0
        if scissor is not None:
            for i in range(4):
                st.scissor[i] = scissor[i]
        for i in range(4):
            st.blend_color[i] = blend_color[i]
        inst = np.ascontiguousarray(inst)
        n, stride = inst.shape
        tex = (C.c_uint32 * n)(*textures)
        self._check(self._f("draw_composite_tiles")(self.ctx, features, C.byref(st), inst.ctypes.data, stride, n, tex))


class CudaDevice(DeviceBase):
    """wrcu context on one GPU (one per process / GPU)."""
    prefix = "wrcu_"

    def __init__(self, device_ordinal=0, lib_path=LIB_PATH):
        self.lib = load_library(lib_path)
        bind_prefixed(self.lib, "wrcu_")
        self.lib.wrcu_ctx_create.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
        self.lib.wrcu_ctx_destroy.argtypes = [C.c_void_p]
        self.lib.wrcu_finish.argtypes = [C.c_void_p]
        self.lib.wrcu_get_stats.argtypes = [C.c_void_p, C.POINTER(abi.Stats)]
        self.lib.wrcu_reset_stats.argtypes = [C.c_void_p]
        self.lib.wrcu_timer_begin.argtypes = [C.c_void_p]
        self.lib.wrcu_timer_end.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
        self.lib.wrcu_texture_device_ptr.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_void_p),
                                                     C.POINTER(C.c_size_t)]
        self.lib.wrcu_stream.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
        self.lib.wrcu_host_alloc.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p)]
        self.lib.wrcu_host_free.argtypes = [C.c_void_p, C.c_void_p]
        self.lib.wrcu_read_pixels_async.argtypes = [C.c_void_p, C.c_uint32, C.c_int32, C.c_int32, C.c_int32,
                                                    C.c_int32, C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64)]
        self.lib.wrcu_fence_wait.argtypes = [C.c_void_p, C.c_uint64]
        self.lib.wrcu_profile_enable.argtypes = [C.c_void_p, C.c_int]
        self.lib.wrcu_last_raster_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
        self.lib.wrcu_texture_export.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(abi.IpcTexture)]
        self.lib.wrcu_texture_import.argtypes = [C.c_void_p, C.POINTER(abi.IpcTexture), C.POINTER(C.c_uint32)]
        self.lib.wrcu_peer_flags_create.argtypes = [C.c_void_p, C.c_int, C.POINTER(abi.IpcFlags)]
        self.lib.wrcu_peer_flags_open.argtypes = [C.c_void_p, C.POINTER(abi.IpcFlags), C.POINTER(C.c_int)]
        self.lib.wrcu_peer_signal.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_uint32]
        self.lib.wrcu_peer_wait.argtypes = [C.c_void_p, C.c_int, C.c_uint32]
        self.lib.wrcu_fence_insert.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
        ctx = C.c_void_p()
        rc = self.lib.wrcu_ctx_create(device_ordinal, C.byref(ctx))
        if rc != 0:
            raise WrcuError(rc, "wrcu_ctx_create failed: no usable CUDA device (this backend has no CPU path)")
        self.ctx = ctx

    def close(self):
        if getattr(self, "ctx", None):
            for p in getattr(self, "_pinned", []):
                self.lib.wrcu_host_free(self.ctx, p)
            self._pinned = []
            self.lib.wrcu_ctx_destroy(self.ctx)
            self.ctx = None

    def finish(self):
        self._check(self.lib.wrcu_finish(self.ctx))

    def stats(self):
        s = abi.Stats()
        self.lib.wrcu_get_stats(self.ctx, C.byref(s))
        return {k: getattr(s, k) for k, _ in abi.Stats._fields_}

    def reset_stats(self):
        self.lib.wrcu_reset_stats(self.ctx)

    def timer_begin(self):
        self._check(self.lib.wrcu_timer_begin(self.ctx))

    def timer_end(self):
        ms = C.c_float(0)
        self._check(self.lib.wrcu_timer_end(self.ctx, C.byref(ms)))
        return ms.value

    def profile_enable(self, on=True):
        self._check(self.lib.wrcu_profile_enable(self.ctx, 1 if on else 0))

    def last_raster_ms(self):
        ms = C.c_float(0)
        self._check(self.lib.wrcu_last_raster_ms(self.ctx, C.byref(ms)))
        return ms.value

    def texture_device_ptr(self, tex):
        p, pitch = C.c_void_p(), C.c_size_t()
        self._check(self.lib.wrcu_texture_device_ptr(self.ctx, tex, C.byref(p), C.byref(pitch)))
        return p.value, pitch.value

    def host_alloc(self, shape, dtype=np.uint8):
        """Page-locked host array (the PBO analogue) owned by the context."""
        nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
        p = C.c_void_p()
        self._check(self.lib.wrcu_host_alloc(self.ctx, nbytes, C.byref(p)))
        buf = (C.c_uint8 * nbytes).from_address(p.value)
        arr = np.frombuffer(buf, dtype=dtype).reshape(shape)
        self._pinned = getattr(self, "_pinned", [])
        self._pinned.append(p.value)
        return arr

    def read_pixels_async(self, tex, x, y, w, h, out):
        """Queue a readback into a (pinned) host array; returns a fence."""
        f = C.c_uint64(0)
        self._check(self.lib.wrcu_read_pixels_async(self.ctx, tex, x, y, w, h, out.ctypes.data, out.strides[0],
                                                    C.byref(f)))
        return f.value

    # -- multi-GPU (SURVEY.md §8e): shared framebuffer + stream-ordered flags -----------------------
    def texture_export(self, tex):
        """bytes of a wrcu_ipc_texture other contexts / processes can import"""
        h = abi.IpcTexture()
        self._check(self.lib.wrcu_texture_export(self.ctx, tex, C.byref(h)))
        return bytes(h)

    def texture_import(self, blob):
        h = abi.IpcTexture.from_buffer_copy(blob)
        out = C.c_uint32(0)
        self._check(self.lib.wrcu_texture_import(self.ctx, C.byref(h), C.byref(out)))
        return out.value

    def peer_flags_create(self, count):
        h = abi.IpcFlags()
        self._check(self.lib.wrcu_peer_flags_create(self.ctx, count, C.byref(h)))
        return bytes(h)

    def peer_flags_open(self, blob):
        h = abi.IpcFlags.from_buffer_copy(blob)
        out = C.c_int(0)
        self._check(self.lib.wrcu_peer_flags_open(self.ctx, C.byref(h), C.byref(out)))
        return out.value

    def peer_signal(self, peer_id, slot, value):
        self._check(self.lib.wrcu_peer_signal(self.ctx, peer_id, slot, value & 0xFFFFFFFF))

    def peer_wait(self, slot, value):
        self._check(self.lib.wrcu_peer_wait(self.ctx, slot, value & 0xFFFFFFFF))

    def fence_insert(self):
        """glFenceSync on the draw stream; page-locked upload buffers are free again once it is waited on."""
        f = C.c_uint64(0)
        self._check(self.lib.wrcu_fence_insert(self.ctx, C.byref(f)))
        return f.value

    def fence_wait(self, fence):
        self._check(self.lib.wrcu_fence_wait(self.ctx, fence))

    def stream(self):
        s = C.c_void_p()
        self.lib.wrcu_stream(self.ctx, C.byref(s))
        return s.value
