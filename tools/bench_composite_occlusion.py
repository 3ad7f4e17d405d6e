"""Time composite_simple with occlusion culling and the narrowed clear against the painter's order.

One 3840x2160 framebuffer holds 20 opaque picture-cache tiles, a full-width opaque header over them, a
1920x1080 opaque NV12 video surface, and two alpha tiles, one of them partly behind the header.  Each case
is timed device-side (CUDA events, the 50 MB L2 flushed before every step, as bench.py does):

  occlusion      wr::Renderer::render of the composite state: opaque pieces, alpha pieces back to front,
                 and a clear of only what no opaque piece covers
  painter        the same tiles through wrcu directly: a full clear, then every tile unsplit, back to front
  dirty_rect     the occlusion case under partial present, with one 256x256 tile region changed
  dirty_painter  the painter's order clipped to that dirty rect (a rect clear, then every tile unsplit)

It prints one JSON line per case: median ms, kernel launches per frame, and the bytes the frame writes
(clears plus tile pixels; the video surface's plane reads and alpha reads are not counted).

  python tools/bench_composite_occlusion.py [--steps 50] [--warmup 5] [--out FILE]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

W, H = 3840, 2160
DIRTY = (1792.0, 256.0, 2048.0, 512.0)   # one 256x256 region of tile 2


def build_scene():
    """(textures, tiles): tiles as (kind, texture names, instance, z_id), lower z_id in front."""
    from webrender_b200 import abi
    from webrender_b200.frame import TextureDesc
    from webrender_b200.gpu_types import composite_instance, composite_yuv_instance, YUV_FORMAT_NV12
    from webrender_b200.host import TILE_ALPHA, TILE_OPAQUE
    from workloads import scenes
    textures = {"fb": TextureDesc(abi.FMT_RGBA8, W, H)}
    tiles = []
    tw, th = 768, 540                       # 5 x 4 picture-cache tiles cover the framebuffer
    for i in range(20):
        name = "tile%d" % i
        textures[name] = TextureDesc(abi.FMT_RGBA8, tw, th, data=scenes.tile_texture(tw, th, 10 + i), filter=abi.NEAREST)
        x0, y0 = float(tw * (i % 5)), float(th * (i // 5))
        tiles.append((TILE_OPAQUE, (name,), composite_instance((x0, y0, x0 + tw, y0 + th), (0.0, 0.0, W, H)), 100 + i))
    textures["header"] = TextureDesc(abi.FMT_RGBA8, W, 160, data=scenes.tile_texture(W, 160, 3), filter=abi.NEAREST)
    tiles.append((TILE_OPAQUE, ("header",), composite_instance((0.0, 0.0, W, 160.0), (0.0, 0.0, W, H)), 10))
    vy, vuv = scenes.yuv_planes(1920, 1080, 7, "nv12")
    textures["vy"] = TextureDesc(abi.FMT_R8, 1920, 1080, data=vy, filter=abi.LINEAR)
    textures["vuv"] = TextureDesc(abi.FMT_RG8, 960, 540, data=vuv, filter=abi.LINEAR)
    r = (960.0, 540.0, 2880.0, 1620.0)
    ry, rc = (0.0, 0.0, 1920.0, 1080.0), (0.0, 0.0, 960.0, 540.0)
    tiles.append((TILE_OPAQUE, ("vy", "vuv", ""), composite_yuv_instance(r, r, 2, YUV_FORMAT_NV12, 8, (ry, rc, rc)), 20))
    for k, (rect, z) in enumerate((((3000.0, 1700.0, 3600.0, 2100.0), 0), ((200.0, 60.0, 1000.0, 460.0), 50))):
        name = "alpha%d" % k
        w, h = int(rect[2] - rect[0]), int(rect[3] - rect[1])
        textures[name] = TextureDesc(abi.FMT_RGBA8, w, h, data=scenes.tile_texture(w, h, 40 + k, False), filter=abi.NEAREST)
        tiles.append((TILE_ALPHA, (name,), composite_instance(rect, (0.0, 0.0, W, H)), z))
    return textures, tiles


def painter_frame(textures, tiles, clip=None):
    """A full clear (or a clear of `clip`), then every tile unsplit, back to front, clipped to `clip`."""
    from webrender_b200 import abi
    from webrender_b200.frame import Batch, Clear, Frame, Target
    from webrender_b200.host import TILE_OPAQUE
    from workloads import scenes
    ops = [Clear(color=(0.0, 0.0, 0.0, 1.0),
                 rect=None if clip is None else tuple(int(v) for v in (clip[0], clip[1], clip[2] - clip[0], clip[3] - clip[1])))]
    for kind, names, inst, z in sorted(tiles, key=lambda t: -t[3]):
        inst = inst.copy()
        if clip is not None:
            v = inst.view(np.float32)
            v[4:8] = (max(v[4], clip[0]), max(v[5], clip[1]), min(v[6], clip[2]), min(v[7], clip[3]))
        yuv = names[0] == "vy"
        ops.append(Batch(abi.KIND_COMPOSITE, inst[None, :], blend=abi.BLEND_NONE if kind == TILE_OPAQUE else abi.BLEND_PREMULTIPLIED_ALPHA,
                         features=abi.FEAT_TEXTURE_2D | (abi.FEAT_YUV if yuv else abi.FEAT_FAST_PATH),
                         color=names if yuv else (names[0], "", "")))
    return Frame(scenes.FrameTables().arrays(), textures, [[Target("fb", ops=ops)]])


def _area(r, clip):
    x0, y0, x1, y1 = max(r[0], clip[0]), max(r[1], clip[1]), min(r[2], clip[2]), min(r[3], clip[3])
    return max(0.0, x1 - x0) * max(0.0, y1 - y0)


def bytes_written(tiles, host, clip=(0.0, 0.0, W, H)):
    """Clear plus tile pixels, 4 bytes each, of one frame of the given path."""
    import ctypes as C
    from webrender_b200.host import TILE_OPAQUE, occlusion_build
    rects = []
    for kind, names, inst, z in sorted(tiles, key=lambda t: t[3]):
        v = inst.view(np.float32)
        rects.append((max(v[0], v[4], clip[0]), max(v[1], v[5], clip[1]), min(v[2], v[6], clip[2]), min(v[3], v[7], clip[3])))
    front_to_back = sorted(tiles, key=lambda t: t[3])
    if not host:
        return 4 * int(_area(clip, clip) + sum(_area(r, clip) for r in rects))
    lib = C.CDLL(os.path.join(ROOT, "webrender_b200", "libwrhost.so"))
    op_items, al_items, _, _ = occlusion_build(lib, rects, [t[0] == TILE_OPAQUE for t in front_to_back])
    covered = np.zeros((H, W), bool)
    for _, r in op_items:
        covered[int(r[1]):int(r[3]), int(r[0]):int(r[2])] = True
    region = np.zeros((H, W), bool)
    region[int(clip[1]):int(clip[3]), int(clip[0]):int(clip[2])] = True
    clear = int((region & ~covered).sum())
    return 4 * int(clear + sum(_area(r, clip) for _, r in op_items + al_items))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", help="also write the JSON lines here")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_composite_occlusion: no CUDA device; the wrcu backend has no CPU path")
    from bench import l2_flush
    from webrender_b200.device import CudaDevice
    from webrender_b200.frame import draw_frame
    from webrender_b200.host import CompositeTile, HostRenderer

    textures, tiles = build_scene()
    dev = CudaDevice(0)
    hr = HostRenderer(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    handles = draw_frame(dev, painter_frame(textures, tiles))   # creates and uploads every texture
    empty = (0.0, 0.0, 0.0, 0.0)

    def host_frame(dirty):
        ts = [CompositeTile(k, [handles[n] if n else 0 for n in names], inst, z,
                            dirty_rect=(DIRTY if dirty and names[0] == "tile2" else (empty if dirty else None)),
                            fast_path=names[0] != "vy")
              for k, names, inst, z in tiles]
        return hr.build_composite(handles["fb"], W, H, (0.0, 0.0, 0.0, 1.0), ts)

    full_nf, dirty_nf = host_frame(False), host_frame(True)
    painter, dirty_painter = painter_frame(textures, tiles), painter_frame(textures, tiles, DIRTY)

    def run_occlusion():
        hr.set_partial_present(0)
        hr.render_native(full_nf)

    def run_dirty():
        hr.set_partial_present(1)
        hr.render_with_age(dirty_nf, 1)

    cases = {
        "occlusion": (run_occlusion, bytes_written(tiles, True)),
        "painter": (lambda: draw_frame(dev, painter, handles, tile_lists=True), bytes_written(tiles, False)),
        "dirty_rect": (run_dirty, bytes_written(tiles, True, DIRTY)),
        "dirty_painter": (lambda: draw_frame(dev, dirty_painter, handles, tile_lists=True), bytes_written(tiles, False, DIRTY)),
    }
    # the first partial-present frame is always drawn whole: present one before timing the dirty case
    hr.set_partial_present(1)
    hr.render_with_age(full_nf, 0)
    gpu = torch.cuda.get_device_name(0)
    lines = []
    for name, (run, nbytes) in cases.items():
        for _ in range(args.warmup):
            run()
        dev.finish()
        dev.reset_stats()
        ms = []
        for _ in range(args.steps):
            l2_flush(flush)
            dev.timer_begin()
            run()
            ms.append(dev.timer_end())
        launches = dev.stats()["kernel_launches"] / args.steps
        ms.sort()
        lines.append({"case": name, "ms": ms[len(ms) // 2], "ms_min": ms[0], "launches": launches,
                      "bytes_written": nbytes, "steps": args.steps, "framebuffer": [W, H], "gpu": gpu})
    full_nf.destroy()
    dirty_nf.destroy()
    hr.close()
    dev.close()
    for line in lines:
        print(json.dumps(line))
    if args.out:
        with open(args.out, "w") as f:
            f.write("".join(json.dumps(line) + "\n" for line in lines))


if __name__ == "__main__":
    main()
