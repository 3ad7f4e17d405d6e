"""composite_simple as the reference runs it (renderer/mod.rs:3340-3484): tiles clipped to their valid, clip
and partial-present rects, culled front to back by the occlusion builder (rectangle_occlusion.rs), opaque
pieces drawn first, then clear tiles, then alpha pieces back to front, and the framebuffer cleared only where
no opaque piece covers it (wrcu_clear_rects).

CPU tier: the builder through its test hook (libwrhost.so needs no device).
GPU tier: the host renderer's framebuffer against the painter's order (full clear, every tile unsplit, back
to front) drawn by the oracle, and by SWGL where the reference rasteriser is built; wrcu_clear_rects against
wrcu_clear issued rect by rect; partial present over two frames; launch counts."""
import os

import numpy as np
import pytest

from oracle.backends import OracleDevice, SwglDevice, have_swgl
from webrender_b200 import abi
from webrender_b200.frame import Batch, Clear, Frame, Target, TextureDesc, draw_frame, ortho
from webrender_b200.gpu_types import composite_instance, composite_yuv_instance, YUV_FORMAT_NV12
from webrender_b200.host import TILE_ALPHA, TILE_CLEAR, TILE_OPAQUE, CompositeTile, occlusion_build
from workloads import scenes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST_LIB = os.path.join(ROOT, "webrender_b200", "libwrhost.so")


def _hostlib():
    import ctypes as C
    return C.CDLL(HOST_LIB)


# ---- CPU tier: the occlusion builder ---------------------------------------------------------------------
def _mask(rects, size, scale, origin=-8):
    """Per-cell coverage of `rects` on a grid of 1/scale pixel cells from `origin` (every edge lies on the
    grid, every rect inside it)."""
    m = np.zeros((size * scale, size * scale), bool)
    for r in rects:
        x0, y0, x1, y1 = (int(round((v - origin) * scale)) for v in r)
        assert 0 <= x0 and 0 <= y0 and x1 <= size * scale and y1 <= size * scale
        m[y0:y1, x0:x1] = True
    return m


def _overlap(a, b):
    return max(a[0], b[0]) < min(a[2], b[2]) and max(a[1], b[1]) < min(a[3], b[3])


@pytest.mark.parametrize("seed", range(8))
@pytest.mark.parametrize("step", [1.0, 0.5], ids=["integer", "half_pixel"])
def test_builder_random_rects(seed, step):
    rng = np.random.RandomState(seed * 7 + int(step * 2))
    size, n = 96, 14
    rects = []
    for _ in range(n):   # every edge on a multiple of `step`, some past the grid's left and top edges
        x0, y0 = rng.randint(-16, 96, 2) * 0.5
        w, h = rng.randint(2, 48, 2) * 0.5
        r = (x0, y0, x0 + w, y0 + h)
        rects.append(tuple(float(np.floor(v)) for v in r) if step == 1.0 else r)
    opaque = rng.rand(n) < 0.6
    op_items, al_items, tested, added = occlusion_build(_hostlib(), rects, opaque)
    assert np.array_equal(tested, added)
    scale = int(1 / step)
    by_key = {}
    for k, r in op_items + al_items:
        by_key.setdefault(k, []).append(r)
    for i, rect in enumerate(rects):
        frags = by_key.get(i, [])
        assert all(opaque[i] == ((i, f) in op_items) for f in frags)
        for f in frags:   # inside its rect, never empty
            assert rect[0] <= f[0] < f[2] <= rect[2] and rect[1] <= f[1] < f[3] <= rect[3], (i, f, rect)
        for a in range(len(frags)):
            for b in range(a):
                assert not _overlap(frags[a], frags[b]), (i, frags[a], frags[b])
        hidden = _mask([rects[j] for j in range(i) if opaque[j]], size, scale)
        want = _mask([rect], size, scale) & ~hidden
        assert np.array_equal(_mask(frags, size, scale), want), i
        assert added[i] == bool(want.any())
    for a in range(len(op_items)):
        for b in range(a):
            assert not _overlap(op_items[a][1], op_items[b][1])


def _composite_tiles(frame):
    """The framebuffer tiles HostRenderer.build hands over for a flat frame, back to front: (kind, rect)."""
    for rpass in frame.passes:
        for t in rpass:
            batches = [o for o in t.ops if isinstance(o, Batch)]
            if not batches or any(b.kind != abi.KIND_COMPOSITE for b in batches):
                continue
            out = []
            for b in [b for b in batches if b.blend == abi.BLEND_NONE] + [b for b in batches if b.blend != abi.BLEND_NONE]:
                kind = TILE_OPAQUE if b.blend == abi.BLEND_NONE else (
                    TILE_CLEAR if b.blend == abi.BLEND_PREMULTIPLIED_DEST_OUT else TILE_ALPHA)
                for row in b.instance_bytes():
                    v = np.ascontiguousarray(row).view(np.float32)
                    out.append((kind, (max(v[0], v[4]), max(v[1], v[5]), min(v[2], v[6]), min(v[3], v[7]))))
            return out
    raise AssertionError("no composite target")


# Every scene whose opaque tiles do not overlap one another.  yuv_composite_frame's opaque surfaces and
# composite_frame(fractional=True)'s jittered grid do overlap: the builder splits the tiles behind, and
# test_host_renderer.py checks that the bytes are still those of the flat frame.
SCENES = {
    "composite": lambda: scenes.composite_frame(seed=1),
    "composite_external": lambda: scenes.composite_frame(seed=2, external=True),
    "composite_4k": lambda: scenes.composite_frame(3840, 2160, 1024, 512, seed=4),
    "page": lambda: scenes.page_frame(width=2048, height=1024, seed=2),
    "page_4k": lambda: scenes.page_frame(3840, 2160, 1024, 512, seed=1),
    "yuv_alpha": lambda: scenes.yuv_composite_frame("nv12", 0, seed=2, opaque=False),
    "video": lambda: scenes.video_frame(3840, 2160, 1920, 1080, "nv12"),
    "box_shadow_through_tile": scenes.reftest_box_shadow_suite_composited_frame,
}


@pytest.mark.parametrize("name", list(SCENES))
def test_existing_scenes_pass_through_unchanged(name):
    tiles = [t for t in _composite_tiles(SCENES[name]()) if t[0] != TILE_CLEAR]
    front_to_back = tiles[::-1]
    rects = [r for _, r in front_to_back]
    op_items, al_items, _, added = occlusion_build(_hostlib(), rects, [k == TILE_OPAQUE for k, _ in front_to_back])
    assert added.all()
    got = sorted((k, tuple(np.float32(v) for v in r)) for k, r in op_items + al_items)
    want = sorted((i, tuple(np.float32(v) for v in r)) for i, r in enumerate(rects))
    assert got == want


# ---- GPU tier ----------------------------------------------------------------------------------------------
def _tex(desc, dev):
    h = dev.texture_create(desc.fmt, desc.width, desc.height)
    dev.texture_set_filter(h, desc.filter)
    if desc.data is not None:
        dev.texture_upload(h, 0, 0, desc.width, desc.height, desc.data)
    return h


class Scene:
    """Tiles of one framebuffer: textures by name, and per tile (kind, texture names, instance, z_id,
    valid_rect)."""

    def __init__(self, w, h, clear=(0.1, 0.2, 0.3, 1.0)):
        self.w, self.h, self.clear = w, h, clear
        self.textures = {"fb": TextureDesc(abi.FMT_RGBA8, w, h),
                         "dummy": TextureDesc(abi.FMT_RGBA8, 1, 1, data=np.full((1, 4), 255, np.uint8),
                                              filter=abi.NEAREST)}
        self.tiles = []

    def add(self, kind, names, inst, z, valid=None, fast_path=False):
        self.tiles.append((kind, tuple(names), inst, z, valid, fast_path))

    def host_tiles(self, handles):
        return [CompositeTile(k, [handles[n] for n in names], inst, z, valid, fast_path=fp)
                for k, names, inst, z, valid, fp in self.tiles]

    def painter_frame(self):
        """Full clear, then every tile unsplit, back to front (clipped to its valid rect)."""
        ops = [Clear(color=self.clear)]
        back_to_front = [t for _, t in sorted(enumerate(self.tiles), key=lambda it: (-it[1][3], -it[0]))]
        for k, names, inst, z, valid, fp in back_to_front:
            inst = inst.copy()
            v = inst.view(np.float32)
            if valid is not None:
                v[4:8] = (max(v[4], valid[0]), max(v[5], valid[1]), min(v[6], valid[2]), min(v[7], valid[3]))
            blend = {TILE_OPAQUE: abi.BLEND_NONE, TILE_CLEAR: abi.BLEND_PREMULTIPLIED_DEST_OUT,
                     TILE_ALPHA: abi.BLEND_PREMULTIPLIED_ALPHA}[k]
            feats = abi.FEAT_TEXTURE_2D | (abi.FEAT_YUV if len(names) == 3 else 0) | (abi.FEAT_FAST_PATH if fp else 0)
            ops.append(Batch(abi.KIND_COMPOSITE, inst[None, :], blend=blend, features=feats,
                             color=names if len(names) == 3 else (names[0], "", "")))
        return Frame(scenes.FrameTables().arrays(), self.textures, [[Target("fb", ops=ops)]])


def _tile_tex(sc, name, w, h, seed, opaque=True):
    sc.textures[name] = TextureDesc(abi.FMT_RGBA8, w, h, data=scenes.tile_texture(w, h, seed, opaque), filter=abi.NEAREST)


def _random_scene(w, h, seed, fractional=False, with_yuv=False, n=14):
    """Overlapping opaque tiles, alpha tiles in front of and behind them, tiles off every edge, optionally
    a YUV surface in front of the page."""
    rng = np.random.RandomState(seed)
    sc = Scene(w, h)
    for i in range(n):
        tw, th = int(rng.randint(w // 8, w // 2)), int(rng.randint(h // 8, h // 2))
        opaque = rng.rand() < 0.6
        name = "t%d" % i
        _tile_tex(sc, name, tw, th, seed * 100 + i, opaque)
        x0, y0 = float(rng.randint(-tw // 3, w - 2 * tw // 3)), float(rng.randint(-th // 3, h - 2 * th // 3))
        if fractional:
            x0 += float(rng.choice([0.0, 0.25, 0.5, 0.75]))
            y0 += float(rng.choice([0.0, 0.5]))
        rect = (x0, y0, x0 + tw, y0 + th)
        clip = rect if i % 3 else (rect[0] + 3.0, rect[1] + 2.0, rect[2] - 5.0, rect[3] - 1.5 * fractional)
        sc.add(TILE_OPAQUE if opaque else TILE_ALPHA, (name,), composite_instance(rect, clip), int(rng.randint(0, 1000)),
               fast_path=True)
    if with_yuv:
        vw, vh = 192, 128
        planes = scenes.yuv_planes(vw, vh, seed + 5, "nv12")
        sc.textures["vy"] = TextureDesc(abi.FMT_R8, vw, vh, data=planes[0], filter=abi.LINEAR)
        sc.textures["vuv"] = TextureDesc(abi.FMT_RG8, vw // 2, vh // 2, data=planes[1], filter=abi.LINEAR)
        r = (w * 0.25, h * 0.25, w * 0.75, h * 0.75)
        ry = (0.0, 0.0, float(vw), float(vh))
        inst = composite_yuv_instance(r, r, 2, YUV_FORMAT_NV12, 8, (ry, tuple(v * 0.5 for v in ry), tuple(v * 0.5 for v in ry)))
        sc.add(TILE_OPAQUE, ("vy", "vuv", ""), inst, -1)   # in front of every page tile
        sc.add(TILE_ALPHA, ("t0",), composite_instance((w * 0.6, h * 0.1, w * 0.9, h * 0.5), (0, 0, w, h)), -2,
               fast_path=True)
    return sc


def _render_host(sc, dev, hr, clear=True, buffer_age=None, dirty_valid=True):
    handles = {n: _tex(d, dev) for n, d in sc.textures.items()}
    handles[""] = 0
    nf = hr.build_composite(handles["fb"], sc.w, sc.h, sc.clear if clear else None, sc.host_tiles(handles), dirty_valid)
    try:
        res = hr.render_native(nf) if buffer_age is None else hr.render_with_age(nf, buffer_age)
    finally:
        nf.destroy()
    return dev.read_pixels(handles["fb"], 0, 0, sc.w, sc.h, 4), res


def _reference(frame, w, h):
    """The painter's-order frame drawn by the oracle, and by SWGL when the reference rasteriser is built
    (the two must agree)."""
    outs = []
    for D in (OracleDevice, SwglDevice) if have_swgl() else (OracleDevice,):
        d = D()
        try:
            hd = draw_frame(d, frame)
            outs.append(d.read_pixels(hd["fb"], 0, 0, w, h, 4))
        finally:
            d.close()
    for o in outs[1:]:
        assert np.array_equal(o, outs[0]), "oracle and SWGL disagree"
    return outs[0]


def _reference_order_frame(sc):
    """The reference's order (mod.rs:3447-3483) as a flat frame built from the builder's items: a full
    clear, the opaque pieces, the clear tiles, the alpha pieces reversed, each piece its tile's instance
    clipped to the piece."""
    order = sorted(range(len(sc.tiles)), key=lambda i: sc.tiles[i][3])   # front to back, stable
    rects, opaque, keys, clears = [], [], [], []
    for i in order:
        k, names, inst, z, valid, fp = sc.tiles[i]
        v = inst.view(np.float32)
        r = (max(v[0], v[4]), max(v[1], v[5]), min(v[2], v[6]), min(v[3], v[7]))
        if valid is not None:
            r = (max(r[0], valid[0]), max(r[1], valid[1]), min(r[2], valid[2]), min(r[3], valid[3]))
        if not (r[2] > r[0] and r[3] > r[1]):
            continue
        if k == TILE_CLEAR:
            clears.append((i, r))
            continue
        rects.append(r)
        opaque.append(k == TILE_OPAQUE)
        keys.append(i)
    op_items, al_items, _, _ = occlusion_build(_hostlib(), rects, opaque)

    def batch(tile_idx, rect, blend):
        k, names, inst, z, valid, fp = sc.tiles[tile_idx]
        inst = inst.copy()
        inst.view(np.float32)[4:8] = rect
        yuv = len(names) == 3
        return Batch(abi.KIND_COMPOSITE, inst[None, :], blend=blend,
                     features=abi.FEAT_TEXTURE_2D | (abi.FEAT_YUV if yuv else 0) | (abi.FEAT_FAST_PATH if fp else 0),
                     color=names if yuv else (names[0], "", ""))
    ops = [Clear(color=sc.clear)]
    ops += [batch(keys[k], r, abi.BLEND_NONE) for k, r in op_items]
    ops += [batch(i, r, abi.BLEND_PREMULTIPLIED_DEST_OUT) for i, r in clears]
    ops += [batch(keys[k], r, abi.BLEND_PREMULTIPLIED_ALPHA) for k, r in al_items[::-1]]
    return Frame(scenes.FrameTables().arrays(), sc.textures, [[Target("fb", ops=ops)]])


@pytest.fixture
def cuda():
    from webrender_b200.device import CudaDevice
    from webrender_b200.host import HostRenderer
    dev = CudaDevice(0)
    hr = HostRenderer(dev)
    yield dev, hr
    hr.close()
    dev.close()


# Whole-pixel 1:1 tiles: a piece of a tile has the bytes of that part of the whole tile, so the reference's
# order gives the painter's bytes.
PAINTER_CASES = {
    "overlap_integer": lambda: _random_scene(320, 200, 1),
    "overlap_integer_2": lambda: _random_scene(257, 181, 2, n=20),
    "yuv_in_front": lambda: _random_scene(384, 256, 5, with_yuv=True),
    "1080p": lambda: _random_scene(1920, 1080, 6, n=24),
}
# Fractional edges and scaled video: a piece's rows start sampling where the piece starts, as the reference's
# do, so these are compared with the reference's order drawn from the builder's items.
REFERENCE_ORDER_CASES = {
    "fractional": lambda: _random_scene(320, 200, 3, fractional=True),
    "fractional_2": lambda: _random_scene(203, 151, 4, fractional=True, n=18),
    "yuv_behind": lambda: _yuv_behind_scene(),
    "1080p_fractional_yuv": lambda: _random_scene(1920, 1080, 7, fractional=True, with_yuv=True, n=24),
}


def _yuv_behind_scene():
    """A scaled video surface with opaque page tiles in front of parts of it: the surface is split."""
    sc = _random_scene(384, 256, 8, with_yuv=True, n=6)
    sc.tiles = [t if t[1][0] != "vy" else t[:3] + (2000,) + t[4:] for t in sc.tiles]
    return sc


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PAINTER_CASES))
def test_matches_painters_order(cuda, name):
    dev, hr = cuda
    sc = PAINTER_CASES[name]()
    got, _ = _render_host(sc, dev, hr)
    want = _reference(sc.painter_frame(), sc.w, sc.h)
    assert np.array_equal(got, want), f"{(got != want).sum()} bytes differ"


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(REFERENCE_ORDER_CASES))
def test_matches_reference_order(cuda, name):
    dev, hr = cuda
    sc = REFERENCE_ORDER_CASES[name]()
    got, _ = _render_host(sc, dev, hr)
    want = _reference(_reference_order_frame(sc), sc.w, sc.h)
    assert np.array_equal(got, want), f"{(got != want).sum()} bytes differ"


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [1, 2])
def test_clear_tiles_in_reference_order(cuda, seed):
    """Clear tiles punch through whatever lies under them: the reference's order (opaque items, clear tiles,
    alpha items reversed) built from the builder's items, against the host renderer."""
    dev, hr = cuda
    sc = _random_scene(320, 200, 10 + seed)
    rng = np.random.RandomState(seed)
    for i in range(2):
        r = scenes._rand_rect(rng, 320, 200, 30, 120)
        sc.add(TILE_CLEAR, ("dummy",), composite_instance(r, r, (0.0, 0.0, 0.0, 1.0)), int(rng.randint(0, 1000)))
    got, _ = _render_host(sc, dev, hr)
    want = _reference(_reference_order_frame(sc), sc.w, sc.h)
    assert np.array_equal(got, want), f"{(got != want).sum()} bytes differ"


def _launches(dev):
    return dev.stats()["kernel_launches"]


@pytest.mark.gpu
def test_launch_counts(cuda):
    dev, hr = cuda
    # opaque tiles covering the framebuffer: no clear launch at all
    covered = Scene(512, 256)
    for i in range(4):
        _tile_tex(covered, "c%d" % i, 128, 256, 50 + i)
        covered.add(TILE_OPAQUE, ("c%d" % i,), composite_instance((128.0 * i, 0, 128.0 * (i + 1), 256), (0, 0, 512, 256)),
                    i, fast_path=True)
    _render_host(covered, dev, hr)                      # warm
    dev.finish()
    n0 = _launches(dev)
    _render_host(covered, dev, hr, clear=True)
    n1 = _launches(dev)
    _render_host(covered, dev, hr, clear=False)
    n2 = _launches(dev)
    assert n1 - n0 == n2 - n1, "a fully covered framebuffer still got a clear launch"
    # a framebuffer with gaps: exactly one clear launch, however many rects the gaps need
    gaps = Scene(512, 256)
    for i in range(3):
        _tile_tex(gaps, "g%d" % i, 100, 100, 60 + i)
        gaps.add(TILE_OPAQUE, ("g%d" % i,), composite_instance((150.0 * i + 10, 40.0 * i + 5, 150.0 * i + 110, 40.0 * i + 105),
                                                              (0, 0, 512, 256)), i, fast_path=True)
    n0 = _launches(dev)
    got, _ = _render_host(gaps, dev, hr, clear=True)
    n1 = _launches(dev)
    _render_host(gaps, dev, hr, clear=False)
    n2 = _launches(dev)
    assert (n1 - n0) - (n2 - n1) == 1
    assert np.array_equal(got, _reference(gaps.painter_frame(), gaps.w, gaps.h))
    # overlapping opaque tiles are split into pieces of one copy-engine batch: the same launches as the
    # same tiles side by side
    over = Scene(512, 256)
    side = Scene(512, 256)
    for sc in (over, side):
        for i in range(3):
            _tile_tex(sc, "o%d" % i, 200, 200, 70 + i)
    for i in range(3):
        over.add(TILE_OPAQUE, ("o%d" % i,), composite_instance((96.0 * i, 16.0 * i, 96.0 * i + 200, 16.0 * i + 200),
                                                              (0, 0, 512, 256)), i, fast_path=True)
        side.add(TILE_OPAQUE, ("o%d" % i,), composite_instance((160.0 * i, 0, 160.0 * i + 150, 200), (0, 0, 512, 256)), i,
                 fast_path=True)
    n0 = _launches(dev)
    got, _ = _render_host(over, dev, hr, clear=False)
    n1 = _launches(dev)
    _render_host(side, dev, hr, clear=False)
    n2 = _launches(dev)
    assert n1 - n0 == n2 - n1
    got2, _ = _render_host(over, dev, hr)
    assert np.array_equal(got2, _reference(over.painter_frame(), over.w, over.h))


# ---- partial present -----------------------------------------------------------------------------------
def _pp_scene(changed):
    """A page of four opaque tiles and an alpha tile; `changed` swaps tile 1's content, and only its
    dirty rect is non-empty."""
    sc = Scene(320, 200)
    empty = (0.0, 0.0, 0.0, 0.0)
    for i in range(4):
        name = "p%d" % i + ("b" if changed and i == 1 else "")
        _tile_tex(sc, name, 160, 100, 80 + i + (100 if changed and i == 1 else 0))
        x0, y0 = 160.0 * (i % 2), 100.0 * (i // 2)
        sc.add(TILE_OPAQUE, (name,), composite_instance((x0, y0, x0 + 160, y0 + 100), (0, 0, 320, 200)), 10 + i,
               fast_path=True)
    _tile_tex(sc, "a", 80, 60, 90, False)
    sc.add(TILE_ALPHA, ("a",), composite_instance((200.0, 20, 280, 80), (0, 0, 320, 200)), 0, fast_path=True)
    dirty = {1: (180.0, 10.0, 250.0, 60.0)} if changed else {}
    return sc, [dirty.get(i, empty) for i in range(5)]


def _render_pp(dev, hr, handles, sc, dirty, age, dirty_valid=True):
    tiles = sc.host_tiles(handles)
    for t, d in zip(tiles, dirty):
        t.dirty_rect = d
    nf = hr.build_composite(handles["fb"], sc.w, sc.h, sc.clear, tiles, dirty_valid)
    try:
        return hr.render_with_age(nf, age)
    finally:
        nf.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("draw_previous", [False, True], ids=["no_previous", "draw_previous"])
@pytest.mark.parametrize("age", [0, 1, 2])
@pytest.mark.parametrize("dirty_valid", [True, False], ids=["dirty_valid", "dirty_invalid"])
def test_partial_present_two_frames(cuda, age, draw_previous, dirty_valid):
    dev, hr = cuda
    hr.set_partial_present(1, draw_previous)
    s1, d1 = _pp_scene(False)
    s2, d2 = _pp_scene(True)
    textures = dict(s1.textures)
    textures.update(s2.textures)
    handles = {n: _tex(d, dev) for n, d in textures.items()}
    # frame 1: the first frame is always presented whole
    _, rects1 = _render_pp(dev, hr, handles, s1, d1, 0)
    assert rects1 == [(0, 0, 320, 200)]
    f1 = dev.read_pixels(handles["fb"], 0, 0, 320, 200, 4)
    assert np.array_equal(f1, _reference(s1.painter_frame(), 320, 200))
    # frame 2 into a back buffer `age` frames old
    _, rects2 = _render_pp(dev, hr, handles, s2, d2, age, dirty_valid)
    f2 = dev.read_pixels(handles["fb"], 0, 0, 320, 200, 4)
    full2 = _reference(s2.painter_frame(), 320, 200)
    if not dirty_valid:
        # calculate_dirty_rects: no valid dirty rects, so one rect covering the framebuffer and a full redraw
        assert rects2 == [(0, 0, 320, 200)]
        assert np.array_equal(f2, full2)
        return
    assert rects2 == [(180, 10, 250, 60)]
    # the region redrawn: this frame's dirty rect, plus what changed since the buffer was last drawn when
    # the host keeps no copy (age 1: nothing; age 2: frame 1's whole-frame damage; age 0: everything)
    region = (180, 10, 250, 60) if (not draw_previous or age == 1) else (0, 0, 320, 200)
    want = f1.reshape(200, 320, 4).copy()
    x0, y0, x1, y1 = region
    want[y0:y1, x0:x1] = full2.reshape(200, 320, 4)[y0:y1, x0:x1]
    assert np.array_equal(f2.reshape(200, 320, 4), want)


@pytest.mark.gpu
def test_partial_present_occluded_dirty_rect_gets_no_clear(cuda):
    dev, hr = cuda
    hr.set_partial_present(1, False)
    s1, d1 = _pp_scene(False)
    s2, _ = _pp_scene(True)
    textures = dict(s1.textures)
    textures.update(s2.textures)
    handles = {n: _tex(d, dev) for n, d in textures.items()}
    _render_pp(dev, hr, handles, s1, d1, 0)
    d2 = [(0.0, 0.0, 0.0, 0.0)] * 5
    d2[1] = (170.0, 85.0, 190.0, 99.0)   # inside tile 1, away from the alpha tile
    f1 = dev.read_pixels(handles["fb"], 0, 0, 320, 200, 4)
    dev.finish()
    n0 = _launches(dev)
    _, rects = _render_pp(dev, hr, handles, s2, d2, 1)
    n1 = _launches(dev)
    assert rects == [(170, 85, 190, 99)]
    # the same frame without a clear colour launches the same kernels
    nf = hr.build_composite(handles["fb"], 320, 200, None, [
        CompositeTile(t.kind, t.textures, t.instance, t.z_id, dirty_rect=d) for t, d in zip(s2.host_tiles(handles), d2)])
    try:
        hr.render_with_age(nf, 1)
    finally:
        nf.destroy()
    n2 = _launches(dev)
    assert n1 - n0 == n2 - n1
    f2 = dev.read_pixels(handles["fb"], 0, 0, 320, 200, 4).reshape(200, 320, 4)
    want = f1.reshape(200, 320, 4).copy()
    want[85:99, 170:190] = _reference(s2.painter_frame(), 320, 200).reshape(200, 320, 4)[85:99, 170:190]
    assert np.array_equal(f2, want)


# ---- wrcu_clear_rects on its own ------------------------------------------------------------------------
def _rect_list(rng, w, h, n):
    out = []
    for i in range(n):
        k = i % 6
        if k == 0:     # anywhere, possibly past the edges
            x, y = int(rng.randint(-20, w)), int(rng.randint(-20, h))
            out.append((x, y, int(rng.randint(0, w // 2 + 30)), int(rng.randint(0, h // 2 + 30))))
        elif k == 1:   # on the right / bottom edge
            out.append((w - int(rng.randint(1, 9)), h - int(rng.randint(1, 9)), 16, 16))
        elif k == 2:   # out of range or empty
            out.append([(w + 5, 0, 10, 10), (0, -30, 10, 10), (3, 3, 0, 7), (3, 3, 7, -2)][int(rng.randint(0, 4))])
        else:          # narrow, unaligned x0, width not a multiple of 4
            out.append((int(rng.randint(0, w)), int(rng.randint(0, h)), int(rng.randint(1, 11)), int(rng.randint(1, 40))))
    return out


CLEAR_ENVS = {"default": {}, "streams1": {"WRCU_STREAMS": 1}, "immediate": {"WRCU_IMMEDIATE": 1}}


@pytest.mark.gpu
@pytest.mark.parametrize("env", list(CLEAR_ENVS))
@pytest.mark.parametrize("fmt", [abi.FMT_RGBA8, abi.FMT_R8], ids=["rgba8", "r8"])
@pytest.mark.parametrize("n", [0, 1, 64, 65, 1000])
def test_clear_rects_matches_clear(monkeypatch, env, fmt, n):
    for k, v in CLEAR_ENVS[env].items():
        monkeypatch.setenv(k, str(v))
    from webrender_b200.device import CudaDevice
    dev = CudaDevice(0)
    try:
        rng = np.random.RandomState(n * 3 + fmt)
        w, h = 157, 93
        bpp = 4 if fmt == abi.FMT_RGBA8 else 1
        init = rng.randint(0, 256, (h, w * bpp)).astype(np.uint8)
        rects = _rect_list(rng, w, h, n)
        color = (0.2, 0.55, 0.8, 0.6)
        out = []
        for use_list in (False, True):
            t = dev.texture_create(fmt, w, h)
            dev.texture_upload(t, 0, 0, w, h, init)
            dev.frame_begin(scenes.FrameTables().arrays())
            dev.target_bind(t, 0, ortho(w, h), (0, 0, w, h))
            if use_list:
                dev.clear_rects(rects, color)
            else:
                for r in rects:
                    dev.clear(r, color, None)
            dev.frame_end()
            out.append(dev.read_pixels(t, 0, 0, w, h, bpp))
        assert np.array_equal(out[0], out[1]), f"{(out[0] != out[1]).sum()} bytes differ"
        if n == 0:
            assert np.array_equal(out[1], init)
    finally:
        dev.close()


@pytest.mark.gpu
@pytest.mark.parametrize("env", list(CLEAR_ENVS))
def test_clear_rects_between_batches(monkeypatch, env):
    """A rect-list clear queued between two batches of one submission stays between them."""
    for k, v in CLEAR_ENVS[env].items():
        monkeypatch.setenv(k, str(v))
    from webrender_b200.device import CudaDevice
    frame = scenes.composite_frame(seed=3)
    target = frame.passes[0][0]
    batches = [o for o in target.ops if isinstance(o, Batch)]
    rects = _rect_list(np.random.RandomState(9), 640, 384, 70)
    color = (0.9, 0.1, 0.4, 1.0)
    outs = []
    for use_list in (False, True):
        dev = CudaDevice(0)
        try:
            handles = {}
            for name, d in frame.textures.items():
                handles[name] = _tex(d, dev)
            dev.frame_begin(frame.tables)
            dev.target_bind(handles["fb"], 0, ortho(640, 384), (0, 0, 640, 384))
            dev.clear(None, (0.0, 0.0, 0.0, 0.0), None)
            for i, b in enumerate(batches):
                if i == len(batches) // 2:
                    if use_list:
                        dev.clear_rects(rects, color)
                    else:
                        for r in rects:
                            dev.clear(r, color, None)
                dev.draw_batch(b.kind, b.features, b.blend, b.depth, [handles.get(n, 0) if n else 0 for n in b.color],
                               0, b.scissor, b.blend_color, b.instance_bytes())
            dev.frame_end()
            outs.append(dev.read_pixels(handles["fb"], 0, 0, 640, 384, 4))
        finally:
            dev.close()
    assert np.array_equal(outs[0], outs[1]), f"{(outs[0] != outs[1]).sum()} bytes differ"
