"""The launch choices the draw path makes on the host (csrc/wrcu_api.cu: draw_batch_impl, launch_raster,
flush_pending, flush_multi_stream), each pinned on both sides of its threshold and compared byte for byte with
the oracle (oracle/wr_oracle.c).  Most of these choices exist only in the GPU build: the host emulation compiles
them out and takes one path per kind, so its tier here checks the frames and the oracle, and a GPU-tier failure
points at the GPU-only path rather than at the scene.

Where a path adds a launch the test asserts it through `kernel_launches` deltas between the two sides; where it
does not, the default run is compared with a run whose WRCU_* switch forces the other side, and both with the
oracle.

Which side of each threshold the cases sit on (line numbers are csrc/wrcu_api.cu unless named):

 choice                          | threshold                                         | below / off            | at / above / on
 --------------------------------+---------------------------------------------------+------------------------+------------------------
 streaming solid kernel          | n <= flat_max (1816); flat_max 1, WRCU_FLAT_MAX   | WRCU_FLAT_MAX=0 (all n)| n=1 default; n<=32 with
   wr_raster_solid_flat          |   clamped to FLAT_MAX=32 (295-298, raster.cuh:1461)| n=2..32 default       |   WRCU_FLAT_MAX=32
   (returns for non-simple:      |   raster.cuh:1469)                                | test_flat_declines_non_simple: n=1 with AA
 fold (+1 launch)                | n >= fold_min = 8 (305, 1837)                     | n=2 in the flat cases  | n=16,31,32: the fold launch
                                 |                                                   |                        |   replaces the flat kernel
 strip mode (WrRowReuse,         | strip && n <= 16 && K.strip (1858), and seg > 1:  | n=17; WRCU_STRIP=0     | n=1, 16 at 1920x1080: seg
   raster.cuh:1139)              |   ceil(grid_x/seg)*grid_y >= 2*max_ctas (1860)     |                        |   stays > 1 for up to 180
                                 |                                                   |                        |   SMs at 3 CTAs/SM
 side_reduce max_ctas            | >= 4 targets (2041) and n <= 256 (1853)           | 1 target               | 4 targets (strip, scheduler)
 warp-per-instance set-up        | n <= 64 (1721; setup_common.cuh:189,              | n=65                   | n=64
                                 |   shader_composite.cuh:193)                       |                        |
 bitmask bins                    | n >= 512 (1709); the 96 MiB guard needs ~400 K    | n=511                  | n=512, 8192, 8193
                                 |   commands on a 1080p target: not tested          |                        |
 list passes                     | 8192 commands per pass (raster.cuh:892)           | n=8192 (one pass)      | n=8193 (two passes)
 depth-fail grid (+1 launch per  | n >= 48: a CTA per command; else row groups, a    | n_alpha=47             | n_alpha=48 (the opaque batch
   depth-tested batch)           |   side_reduce share on >= 4 targets (1784-1787)   |                        |   of 8 is always below)
 side streams                    | n_streams 8 (273); target index % NS (2039);      | T=1,2,3,4,8;           | T=9,17 (streams wrap);
                                 |   events from uses_conflict (1980)                 | WRCU_STREAMS=1         | WRCU_STREAMS=3
 hazards                         | RAW / WAR / WAW between ops on different streams  | test_hazards: raw, war, clip_mask
 submission split                | QMAX = 1024 queued ops (1398, 1763); BatchInfo    | every other frame      | split: ~1130 ops over 3
                                 |   and pool-counter ring halves (2102-2105)        |                        |   targets, folds both sides
 glyph-major text (+1 launch)    | n >= 8 (1865)                                     | n=7; WRCU_GLYPH_MAJOR=0| n=8; WRCU_GLYPH_CTAS 1, 16
 copy-engine composite (+1)      | copy_ok: blend NONE / PM, no depth (1674),        | n=129; an overlapping  | n=128 non-overlapping
                                 |   n <= WR_COPY_MAX_CMDS = 128 (1680), no overlap  |   pair                 |
                                 |   (1689-1693); target with a tensor map (543)     |                        |
 env switches                    | WRCU_PDL=0, WRCU_IMMEDIATE=1, WRCU_EARLY_CLEAR=0, WRCU_STREAMS, WRCU_SIDE_CTAS: scheduler and hazard cases
"""
import dataclasses

import numpy as np
import pytest

from oracle.backends import OracleDevice
from webrender_b200 import abi, draw_frame
from webrender_b200.device import CudaDevice
from webrender_b200.frame import Batch, Clear, Frame, Target, TextureDesc
from webrender_b200.gpu_types import (CLIP_TASK_EMPTY, FrameTables, INVALID_SEGMENT_INDEX, PART_ALL,
                                      QF_APPLY_DEVICE_CLIP, brush_instance, clip_rect_instance, composite_instance,
                                      quad_instance)
from workloads import scenes

from common import assert_same, render
from emu import EmuDevice

gpu = pytest.mark.gpu

FOLD_MIN = 8         # fold_min's default (wrcu_api.cu:305)
FLAT_MAX = 32        # FLAT_MAX (raster.cuh:1461)
COPY_MAX = 128       # WR_COPY_MAX_CMDS (shader_composite.cuh:15)
PM = abi.BLEND_PREMULTIPLIED_ALPHA
CLEAR = (0.4, 0.7, 0.2, 0.8)
AA_ALL = 0xF         # edge flags with PART_ALL: every edge anti-aliased (setup_quad.cuh:73), so not a simple batch

SWITCHES = ("WRCU_FLAT_MAX", "WRCU_FOLD_MIN", "WRCU_STRIP", "WRCU_STREAMS", "WRCU_EARLY_CLEAR", "WRCU_SIDE_CTAS",
            "WRCU_PDL", "WRCU_IMMEDIATE", "WRCU_GLYPH_MAJOR", "WRCU_GLYPH_CTAS", "WRCU_YUV_WIDE")


def render_with(monkeypatch, env, frame, names=None, tile_lists=False):
    """Draw `frame` on a CudaDevice created under the WRCU_* switches `env` (read in wrcu_ctx_create, so they are
    set before the device exists; every other switch is unset).  Returns ({name: bytes}, kernel launches)."""
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, str(v))
    d = CudaDevice()
    try:
        handles = draw_frame(d, frame, tile_lists=tile_lists)
        launches = d.stats()["kernel_launches"]
        out = {}
        for n in names or _targets(frame):
            desc = frame.textures[n]
            out[n] = d.read_pixels(handles[n], 0, 0, desc.width, desc.height, abi.FMT_BPP[desc.fmt])
        return out, launches
    finally:
        d.close()


def _targets(frame):
    return sorted({t.texture for p in frame.passes for t in p})


def oracle(frame, names=None):
    return render(OracleDevice, frame, names or _targets(frame))


# ---- frames ------------------------------------------------------------------------------------------------


def quads_frame(w, h, targets, blend=PM):
    """Solid quads (ps_quad_textured) over cleared RGBA8 targets of one pass.  targets = one list of batches per
    target; a batch is [(rect, colour, edge_flags), ...]."""
    t = FrameTables()
    task = t.add_render_task((0.0, 0.0, float(w), float(h)), 1.0, (0.0, 0.0))
    z = 0
    textures, tlist = {}, []
    for ti, batches in enumerate(targets):
        ops = [Clear(color=CLEAR)]
        for cmds in batches:
            inst = []
            for rect, color, edge in cmds:
                z += 1
                rect = tuple(float(v) for v in rect)
                prim_f = t.add_quad_prim(rect, rect, color)
                prim_i = t.add_quad_header(0, z)
                inst.append(quad_instance(prim_i, prim_f, QF_APPLY_DEVICE_CLIP, edge, PART_ALL, INVALID_SEGMENT_INDEX,
                                          task))
            ops.append(Batch(abi.KIND_QUAD_TEXTURED, np.stack(inst), blend=blend))
        textures[f"t{ti}"] = TextureDesc(abi.FMT_RGBA8, w, h)
        tlist.append(Target(f"t{ti}", ops=ops))
    return Frame(t.arrays(), textures, [tlist])


N_SHAPES = 8


def shape(w, h, k, rng):
    """Integer rect number k % 8: full cover, over every edge, ragged, zero width, zero height, off screen,
    negative origin, the bottom-right corner pixel hanging off the target."""
    k %= N_SHAPES
    r = lambda lo, hi: int(rng.randint(lo, max(lo + 1, hi)))  # noqa: E731
    if k == 0:
        return (0, 0, w, h)
    if k == 1:
        return (-r(1, 9), -r(1, 5), w + r(1, 9), h + r(1, 5))
    if k == 2:
        x0, y0 = r(-3, w), r(-2, h)
        return (x0, y0, x0 + r(1, w + 4), y0 + r(1, h + 3))
    if k == 3:
        x = r(0, w)
        return (x, 0, x, h)
    if k == 4:
        y = r(0, h)
        return (0, y, w, y)
    if k == 5:
        return (w + 3, -r(0, 4), w + 40, h) if rng.randint(2) else (-50, h + 1, w, h + 20)
    if k == 6:
        return (-r(1, 7), -r(1, 7), r(1, w + 1), r(1, h + 1))
    return (w - 1, h - 1, w + 2, h + 2)


def colour(k, rng):
    """k % 4: alpha 0 with non-zero colour lanes, opaque, over-range (colour above alpha), valid premultiplied."""
    k %= 4
    if k == 0:
        return tuple(float(v) for v in rng.uniform(0, 1, 3)) + (0.0,)
    if k == 1:
        return tuple(float(v) for v in rng.uniform(0, 1, 3)) + (1.0,)
    a = float(rng.uniform(0.05, 0.6))
    hi = 1.0 if k == 2 else a
    return tuple(float(v) for v in rng.uniform(0, hi, 3)) + (a,)


def flat_frame(w, h, n, seed, edge=0):
    """n = 1: one target per shape, each drawn by a one-command batch (every shape and colour reaches the
    one-command path).  n > 1: one target, one batch of n commands cycling through the shapes and colours."""
    rng = np.random.RandomState(seed)
    if n == 1:
        return quads_frame(w, h, [[[(shape(w, h, k, rng), colour(k + seed, rng), edge)]] for k in range(N_SHAPES)])
    return quads_frame(w, h, [[[(shape(w, h, i, rng), colour(i // 3, rng), edge) for i in range(n)]]])


def many_quads_frame(w, h, n, seed, blend=abi.BLEND_ALPHA):
    """One batch of n small random quads (8..96 px, some over the edges) with a full-target quad every 997th and
    last, so every tile has commands in every 8192-command pass.  BLEND_ALPHA keeps it off the solid kernels."""
    rng = np.random.RandomState(seed)
    cmds = []
    for i in range(n):
        if i % 997 == 500 or i == n - 1:
            rect = (0, 0, w, h)
        else:
            sw, sh = int(rng.randint(8, 97)), int(rng.randint(8, 97))
            x0, y0 = int(rng.randint(-sw // 2, w)), int(rng.randint(-sh // 2, h))
            rect = (x0, y0, x0 + sw, y0 + sh)
        c = tuple(float(v) for v in rng.uniform(0, 1, 3)) + (float(rng.uniform(0.1, 0.9)),)
        cmds.append((rect, c, 0))
    return quads_frame(w, h, [[cmds]], blend=blend)


def composite_list_frame(w, h, n, tile=(256, 16), tex=None, blend=abi.BLEND_NONE, overlap=False, seed=1):
    """A picture-cache tile list: n composite batches of one tile each into `fb`, in a grid of `tile`-sized rects.
    tex=None: tile-sized power-of-two textures drawn 1:1 (copy class, FAST_PATH, white); tex=(tw, th): scaled
    through the linear filter (never copy class).  overlap: the second tile is moved over the first by 8 px."""
    tw, th = tile
    cols = w // tw
    textures = {"fb": TextureDesc(abi.FMT_RGBA8, w, h)}
    sw, sh = tex or tile
    for j in range(4):
        textures[f"src{j}"] = TextureDesc(abi.FMT_RGBA8, sw, sh, data=scenes.tile_texture(sw, sh, seed * 10 + j,
                                                                                            blend == abi.BLEND_NONE),
                                          filter=abi.NEAREST if tex is None else abi.LINEAR)
    feats = abi.FEAT_TEXTURE_2D | (abi.FEAT_FAST_PATH if tex is None else 0)
    ops = [Clear(color=(0.1, 0.0, 0.2, 1.0))]
    for i in range(n):
        x, y = (i % cols) * tw, (i // cols) * th
        if overlap and i == 1:
            x -= 8
        rect = (float(x), float(y), float(x + tw), float(y + th))
        ops.append(Batch(abi.KIND_COMPOSITE, composite_instance(rect, rect)[None, :], blend=blend, features=feats,
                         color=(f"src{i % 4}", "", "")))
    return Frame(FrameTables().arrays(), textures, [[Target("fb", ops=ops)]])


def repeated_instances(frame, kind, n):
    """`frame` with the instances of its `kind` batch cycled to n."""
    out = []
    for p in frame.passes:
        tp = []
        for tgt in p:
            ops = []
            for op in tgt.ops:
                if isinstance(op, Batch) and op.kind == kind:
                    idx = np.arange(n) % op.instances.shape[0]
                    op = dataclasses.replace(op, instances=op.instances[idx])
                ops.append(op)
            tp.append(Target(tgt.texture, depth=tgt.depth, ops=ops))
        out.append(tp)
    return Frame(frame.tables, frame.textures, out)


def replicate(frame, count):
    """The one target of `frame` drawn `count` times, as the targets t0.. of one pass (each with a depth target
    d0.. of its own when the original has one)."""
    [[tgt]] = frame.passes
    textures = {k: v for k, v in frame.textures.items() if k not in (tgt.texture, tgt.depth)}
    targets = []
    for i in range(count):
        textures[f"t{i}"] = frame.textures[tgt.texture]
        if tgt.depth:
            textures[f"d{i}"] = frame.textures[tgt.depth]
        targets.append(Target(f"t{i}", depth=f"d{i}" if tgt.depth else "", ops=list(tgt.ops)))
    return Frame(frame.tables, textures, [targets])


def without_depth(frame):
    """`frame` with no depth target and every batch DEPTH_OFF (a depth clear then clears nothing)."""
    return Frame(frame.tables, frame.textures,
                 [[Target(t.texture, ops=[dataclasses.replace(op, depth=abi.DEPTH_OFF) if isinstance(op, Batch) else op
                                          for op in t.ops]) for t in p] for p in frame.passes])


def depth_launches(frame):
    """Launches that only a bound depth target adds: a depth clear per clear with a depth value, and a
    wr_depth_fail_rows prepass per depth-tested batch (brush_image: failing-sample bitmaps always, 1656)."""
    return sum(1 for p in frame.passes for t in p if t.depth for op in t.ops
               if (isinstance(op, Clear) and op.depth is not None) or (isinstance(op, Batch) and op.depth != abi.DEPTH_OFF))


def _quads(t, task, rng, w, h, n, z0):
    inst = []
    for i in range(n):
        x0, y0 = int(rng.randint(-20, w - 10)), int(rng.randint(-10, h - 10))
        rect = (float(x0), float(y0), float(x0 + rng.randint(10, w // 2)), float(y0 + rng.randint(10, h // 2)))
        a = float(rng.uniform(0.3, 1.0))
        c = tuple(float(v * a) for v in rng.uniform(0, 1, 3)) + (a,)
        inst.append(quad_instance(t.add_quad_header(0, z0 + i), t.add_quad_prim(rect, rect, c), QF_APPLY_DEVICE_CLIP, 0,
                                  PART_ALL, INVALID_SEGMENT_INDEX, task))
    return Batch(abi.KIND_QUAD_TEXTURED, np.stack(inst), blend=PM)


def sampled_target_frame(src=(1024, 512), dst=(1920, 1080), war=True, seed=1):
    """RAW: t0 is drawn, then a composite samples it, scaled through the linear filter, into fb.  war: afterwards,
    in the same submission, t0 is cleared to another colour and redrawn: fb must show the old t0, t0 the new."""
    rng = np.random.RandomState(seed)
    (sw, sh), (dw, dh) = src, dst
    t = FrameTables()
    task = t.add_render_task((0.0, 0.0, float(sw), float(sh)), 1.0, (0.0, 0.0))
    textures = {"t0": TextureDesc(abi.FMT_RGBA8, sw, sh, filter=abi.LINEAR), "fb": TextureDesc(abi.FMT_RGBA8, dw, dh)}
    full = (0.0, 0.0, float(dw), float(dh))
    passes = [[Target("t0", ops=[Clear(color=(0.9, 0.1, 0.1, 1.0)), _quads(t, task, rng, sw, sh, 12, 1)])],
              [Target("fb", ops=[Clear(color=(0.0, 0.0, 0.0, 1.0)),
                                 Batch(abi.KIND_COMPOSITE, composite_instance(full, full)[None, :], blend=abi.BLEND_NONE,
                                       features=abi.FEAT_TEXTURE_2D, color=("t0", "", ""))])]]
    if war:
        passes.append([Target("t0", ops=[Clear(color=(0.1, 0.2, 0.9, 1.0)), _quads(t, task, rng, sw, sh, 12, 100)])])
    return Frame(t.arrays(), textures, passes)


def clip_mask_hazard_frame(w=512, h=256, seed=1):
    """An R8 clip mask (cs_clip_rectangle) is drawn, consumed by masked brush_solid quads on `a`, then cleared and
    redrawn with other clips and consumed again on `b`, all in one submission."""
    rng = np.random.RandomState(seed)
    t = FrameTables()
    pic = t.add_render_task((0.0, 0.0, float(w), float(h)), 1.0, (0.0, 0.0))
    noclip = (-1e9, -1e9, 1e9, 1e9)

    def clips(mode, z0):
        inst, tasks = [], []
        for i in range(6):
            cw, ch = int(rng.randint(40, 160)), int(rng.randint(30, 100))
            tx, ty = (i % 3) * 170, (i // 3) * 128
            sx, sy = int(rng.randint(0, w - cw)), int(rng.randint(0, h - ch))
            rect = (float(sx + 2), float(sy + 2), float(sx + cw - 2), float(sy + ch - 2))
            r = float(rng.randint(3, 15))
            inst.append(clip_rect_instance((0.0, 0.0, float(cw), float(ch)), (float(tx), float(ty)), (float(sx), float(sy)),
                                           1.0, 0, 0, (rect[0], rect[1]), rect, mode, ((r, r),) * 4))
            tasks.append((t.add_render_task((float(tx), float(ty), float(tx + cw), float(ty + ch)), 1.0,
                                            (float(sx), float(sy))), sx, sy, cw, ch))
        prims = []
        for i, (task, sx, sy, cw, ch) in enumerate(tasks):
            a = float(rng.uniform(0.4, 1.0))
            c = tuple(float(v * a) for v in rng.uniform(0, 1, 3)) + (a,)
            hdr = t.add_prim_header((float(sx), float(sy), float(sx + cw), float(sy + ch)), noclip, z0 + i,
                                    t.push_gpu_cache([c]), 0, pic, (65535, 0, 0, 0))
            prims.append(brush_instance(hdr, task, 0xFFFF, 0, 0, 0))
        return (Batch(abi.KIND_CLIP_RECTANGLE, np.stack(inst), blend=abi.BLEND_NONE, features=abi.FEAT_FAST_PATH),
                Batch(abi.KIND_BRUSH_SOLID, np.stack(prims), blend=PM, features=abi.FEAT_ALPHA_PASS, clip_mask="mask"))
    m1, use1 = clips(0.0, 1)
    m2, use2 = clips(1.0, 50)
    textures = {"mask": TextureDesc(abi.FMT_R8, w, h), "a": TextureDesc(abi.FMT_RGBA8, w, h),
                "b": TextureDesc(abi.FMT_RGBA8, w, h)}
    white = Clear(color=(1.0, 1.0, 1.0, 1.0))
    return Frame(t.arrays(), textures, [[Target("mask", ops=[white, m1])], [Target("a", ops=[Clear(color=CLEAR), use1])],
                                        [Target("mask", ops=[white, m2])], [Target("b", ops=[Clear(color=CLEAR), use2])]])


def split_frame(w=256, h=64, singles=1100, targets=3, seed=1):
    """More than QMAX (1024) queued ops in one frame: `singles` one-command solid batches spread over `targets`
    targets of one pass, with a 12-command full-target batch (folded) after every 40th, so the submission splits
    inside the last target with folded batches on both sides of the split."""
    rng = np.random.RandomState(seed)
    per = [[] for _ in range(targets)]
    for i in range(singles):
        ti = i * targets // singles
        per[ti].append([(shape(w, h, int(rng.randint(N_SHAPES)), rng), colour(i, rng), 0)])
        if i % 40 == 39:
            per[ti].append([((0, 0, w, h), colour(k, rng), 0) for k in range(12)])
    return quads_frame(w, h, per)


HAZARDS = {
    "raw": lambda: sampled_target_frame(war=False),
    "war": lambda: sampled_target_frame(war=True),
    "clip_mask": clip_mask_hazard_frame,
    "split": split_frame,
}


# ---- host emulation: the frames above against the oracle --------------------------------------------------


def _emu(frame, names=None, tile_lists=False):
    names = names or _targets(frame)
    assert_same(render(EmuDevice, frame, names, tile_lists=tile_lists), render(OracleDevice, frame, names))


@pytest.mark.parametrize("n", [1, 2, 9])
def test_emu_flat_frames(n):
    _emu(flat_frame(129, 9, n, seed=n))
    _emu(flat_frame(5, 3, n, seed=n + 1, edge=AA_ALL))


def test_emu_many_quads():
    _emu(many_quads_frame(257, 41, 600, seed=1))


@pytest.mark.parametrize("variant", ["copy", "overlap", "scaled", "alpha"])
def test_emu_composite_lists(variant):
    f = composite_list_frame(512, 48, 6, tex=(64, 32) if variant == "scaled" else None, overlap=variant == "overlap",
                             blend=PM if variant == "alpha" else abi.BLEND_NONE)
    _emu(f, tile_lists=True)


@pytest.mark.parametrize("hazard", ["raw", "war", "clip_mask", "split"])
def test_emu_hazard_frames(hazard):
    f = (sampled_target_frame((96, 40), (160, 72), war=hazard == "war") if hazard in ("raw", "war")
         else clip_mask_hazard_frame() if hazard == "clip_mask" else split_frame(40, 16))
    _emu(f)


def test_emu_replicated_depth_frame():
    _emu(replicate(scenes.image_frame(160, 96, n_opaque=3, n_alpha=6, seed=4, occlude_alpha=True), 3))


def test_emu_repeated_yuv_instances():
    _emu(repeated_instances(scenes.yuv_image_frame("nv12", 2, seed=1, width=200, height=120), abi.KIND_BRUSH_YUV_IMAGE, 9))


# ---- GPU: the streaming solid kernel ----------------------------------------------------------------------

FLAT_SIZES = [(1, 1), (3, 2), (5, 3), (127, 7), (129, 9), (515, 131), (1920, 1080)]


@gpu
@pytest.mark.parametrize("size", FLAT_SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("n", [1, 2, 16, 31, 32])
def test_flat_solid(monkeypatch, n, size):
    f = flat_frame(*size, n, seed=n + size[0])
    want = oracle(f)
    default, l_default = render_with(monkeypatch, {}, f)
    flat, l_flat = render_with(monkeypatch, {"WRCU_FLAT_MAX": FLAT_MAX}, f)
    tiled, l_tiled = render_with(monkeypatch, {"WRCU_FLAT_MAX": 0}, f)
    assert_same(default, want, f"default n={n}")
    assert_same(flat, want, f"WRCU_FLAT_MAX={FLAT_MAX} n={n}")
    assert_same(tiled, want, f"WRCU_FLAT_MAX=0 n={n}")
    # the streaming kernel takes the place of the tile kernel, and of the fold in front of it (n >= fold_min)
    fold = 1 if n >= FOLD_MIN else 0
    assert l_flat == l_tiled - fold, (l_flat, l_tiled)
    assert l_default == (l_flat if n == 1 else l_tiled), (l_default, l_flat, l_tiled)


@gpu
@pytest.mark.parametrize("size", [(5, 3), (129, 9), (515, 131)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_flat_declines_non_simple(monkeypatch, size):
    """One AA quad per target: the streaming kernel runs, finds the batch not simple and returns; the generic
    tile kernel draws it."""
    f = flat_frame(*size, 1, seed=3, edge=AA_ALL)
    want = oracle(f)
    for env in ({}, {"WRCU_FLAT_MAX": 0}):
        got, _ = render_with(monkeypatch, env, f)
        assert_same(got, want, f"{env}")


# ---- GPU: strip mode ---------------------------------------------------------------------------------------


def strip_frame(kind, n, targets=1):
    if kind == "linear_gradient":
        f = scenes.gradient_frame(1920, 1080, n_grad=n, seed=n, blend=PM)
    elif kind == "composite":
        f = composite_list_frame(1920, 1080, n, tile=(480, 270), tex=(200, 120), blend=PM, seed=n)
    else:
        f = repeated_instances(scenes.yuv_image_frame("nv12", 2, seed=n, width=1920, height=1080),
                               abi.KIND_BRUSH_YUV_IMAGE, n)
    return replicate(f, targets) if targets > 1 else f


@gpu
@pytest.mark.parametrize("n", [1, 16, 17])
@pytest.mark.parametrize("kind", ["linear_gradient", "composite", "brush_yuv_image"])
def test_strip(monkeypatch, kind, n):
    f = strip_frame(kind, n)
    tl = kind == "composite"
    want = render(OracleDevice, f, _targets(f))
    strip, l_strip = render_with(monkeypatch, {}, f, tile_lists=tl)
    plain, l_plain = render_with(monkeypatch, {"WRCU_STRIP": 0}, f, tile_lists=tl)
    assert_same(strip, want, f"{kind} n={n} default")
    assert_same(plain, want, f"{kind} n={n} WRCU_STRIP=0")
    assert l_strip == l_plain


@gpu
@pytest.mark.parametrize("n", [1, 16])
def test_strip_four_targets(monkeypatch, n):
    """Four targets in one submission: side_reduce lowers max_ctas to one CTA per SM, so strip mode takes longer
    segments."""
    f = strip_frame("linear_gradient", n, targets=4)
    want = oracle(strip_frame("linear_gradient", n))["target"]
    for env in ({}, {"WRCU_STRIP": 0}, {"WRCU_SIDE_CTAS": 3}):
        got, _ = render_with(monkeypatch, env, f)
        assert_same(got, {k: want for k in got}, f"{env} n={n}")


# ---- GPU: set-up granularity (a warp per instance up to 64) -----------------------------------------------

SETUP_FRAMES = {
    "brush_solid_masks": lambda n: scenes.brush_solid_frame(640, 360, n_opaque=4, n_alpha=n, seed=n),
    "brush_image": lambda n: scenes.image_frame(640, 360, n_opaque=4, n_alpha=n, seed=n),
    "text_run": lambda n: scenes.text_frame(1280, 360, n_runs=1, glyphs_per_run=n, seed=n),
    "composite": lambda n: composite_list_frame(2048, 144, n, seed=n),
    # the first fast-path batch holds n_clips * 2 // 3 / 2 clips (scenes.clip_mask_frame): 64 of 192, 65 of 194
    "cs_clip_rectangle": lambda n: scenes.clip_mask_frame(512, 384, n_clips={64: 192, 65: 194}[n], seed=n),
    # the first batch holds n_clips * 2 // 3 clips (scenes.box_shadow_frame): 64 of 96, 65 of 98
    "cs_clip_box_shadow": lambda n: scenes.box_shadow_frame(512, 384, n_clips={64: 96, 65: 98}[n], seed=n),
}


@gpu
@pytest.mark.parametrize("n", [64, 65])
@pytest.mark.parametrize("kind", list(SETUP_FRAMES))
def test_setup_granularity(monkeypatch, kind, n):
    f = SETUP_FRAMES[kind](n)
    tl = kind == "composite"  # n one-tile batches, drawn as one tile list
    sizes = [op.instances.shape[0] for p in f.passes for t in p for op in t.ops if isinstance(op, Batch)]
    assert (len(sizes) if tl else max(sizes)) == n, sizes
    got, _ = render_with(monkeypatch, {}, f, tile_lists=tl)
    assert_same(got, oracle(f), f"{kind} n={n}")


# ---- GPU: bitmask bins and 8192-command list passes --------------------------------------------------------


@gpu
@pytest.mark.parametrize("n", [511, 512, 8192, 8193])
def test_bins_and_list_passes(monkeypatch, n):
    f = many_quads_frame(1920, 1080, n, seed=n)
    got, _ = render_with(monkeypatch, {}, f)
    assert_same(got, oracle(f), f"n={n}")


@gpu
@pytest.mark.parametrize("runs,glyphs", [(7, 73), (8, 64)], ids=["511", "512"])
def test_bins_text(monkeypatch, runs, glyphs):
    f = scenes.text_frame(1920, 1080, n_runs=runs, glyphs_per_run=glyphs, seed=runs)
    got, _ = render_with(monkeypatch, {}, f)
    assert_same(got, oracle(f), f"{runs * glyphs} glyphs")


# ---- GPU: the depth-run prepass -----------------------------------------------------------------------------


@gpu
@pytest.mark.parametrize("targets", [1, 4])
@pytest.mark.parametrize("n_alpha", [47, 48])
def test_depth_prepass(monkeypatch, n_alpha, targets):
    base = scenes.image_frame(640, 360, n_opaque=8, n_alpha=n_alpha, seed=n_alpha, occlude_alpha=True)
    f = replicate(base, targets)
    want = oracle(base)["target"]
    got, launches = render_with(monkeypatch, {}, f)
    assert_same(got, {k: want for k in _targets(f) if k.startswith("t")}, f"n_alpha={n_alpha} targets={targets}")
    _, plain = render_with(monkeypatch, {}, without_depth(f))
    assert launches - plain == depth_launches(f), (launches, plain, depth_launches(f))


# ---- GPU: the scheduler --------------------------------------------------------------------------------------

SCHED_ENVS = {"default": {}, "streams1": {"WRCU_STREAMS": 1}, "streams3": {"WRCU_STREAMS": 3},
              "no_early_clear": {"WRCU_EARLY_CLEAR": 0}, "side_ctas3": {"WRCU_SIDE_CTAS": 3}, "no_pdl": {"WRCU_PDL": 0},
              "immediate": {"WRCU_IMMEDIATE": 1}}


@gpu
@pytest.mark.parametrize("env", list(SCHED_ENVS))
@pytest.mark.parametrize("targets", [1, 2, 3, 4, 8, 9, 17])
def test_targets_of_one_pass(monkeypatch, targets, env):
    base = scenes.image_frame(320, 192, n_opaque=6, n_alpha=20, seed=5, occlude_alpha=True)
    want = oracle(base)["target"]
    f = replicate(base, targets)
    got, _ = render_with(monkeypatch, SCHED_ENVS[env], f, [f"t{i}" for i in range(targets)])
    assert_same(got, {k: want for k in got}, f"{targets} targets {env}")


@gpu
@pytest.mark.parametrize("env", ["default", "streams1", "streams3", "no_early_clear", "no_pdl", "immediate"])
@pytest.mark.parametrize("hazard", list(HAZARDS))
def test_hazards(monkeypatch, hazard, env):
    f = HAZARDS[hazard]()
    got, _ = render_with(monkeypatch, SCHED_ENVS[env], f)
    assert_same(got, oracle(f), f"{hazard} {env}")


# ---- GPU: glyph-major text and the copy-engine composite ------------------------------------------------------


def _text(n):
    return scenes.text_frame(640, 200, n_runs=1, glyphs_per_run=n, seed=3)


@gpu
def test_glyph_major_edge(monkeypatch):
    got = {}
    for n in (7, 8):
        f = _text(n)
        out, got[n] = render_with(monkeypatch, {}, f)
        assert_same(out, oracle(f), f"n={n}")
    out, tile_only = render_with(monkeypatch, {"WRCU_GLYPH_MAJOR": 0}, _text(8))
    assert_same(out, oracle(_text(8)), "n=8 WRCU_GLYPH_MAJOR=0")
    assert got[8] == got[7] + 1 and tile_only == got[7], (got, tile_only)


@gpu
@pytest.mark.parametrize("ctas", [1, 16])
def test_glyph_ctas(monkeypatch, ctas):
    f = scenes.text_frame(1280, 720, n_runs=30, glyphs_per_run=70, seed=ctas)
    got, _ = render_with(monkeypatch, {"WRCU_GLYPH_CTAS": ctas}, f)
    assert_same(got, oracle(f), f"WRCU_GLYPH_CTAS={ctas}")


@gpu
@pytest.mark.parametrize("blend", [abi.BLEND_NONE, PM], ids=["opaque", "alpha"])
def test_copy_engine_edge(monkeypatch, blend):
    """Tile lists of 256x16 tiles on a 2048x272 target: 128 non-overlapping go through wr_composite_copy (+1
    launch), 129 and 128 with one overlapping pair through the ordered tile kernel alone."""
    launches = {}
    for name, n, overlap in (("128", COPY_MAX, False), ("129", COPY_MAX + 1, False), ("overlap", COPY_MAX, True)):
        f = composite_list_frame(2048, 272, n, blend=blend, overlap=overlap, seed=2)
        out, launches[name] = render_with(monkeypatch, {}, f, tile_lists=True)
        assert_same(out, oracle(f), name)
    assert launches["128"] == launches["129"] + 1 and launches["overlap"] == launches["129"], launches
