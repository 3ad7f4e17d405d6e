"""Solid batches deep enough to fold their layers into per-channel lookup tables (csrc/fold.cuh): tiles inside
the batch's common cover take the tables, every other tile the tile kernel.  Byte-exact against the oracle, in
the host emulation (CPU) and on the GPU."""
import numpy as np
import pytest

from oracle.backends import OracleDevice
from webrender_b200 import abi
from webrender_b200.device import CudaDevice
from webrender_b200.frame import Batch, Clear, Frame, Target, TextureDesc
from webrender_b200.gpu_types import FrameTables, INVALID_SEGMENT_INDEX, PART_ALL, QF_APPLY_DEVICE_CLIP, quad_instance
from workloads import scenes

from common import assert_same, render
from emu import EmuDevice

FOLD_MIN = 8  # the library's default batch depth for folding (WRCU_FOLD_MIN, csrc/wrcu_api.cu)
CLEAR = (0.4, 0.7, 0.2, 0.8)


def rects_frame(width, height, batches, targets=1):
    """`targets` render targets of one pass, each cleared and then drawn by the same batches of solid
    premultiplied-alpha quads; `batches` = [[(rect, colour), ...], ...]."""
    t = FrameTables()
    task = t.add_render_task((0.0, 0.0, float(width), float(height)), 1.0, (0.0, 0.0))
    ops = [Clear(color=CLEAR)]
    z = 0
    for cmds in batches:
        inst = []
        for rect, color in cmds:
            z += 1
            prim_f = t.add_quad_prim(rect, rect, color)
            prim_i = t.add_quad_header(0, z)
            inst.append(quad_instance(prim_i, prim_f, QF_APPLY_DEVICE_CLIP, 0, PART_ALL, INVALID_SEGMENT_INDEX, task))
        ops.append(Batch(abi.KIND_QUAD_TEXTURED, np.stack(inst), blend=abi.BLEND_PREMULTIPLIED_ALPHA))
    names = [f"t{i}" for i in range(targets)]
    return Frame(t.arrays(), {n: TextureDesc(abi.FMT_RGBA8, width, height) for n in names},
                 [[Target(n, ops=list(ops)) for n in names]])


def colors(rng, n, over_range=False):
    """Random colours; every 7th layer fully transparent, every 11th opaque.  over_range: lanes above alpha."""
    out = []
    for i in range(n):
        a = 0.0 if i % 7 == 3 else 1.0 if i % 11 == 5 else float(rng.uniform(0.05, 1.0))
        hi = 1.0 if over_range else a
        out.append(tuple(float(v) for v in rng.uniform(0, hi, 3)) + (a,))
    return out


def full_frame(w, h, n, seed):
    return scenes.alpha_rects_frame(w, h, n, seed=seed, color=None, clear_color=CLEAR)


def over_range_frame(w, h, n, seed):
    rng = np.random.RandomState(seed)
    rect = (0.0, 0.0, float(w), float(h))
    return rects_frame(w, h, [[(rect, c) for c in colors(rng, n, over_range=True)]])


def partial_cover_frame(w, h, n, seed):
    """Rects with ragged edges off the tile grid (the common cover is smaller than the bounding box), some
    hanging over the target's edges, and every 9th command off screen."""
    rng = np.random.RandomState(seed)
    cmds = []
    for i, c in enumerate(colors(rng, n)):
        if i % 9 == 4:
            rect = (float(w + 50), float(h + 20), float(w + 400), float(h + 90))
        else:
            x0, y0 = rng.uniform(-20, 45), rng.uniform(-5, 13)
            x1, y1 = w - rng.uniform(-20, 45), h - rng.uniform(-5, 13)
            rect = (float(np.float32(x0)), float(np.float32(y0)), float(np.float32(x1)), float(np.float32(y1)))
        cmds.append((rect, c))
    return rects_frame(w, h, [cmds])


def empty_cover_frame(w, h, n, seed):
    """Left and right halves overlapping by a few pixels, interleaved: no whole tile lies in every rect."""
    rng = np.random.RandomState(seed)
    m = w // 2
    cmds = [(((0.0, 0.0, float(m + 3), float(h)) if i % 2 else (float(m - 3), 0.0, float(w), float(h))), c)
            for i, c in enumerate(colors(rng, n))]
    return rects_frame(w, h, [cmds])


def two_batches_three_targets_frame(w, h, n, seed):
    """Two folded batches in a row on each of three targets of one pass (side streams, one table per batch)."""
    rng = np.random.RandomState(seed)
    rect = (0.0, 0.0, float(w), float(h))
    return rects_frame(w, h, [[(rect, c) for c in colors(rng, n)], [(rect, c) for c in colors(rng, n + 7)]],
                       targets=3)


SCENES = {"over_range": over_range_frame, "partial_cover": partial_cover_frame, "empty_cover": empty_cover_frame,
          "two_batches_three_targets": two_batches_three_targets_frame}


def _targets(f):
    return sorted(f.textures)


# ---- host emulation --------------------------------------------------------------------------------------


@pytest.mark.parametrize("n", [FOLD_MIN - 1, FOLD_MIN, 129])
def test_emu_full_frame_random_colours(n):
    f = full_frame(300, 77, n, seed=n)
    assert_same(render(EmuDevice, f), render(OracleDevice, f), f"n={n}")


@pytest.mark.parametrize("scene", list(SCENES))
def test_emu_scenes(scene):
    f = SCENES[scene](301, 45, 40, seed=3)
    assert_same(render(EmuDevice, f, _targets(f)), render(OracleDevice, f, _targets(f)), scene)


# ---- GPU --------------------------------------------------------------------------------------------------


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(1000, 333), (515, 131)])
@pytest.mark.parametrize("n", [FOLD_MIN - 1, FOLD_MIN, 127, 128, 129, 1000])
def test_full_frame_random_colours(n, size):
    w, h = size
    f = full_frame(w, h, n, seed=n + w)
    assert_same(render(CudaDevice, f), render(OracleDevice, f), f"n={n} size={size}")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [FOLD_MIN, 300])
@pytest.mark.parametrize("scene", list(SCENES))
def test_scenes(scene, n):
    f = SCENES[scene](1000, 333, n, seed=n)
    assert_same(render(CudaDevice, f, _targets(f)), render(OracleDevice, f, _targets(f)), f"{scene} n={n}")
