"""What wrcu_draw_batch returns for a batch it must refuse, for every program kind: an instance stride below the
kind's record, an unbound or wrongly formatted sampler, an unsupported feature, an unknown kind, the dual-source
blend.  Every case is decided on the host before anything is queued, so the same cases run on the host emulation
(CPU) and on the GPU.

One context per device serves all cases.  The sticky error (wrcu_get_error) is cleared before each draw and read
back after it: it must hold exactly what the draw returned."""
import ctypes as C

import numpy as np
import pytest

from webrender_b200 import abi
from webrender_b200.device import CudaDevice, WrcuError, load_library
from webrender_b200.gpu_types import ortho

import emu
from emu import EmuDevice

W = H = 64
RGBA8, R8 = abi.FMT_RGBA8, abi.FMT_R8

# kind: (minimum instance stride, samplers that must be bound, format sColor0 must have)
KINDS = {
    abi.KIND_QUAD_TEXTURED: (16, (), None),
    abi.KIND_QUAD_MASK: (32, (), None),
    abi.KIND_BRUSH_SOLID: (16, (), None),
    abi.KIND_BRUSH_IMAGE: (16, (0,), None),
    abi.KIND_BRUSH_LINEAR_GRADIENT: (16, (), None),
    abi.KIND_BRUSH_BLEND: (16, (0,), None),
    abi.KIND_BRUSH_MIX_BLEND: (16, (0, 1), None),
    abi.KIND_BRUSH_OPACITY: (16, (0,), None),
    abi.KIND_TEXT_RUN: (16, (0,), None),
    abi.KIND_CLIP_RECTANGLE: (200, (), None),
    abi.KIND_CLIP_BOX_SHADOW: (84, (0,), R8),
    abi.KIND_COMPOSITE: (120, (0,), None),
    abi.KIND_CLEAR: (32, (), None),
    abi.KIND_BLUR: (24, (0,), None),
    abi.KIND_SCALE: (36, (0,), None),
    abi.KIND_FAST_LINEAR_GRADIENT: (52, (), None),
    abi.KIND_LINEAR_GRADIENT: (48, (), None),
    abi.KIND_RADIAL_GRADIENT: (52, (), None),
    abi.KIND_CONIC_GRADIENT: (52, (), None),
    abi.KIND_LINE_DECORATION: (36, (), None),
    abi.KIND_BORDER_SOLID: (108, (), None),
    abi.KIND_BORDER_SEGMENT: (108, (), None),
    abi.KIND_QUAD_RADIAL_GRADIENT: (16, (), None),
    abi.KIND_QUAD_CONIC_GRADIENT: (16, (), None),
    abi.KIND_BRUSH_YUV_IMAGE: (16, (0,), None),
    abi.KIND_SPLIT_COMPOSITE: (16, (0,), RGBA8),
}
assert sorted(KINDS) == list(range(1, 27))
FMT_NAME = {RGBA8: "RGBA8", R8: "R8"}
EMPTY = (0, 0, 0, 0)


def _case(id, kind, stride, features=None, unbound=(), fmt0=None, blend=abi.BLEND_PREMULTIPLIED_ALPHA,
          scissor=None, rc=abi.ERR_INVALID, msg=None):
    """One draw of a single zero-filled instance.  Samplers the kind requires are bound (sColor0 in the format it
    requires, else `fmt0` or RGBA8) except those in `unbound`; cs_blur gets COLOR_TARGET unless `features` says
    otherwise.  `msg`: a word the error string must contain."""
    if features is None:
        features = abi.FEAT_COLOR_TARGET if kind == abi.KIND_BLUR else 0
    spec = KINDS.get(kind, (0, (), None))
    samplers = {s: (fmt0 or spec[2] or RGBA8) if s == 0 else RGBA8 for s in spec[1] if s not in unbound}
    return pytest.param(kind, features, stride, samplers, blend, scissor, rc, msg, id=id)


CASES = []
for kind, (stride, samplers, fmt0) in KINDS.items():
    name = abi.KIND_PROGRAM[kind]
    CASES.append(_case(f"{name}-short-stride", kind, stride - 1, msg="stride"))
    for s in samplers:
        CASES.append(_case(f"{name}-no-sColor{s}", kind, stride, unbound=(s,), msg=f"sColor{s}"))
    if fmt0 is not None:
        wrong = R8 if fmt0 == RGBA8 else RGBA8
        CASES.append(_case(f"{name}-sColor0-{FMT_NAME[wrong]}", kind, stride, fmt0=wrong, msg=FMT_NAME[fmt0]))
    CASES.append(_case(f"{name}-dual-source-blend", kind, stride, blend=abi.BLEND_SUBPIXEL_DUAL_SOURCE,
                       rc=abi.ERR_UNSUPPORTED))
    # the scissor test comes first: a batch that draws nothing is accepted whatever else is wrong with it
    CASES.append(_case(f"{name}-empty-scissor-short-stride", kind, stride - 1, scissor=EMPTY, rc=abi.OK))
# validation order: stride, then a refused feature, then samplers, then cs_blur's target feature
DUAL = abi.FEAT_DUAL_SOURCE_BLENDING
CASES += [
    _case("brush_image-DUAL_SOURCE_BLENDING", abi.KIND_BRUSH_IMAGE, 16, features=DUAL, rc=abi.ERR_UNSUPPORTED,
          msg="DUAL_SOURCE_BLENDING"),
    _case("brush_image-DUAL_SOURCE_BLENDING-no-sColor0", abi.KIND_BRUSH_IMAGE, 16, features=DUAL, unbound=(0,),
          rc=abi.ERR_UNSUPPORTED, msg="DUAL_SOURCE_BLENDING"),
    _case("brush_image-DUAL_SOURCE_BLENDING-short-stride", abi.KIND_BRUSH_IMAGE, 15, features=DUAL, msg="stride"),
    _case("cs_blur-no-target-feature", abi.KIND_BLUR, 24, features=0, msg="ALPHA_TARGET"),
    _case("cs_blur-no-target-feature-no-sColor0", abi.KIND_BLUR, 24, features=0, unbound=(0,), msg="sColor0"),
]
for kind in (0, 27, -1):
    CASES.append(_case(f"kind{kind}", kind, 256, rc=abi.ERR_UNSUPPORTED))
    CASES.append(_case(f"kind{kind}-empty-scissor", kind, 256, scissor=EMPTY, rc=abi.OK))


@pytest.fixture(scope="module", params=[pytest.param(EmuDevice, id="emu"),
                                        pytest.param(CudaDevice, id="cuda", marks=pytest.mark.gpu)])
def device(request):
    """A device with a bound RGBA8 target and one RGBA8 and one R8 texture to sample."""
    d = request.param()
    tex = {fmt: d.texture_create(fmt, 8, 8) for fmt in (RGBA8, R8)}
    target = d.texture_create(RGBA8, W, H)
    d.target_bind(target, 0, ortho(W, H), (0, 0, W, H))
    yield d, tex
    d.close()


@pytest.mark.parametrize("kind, features, stride, samplers, blend, scissor, rc, msg", CASES)
def test_draw_batch_refuses(device, kind, features, stride, samplers, blend, scissor, rc, msg):
    d, tex = device
    get_error = d._f("get_error")
    get_error(d.ctx)
    colors = [tex[samplers[s]] if s in samplers else 0 for s in range(3)]
    try:
        d.draw_batch(kind, features, blend, abi.DEPTH_OFF, colors, 0, scissor, (0.0,) * 4,
                     np.zeros((1, stride), np.uint8))
        got, text = abi.OK, ""
    except WrcuError as e:
        got, text = e.code, str(e)
    assert got == rc, text
    assert get_error(d.ctx) == rc
    if msg:
        assert msg in text


@pytest.mark.parametrize("lib", ["emu", "cuda"])
@pytest.mark.parametrize("kind", sorted(KINDS), ids=[abi.KIND_PROGRAM[k] for k in sorted(KINDS)])
def test_program_name_round_trips(lib, kind):
    """Host code only: the CUDA library answers without a device."""
    if lib == "emu":
        fn = C.CDLL(emu.build()).wremu_program_from_name
    else:
        fn = load_library().wrcu_program_from_name
    fn.argtypes = [C.c_char_p, C.POINTER(C.c_int), C.POINTER(C.c_uint32)]
    k, f = C.c_int(), C.c_uint32()
    assert fn(abi.KIND_PROGRAM[kind].encode(), C.byref(k), C.byref(f)) == abi.OK
    assert (k.value, f.value) == (kind, 0)
