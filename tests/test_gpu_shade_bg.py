"""The folded background of K3's miss launch.

A background of the form the JSON loader builds (a constant, image or gradient colour with constant strength and offset) is
folded at upload and sampled inline by the miss launch; any other background keeps the node interpreter.

* CPU: the background classification of every golden, bundled and synthetic scene against an independent reading of its graph.
* GPU: the frame digests of tests/golden/shade_frames.sha256.json (test_gpu_shade_order.py, test_gpu_ray_order.py), the aimed
  background directions of test_gpu_shade.py (±y with ±0 components, subnormal and large unnormalised directions, syn_shading's
  gradient with an offset) and the oracle frame tests run the folded miss launch end to end.
"""
import ctypes as C

import pytest

import crgpu
from test_gpu_shade import NODE_DTYPE, _view, scenes          # noqa: F401  (scenes: a fixture flat_scenes uses)
from test_gpu_shade_flat import CLASS_SCENES, _load, flat_scenes   # noqa: F401  (flat_scenes is a fixture)

# include/crscene.h node kinds
BACKGROUND, COLOR_CONSTANT, COLOR_IMAGE, COLOR_GRADIENT, VALUE_CONSTANT = 9, 32, 33, 35, 64
# crgpu_prepared_background
BG_NONE, BG_CONSTANT, BG_IMAGE, BG_GRADIENT = 0, 1, 2, 3


# ------------------------------------------------------------------------------------------------ classification (CPU)
def device_background(path):
    L, f = _load(path)
    L.crgpu_prepare.argtypes = [C.POINTER(crgpu.FlatScene), C.POINTER(C.c_void_p)]
    L.crgpu_prepared_free.argtypes = [C.c_void_p]
    p = C.c_void_p()
    rc = L.crgpu_prepare(C.byref(f), C.byref(p))
    L.crscene_free(C.byref(f))
    assert rc == 0, path
    kind = C.c_uint32(99)
    rc = L.crgpu_prepared_background(p, C.byref(kind))
    L.crgpu_prepared_free(p)
    assert rc == 0
    return kind.value


def expected_background(path):
    """(kind, colour node) read off the node graph here"""
    L, f = _load(path)
    nodes = _view(f.nodes, f.node_count, NODE_DTYPE).copy()
    root = int(f.background)
    L.crscene_free(C.byref(f))
    assert nodes[root]["kind"] == BACKGROUND
    colour, strength, offset = (int(i) for i in nodes[root]["in"])
    if nodes[strength]["kind"] != VALUE_CONSTANT or nodes[offset]["kind"] != VALUE_CONSTANT:
        return BG_NONE, None
    return {COLOR_CONSTANT: BG_CONSTANT, COLOR_IMAGE: BG_IMAGE, COLOR_GRADIENT: BG_GRADIENT}.get(int(nodes[colour]["kind"]), BG_NONE), nodes[offset]


@pytest.mark.parametrize("name", CLASS_SCENES)
def test_background_classification(name, flat_scenes):
    if name not in flat_scenes:
        pytest.skip(f"{name}: bundled scenes need scenes/_built or oracle/_ref/input")
    kind = device_background(flat_scenes[name])
    want, offset = expected_background(flat_scenes[name])
    assert kind == want, (name, kind, want)
    if name in ("hdr", "g_nodes"):                       # an HDR environment map (g_nodes: with an offset)
        assert kind == BG_IMAGE
    if name == "syn_shading":                            # a gradient with an offset
        assert kind == BG_GRADIENT and offset["f"][0] != 0.0
