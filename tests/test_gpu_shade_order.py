"""GPU tests of the shading step (K4 + K3): the order and the batch in which the live rays are shaded never change a frame.

Every path carries its own RNG state and id, so a change to how K3 orders, groups or stages its rays must leave the frames
bit-identical.  tests/golden/shade_frames.sha256.json holds the SHA-256 of frames rendered on an H100 by the global
key-sorted K3 (K4's bucket order, a miss launch and a hit launch): g_nodes, g_f4 (the complete node interpreter), hdr at
240x135x16 with 32 bounces, refraction at 240x135x8 with 512 bounces (the tail kernel), 300 sphere materials (saturated
keys), a scene in which every camera ray misses (the next bounce has no live ray) and one in which every camera ray hits.

The live counts K3 sees are chosen directly by rendering one pass of a pixel set of a given size: the first bounce then has
exactly that many rays.  Each such render must reproduce those pixels of the whole-frame render bit for bit.

Regenerate the digests (only when the frame is meant to change): python tests/test_gpu_shade_order.py tests/golden/shade_frames.sha256.json
"""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

if __name__ == "__main__":
    _root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path[:0] = [os.path.join(_root, "c-ray_b200"), os.path.join(_root, "tests")]

import crgpu
import oracle_lib as O
from conftest import GOLDEN
from test_gpu_trace import _flatten, _write_synthetic

pytestmark = pytest.mark.gpu
DIGESTS = os.path.join(GOLDEN, "shade_frames.sha256.json")
# (name, W, H, spp, bounces, max paths in flight); 0 = the scene's value / the library default.  hdr runs several batches per
# frame, so the two wave sets overlap.
FRAMES = [("g_nodes", 0, 0, 0, 0, 0), ("g_f4", 0, 0, 0, 0, 0), ("hdr", 240, 135, 16, 32, 240 * 135 * 4),
          ("refraction", 240, 135, 8, 512, 0), ("syn_materials", 0, 0, 0, 0, 0), ("syn_allmiss", 0, 0, 0, 0, 0),
          ("syn_nomiss", 0, 0, 0, 0, 0)]
# first-bounce live counts: one ray, partial warps, around one and two blocks of 256 threads, counts that are not a multiple of 16
LIVE_COUNTS = [1, 15, 77, 255, 256, 257, 511, 512, 513, 1003]


def _write_edge_scenes(d):
    """every camera ray misses (a sphere behind the camera), every camera ray hits (the camera inside a sphere)"""
    cam = {"FOV": 70}
    out = {}
    for name, z, r in (("syn_allmiss", -5, 1.0), ("syn_nomiss", 0, 20.0)):
        sc = {"renderer": {"width": 40, "height": 30, "samples": 4, "bounces": 6}, "camera": cam,
              "scene": {"ambientColor": {"down": [1, 1, 1], "up": [0.5, 0.7, 1.0]}, "meshes": [],
                        "primitives": [{"type": "sphere", "radius": r, "color": [0.7, 0.6, 0.5],
                                        "instances": [{"transforms": [{"type": "translate", "Z": z}]}]}]}}
        p = os.path.join(d, name + ".json")
        open(p, "w").write(json.dumps(sc))
        out[name] = p
    return out


def scene_paths(d):
    """name -> flat .crscene of every scene in FRAMES that can be built here"""
    os.makedirs(d, exist_ok=True)
    out = {n: os.path.join(GOLDEN, n + ".crscene") for n in ("g_nodes", "g_f4")}
    for n in ("hdr", "refraction"):
        p = O.bundled_scene(n, d)
        if p:
            out[n] = p
    js = _write_synthetic(os.path.join(d, "syn"))
    js.update(_write_edge_scenes(d))
    for n in ("syn_materials", "syn_allmiss", "syn_nomiss"):
        out[n] = _flatten(js[n], os.path.join(d, n + ".crscene"))
    return out


def render_digests(paths):
    out = {}
    for name, W, H, spp, b, mp in FRAMES:
        if name not in paths:
            continue
        g = crgpu.GpuScene(paths[name], W, H, spp, b)
        if mp:
            g.set_max_paths(mp)
        g.render_frame()
        out[name] = hashlib.sha256(g.read().tobytes()).hexdigest()
        g.close()
    return out


@pytest.fixture(scope="module")
def paths(tmp_path_factory):
    return scene_paths(str(tmp_path_factory.mktemp("shade_scenes")))


def test_frames_match_recorded_digests(paths):
    want = json.load(open(DIGESTS))
    got = render_digests(paths)
    assert {"g_nodes", "g_f4", "syn_materials", "syn_allmiss", "syn_nomiss"} <= set(got)
    bad = [n for n in got if got[n] != want[n]]
    assert not bad, bad


def _pixel_set(W, k):
    """rectangles covering the first k pixels of the frame in row order (y = 0 first; the framebuffer stores y = 0 last)"""
    rects = [(0, 0, W, k // W)] if k >= W else []
    if k % W:
        rects.append((0, k // W, k % W, k // W + 1))
    return rects


@pytest.mark.parametrize("name", ["g_nodes", "hdr"])
def test_live_counts_reproduce_the_frame(name, paths):
    if name not in paths:
        pytest.skip(f"{name} not available")
    W, H = (0, 0) if name == "g_nodes" else (240, 135)
    g = crgpu.GpuScene(paths[name], W, H, 0, 0)
    g.render_tile(0, 0, g.W, g.H, 0, 1)
    whole = g.read()[::-1].reshape(-1, 3)
    assert g.W * g.H > max(LIVE_COUNTS)
    for k in LIVE_COUNTS:
        g.clear()
        st = g.render_tiles(_pixel_set(g.W, k), 0, 1)
        assert st["paths"] == k
        img = g.read()[::-1].reshape(-1, 3)
        assert np.array_equal(img[:k].view(np.uint32), whole[:k].view(np.uint32)), k
        assert not img[k:].any(), k
    g.close()


if __name__ == "__main__":
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        dig = render_digests(scene_paths(d))
    open(sys.argv[1], "w").write(json.dumps(dig, indent=1, sort_keys=True) + "\n")
    print(dig)
