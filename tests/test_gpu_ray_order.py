"""Tests of the order in which the traversal kernel (K2) takes the rays of a bounce (CRGPU_TRACE_SORT).

Modes 1-4 sort the next bounce's rays by a key K3 writes (K4b, `k_bucket<true>`); mode 4's key is the direction octant and a
5-bit Morton cell of the origin inside the bounds of the origins K3 wrote at the same depth in the previous batch of the wave
set (WaveBuffers::box).  The order rays are traced in never changes a result, so every mode must render the recorded frames
bit for bit, including scenes where the bounds are empty (every camera ray misses), a single surface (the camera inside a
sphere) and origins of magnitude 1e6.

The CPU test checks, on the oracle's bounce-1 rays of hdr.json, that mode 4's origin cell is not degenerate: the world box
(mode 3) puts every secondary origin of hdr.json in one cell, because the emissive spheres stretch the box to ~1500 units.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "c-ray_b200"), os.path.join(ROOT, "tests")]

from conftest import GOLDEN   # noqa: E402

SORT_MODES = ["0", "1", "2", "3", "4"]

_CODE = r"""
import hashlib, json, sys
sys.path[:0] = sys.argv[1:3]
import crgpu
out = {}
for name, path, W, H, spp, b, mp in json.loads(sys.argv[3]):
    g = crgpu.GpuScene(path, W, H, spp, b)
    if mp:
        g.set_max_paths(mp)
    st = g.render_frame()
    out[name] = [hashlib.sha256(g.read().tobytes()).hexdigest(), int(st["rays"])]
    g.close()
print("FRAMES " + json.dumps(out))
"""


def _render(env, jobs):
    e = {k: v for k, v in os.environ.items() if not k.startswith("CRGPU_")}
    e.update(env)
    r = subprocess.run([sys.executable, "-c", _CODE, os.path.join(ROOT, "c-ray_b200"), os.path.join(ROOT, "tests"), json.dumps(jobs)],
                       env=e, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("FRAMES ")]
    assert r.returncode == 0 and lines, r.stdout[-2000:]
    return json.loads(lines[-1][7:])


def _write_far_scene(d):
    """every origin of magnitude ~1e6: the camera looks at a sphere of radius 5e5 centred 1e6 units away"""
    sc = {"renderer": {"width": 40, "height": 30, "samples": 4, "bounces": 6}, "camera": {"FOV": 70},
          "scene": {"ambientColor": {"down": [1, 1, 1], "up": [0.5, 0.7, 1.0]}, "meshes": [],
                    "primitives": [{"type": "sphere", "radius": 5.0e5, "color": [0.7, 0.6, 0.5],
                                    "instances": [{"transforms": [{"type": "translate", "X": 1.0e6, "Y": 1.0e6, "Z": 1.0e6}]}]},
                                   {"type": "sphere", "radius": 5.0e5, "color": [0.3, 0.6, 0.5],
                                    "instances": [{"transforms": [{"type": "translate", "Z": 1.0e6}]}]}]}}
    p = os.path.join(d, "syn_far.json")
    open(p, "w").write(json.dumps(sc))
    return p


@pytest.mark.gpu
def test_every_sort_mode_reproduces_the_frames(tmp_path):
    """CRGPU_TRACE_SORT = 0..4: the frames of tests/golden/shade_frames.sha256.json reproduce their digests (hdr at 240x135x16
    runs several batches on two wave sets, so mode 4 keys with the bounds of an earlier batch), the far-origin scene renders the
    bits of the unsorted run, and every mode traces exactly as many rays as the unsorted run."""
    from test_gpu_shade_order import FRAMES, scene_paths
    from test_gpu_trace import _flatten
    paths = scene_paths(str(tmp_path / "scenes"))
    paths["syn_far"] = _flatten(_write_far_scene(str(tmp_path)), str(tmp_path / "syn_far.crscene"))
    jobs = [[n, paths[n], W, H, spp, b, mp] for n, W, H, spp, b, mp in FRAMES if n in paths] + [["syn_far", paths["syn_far"], 0, 0, 0, 0, 0]]
    want = json.load(open(os.path.join(GOLDEN, "shade_frames.sha256.json")))
    base = _render({"CRGPU_TRACE_SORT": "0"}, jobs)
    assert {"g_nodes", "syn_allmiss", "syn_nomiss", "syn_far"} <= set(base)
    bad = [("0", n) for n in base if n in want and base[n][0] != want[n]]
    for mode in SORT_MODES[1:]:
        got = _render({"CRGPU_TRACE_SORT": mode}, jobs)
        bad += [(mode, n) for n in base if got[n] != base[n]]       # digest and ray count
    assert not bad, bad


def _mode4_cells(o):
    """the origin cell of mode 4 (crgpu_shade.cu cr_dir_bin) for origins o (n, 3) float32 in the bounds of the same origins"""
    lo, hi = o.min(axis=0), o.max(axis=0)
    e = hi - lo
    scale = np.where((e > 0) & (e < 3.0e38), np.float32(4.0) / np.where(e > 0, e, 1), 0).astype(np.float32)
    c = np.clip(np.nan_to_num((o - lo) * scale, nan=0.0), 0, 3).astype(np.int64)
    m = (c[:, 0] & 1) | ((c[:, 1] & 1) << 1) | ((c[:, 2] & 1) << 2) | ((c[:, 0] >> 1) << 3) | ((c[:, 1] >> 1) << 4) | ((c[:, 2] >> 1) << 5)
    return m >> 1


def test_origin_cell_spreads_hdr_bounce1():
    """On hdr.json at 240x135, one pass, the oracle's 25,783 bounce-1 rays fill 18 of the 32 cells and the largest cell holds 33%
    of them (measured).  The world box of mode 3 holds every one of them in a single cell."""
    if not os.path.exists(os.path.join(ROOT, "scenes", "_built", "hdr.crscene")):
        pytest.skip("scenes/_built/hdr.crscene not built")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import k2_warp_model as M
    _, geo = M.load_traces("hdr", 240, 135, 0, 0, 240, 135, 1)
    o = geo[1][:, :3].astype(np.float32)
    assert len(o) > 20000
    cnt = np.bincount(_mode4_cells(o), minlength=32)
    assert (cnt > 0).sum() >= 12, cnt
    assert cnt.max() / cnt.sum() < 0.45, cnt

