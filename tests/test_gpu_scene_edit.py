"""Editing a resident GPU scene between renders (crgpu_scene_set_camera / crgpu_scene_set_instances, include/crgpu.h).

The target is exact: a scene A edited with the camera and instances of a scene B renders the same bits as B loaded fresh from its
JSON.  B is loaded from edited JSON text (crscene.load_json_buf) and configured at the test's size, so its camera is the one the
edit installs.  Besides the framebuffer, the instrumented traversal (count = 1) over a fixed ray set must return the same records
and the same P/T/S/I counts, which pins the shape and BFS packing of the rebuilt top-level BVH.

CPU: argument checks of the new entry points.  GPU: everything else.
"""
import copy
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import crgpu
import crscene
from conftest import GOLDEN, ROOT

REFDIR = os.path.join(ROOT, "oracle", "_ref")
DIGESTS = os.path.join(GOLDEN, "shade_frames.sha256.json")
SMALL = (240, 135, 4)                                   # W, H, spp of the comparisons (bounces: the scene's frame setting)
BOUNCES = {"hdr": 32, "venus": 25, "refraction": 512}
STEP = {"hdr": 0.02, "venus": 20.0, "refraction": 20.0}     # a camera / mesh move of about one percent of the scene
# the configurations of tests/golden/shade_frames.sha256.json (W, H, spp, bounces, max paths in flight)
GOLDEN_FRAMES = {"hdr": (240, 135, 16, 32, 240 * 135 * 4), "refraction": (240, 135, 8, 512, 240 * 135 * 2)}


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


# ---- CPU -----------------------------------------------------------------------------------------------------------------------

def test_entry_points_reject_null_arguments():
    L = crgpu.lib()
    cam = crgpu.Camera()
    inst = np.zeros(1, dtype=crscene.INSTANCE)
    assert L.crgpu_scene_set_camera(None, None) == -3
    assert L.crgpu_scene_set_camera(None, C.byref(cam)) == -3
    assert L.crgpu_scene_set_instances(None, None, 0) == -3
    assert L.crgpu_scene_set_instances(None, inst.ctypes.data, 1) == -3


def test_no_scene_to_edit_without_a_device():
    """Without a GPU no scene exists to edit: creating one fails loudly (CRGPU_ERR_NO_DEVICE), never on the CPU."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    L = crgpu.lib()
    h = C.c_void_p()
    flat = crgpu.FlatScene()
    assert L.crscene_load(C.byref(flat), os.path.join(GOLDEN, "g_single.crscene").encode()) == 0
    assert L.crgpu_scene_create(C.byref(flat), 0, C.byref(h)) == -1
    L.crscene_free(C.byref(flat))
    with pytest.raises(crgpu.CrgpuError):
        crgpu.GpuScene(os.path.join(GOLDEN, "g_single.crscene")).set_camera(crgpu.Camera())


# ---- helpers ---------------------------------------------------------------------------------------------------------------------

def scene_json(name):
    path = os.path.join(REFDIR, "input", name + ".json")
    if not os.path.exists(path):
        pytest.skip(f"{name}.json not available")
    return json.load(open(path))


def load(doc, cwd=REFDIR, asset_path="input"):
    """A FlatScene from JSON text, with assets resolved as the bundled scenes are (oracle_lib.bundled_scene) unless the scene's own
    working directory and mesh directory are given."""
    here = os.getcwd()
    os.chdir(cwd)
    try:
        return crscene.load_json_buf(json.dumps(doc), asset_path)
    finally:
        os.chdir(here)


class Loaded:
    """A flat scene configured at W x H x spp, bounces, with its camera and instances kept for edits."""

    def __init__(self, doc, W, H, spp, b, cwd=REFDIR, asset_path="input"):
        self.flat = load(doc, cwd, asset_path)
        crgpu.lib().crscene_set_config(C.byref(self.flat), W, H, spp, b)
        self.cfg = (W, H, spp, b)
        self.camera = crgpu.Camera.from_buffer_copy(self.flat.camera)
        self.instances = crscene.arrays(self.flat)["instances"]

    def upload(self, max_paths=None):
        W, H, spp, b = self.cfg
        g = crgpu.GpuScene.__new__(crgpu.GpuScene)
        g.handle = C.c_void_p()
        crgpu._check(crgpu.lib().crgpu_scene_create(C.byref(self.flat), 0, C.byref(g.handle)), "crgpu_scene_create")
        g.W, g.H, g.samples, g.bounces = W, H, spp, b
        if max_paths:
            g.set_max_paths(max_paths)
        return g

    def free(self):
        crscene.free(self.flat)


def full(g):
    g.clear()
    g.render_tile(0, 0, g.W, g.H)
    return g.read().copy()


def ray_set(cam, n=20000, seed=7):
    """Rays from the camera position in a wide cone around its forward axis, and from points around it."""
    rng = np.random.default_rng(seed)
    A = np.array(cam.A, dtype=np.float64).reshape(4, 4)
    o = np.repeat(A[:3, 3][None, :], n, axis=0)
    fwd = np.array(cam.forward, dtype=np.float64)
    d = fwd[None, :] + 0.4 * rng.standard_normal((n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    o[n // 2:] += rng.standard_normal((n - n // 2, 3)) * 0.05 * np.abs(A[:3, 3]).max()
    return np.concatenate([o, d], axis=1).astype(np.float32)


def traced(g, rays):
    rec, _perm, misses, st = g.trace_rays(rays, count=1)
    return rec, misses, tuple(st[k] for k in ("node_pairs", "tri_tests", "sphere_tests", "inst_visits"))


def assert_same_as_fresh(g, b, rays):
    """g (edited) renders and traces exactly as a fresh upload of b."""
    fresh = b.upload()
    try:
        want_img, want_tr = full(fresh), traced(fresh, rays)
    finally:
        fresh.close()
    img, tr = full(g), traced(g, rays)
    assert img.tobytes() == want_img.tobytes(), "edited frame differs from the fresh scene's"
    assert tr[0].tobytes() == want_tr[0].tobytes(), "edited scene's ray records differ"
    assert tr[1:] == want_tr[1:], f"edited scene traces with other counts: {tr[1:]} vs {want_tr[1:]}"


def edit(g, b):
    g.set_camera(b.camera)
    g.set_instances(b.instances)


def _bump_translate(tr, step):
    for k in ("x", "y", "z"):
        if k in tr:
            tr[k] = tr[k] + step


def edited(doc, step):
    """Camera moved and turned; sphere 0 moved far out (the world box grows); spheres 1 and 2 swap places; the last mesh instance is
    scaled, rotated and moved."""
    d = copy.deepcopy(doc)
    far = 6000.0
    for tr in d["camera"]["transforms"]:
        if tr["type"] == "translate":
            _bump_translate(tr, step)
        elif tr["type"].startswith("rotate"):
            tr["degrees"] = tr.get("degrees", 0) + 2
    prims = d["scene"]["primitives"]
    prims[0]["instances"][0]["transforms"].append({"type": "translate", "x": far, "y": 0, "z": 0})
    prims[1]["instances"], prims[2]["instances"] = prims[2]["instances"], prims[1]["instances"]
    mesh = [m for m in d["scene"]["meshes"] if m["instances"][0]["transforms"]][-1]
    tf = mesh["instances"][0]["transforms"]
    for tr in tf:
        if tr["type"] == "scaleUniform":
            tr["scale"] = tr["scale"] * 1.1
        elif tr["type"] == "rotateY":
            tr["degrees"] = tr.get("degrees", 0) + 10
        elif tr["type"] == "translate":
            _bump_translate(tr, step)
    tf.append({"type": "rotateY", "degrees": 5})
    return d


# ---- GPU: bundled scenes -----------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", ["hdr", "venus", "refraction"])
def test_edited_scene_renders_as_the_fresh_scene(name):
    doc = scene_json(name)
    W, H, spp = SMALL
    a, b = Loaded(doc, W, H, spp, BOUNCES[name]), Loaded(edited(doc, STEP[name]), W, H, spp, BOUNCES[name])
    for f in ("kind", "object"):
        assert np.array_equal(a.instances[f], b.instances[f])
    assert a.instances.tobytes() != b.instances.tobytes()
    g = a.upload()
    try:
        rays = ray_set(b.camera)
        edit(g, b)
        assert_same_as_fresh(g, b, rays)
    finally:
        g.close()
        a.free()
        b.free()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GOLDEN_FRAMES))
def test_editing_back_gives_the_committed_frames(name):
    doc = scene_json(name)
    W, H, spp, bounces, mp = GOLDEN_FRAMES[name]
    a, b = Loaded(doc, W, H, spp, bounces), Loaded(edited(doc, STEP[name]), W, H, spp, bounces)
    g = a.upload(max_paths=mp)
    try:
        edit(g, b)
        moved = full(g)
        edit(g, a)
        back = full(g)
        want = json.load(open(DIGESTS))[name]
        assert digest(back) == want
        assert digest(moved) != want
    finally:
        g.close()
        a.free()
        b.free()


# ---- GPU: generated scenes -----------------------------------------------------------------------------------------------------

def sphere_scene(positions, groups=1, meshes=(), radius=6.0):
    """A JSON scene of sphere instances (split over `groups` sphere primitives, so several instances share an object) and the given
    mesh entries, looking at the region of the bundled refraction scene."""
    base = scene_json("refraction")
    d = {k: copy.deepcopy(base[k]) for k in ("version", "renderer", "display", "camera")}
    d["scene"] = {"ambientColor": copy.deepcopy(base["scene"]["ambientColor"]), "meshes": list(meshes), "primitives": []}
    per = -(-len(positions) // groups)
    for gi in range(groups):
        chunk = positions[gi * per:(gi + 1) * per]
        if not len(chunk):
            continue
        d["scene"]["primitives"].append({
            "type": "sphere", "radius": radius + gi % 5, "bsdf": ("lambertian", "metal")[gi % 2], "reflectivity": 1.0,
            "roughness": 0.1, "color": {"r": 0.2 + 0.6 * (gi % 3) / 2, "g": 0.5, "b": 0.8 - 0.6 * (gi % 4) / 3},
            "instances": [{"transforms": [{"type": "translate", "x": float(p[0]), "y": float(p[1]), "z": float(p[2])}]} for p in chunk]})
    return d


def spread(n, seed):
    rng = np.random.default_rng(seed)
    lo, hi = np.array([700.0, 250.0, 850.0]), np.array([1300.0, 650.0, 1600.0])
    return np.round(lo + (hi - lo) * rng.random((n, 3)), 3)


def teapots(shift=0.0):
    base = scene_json("refraction")
    out = []
    for m in base["scene"]["meshes"]:
        if m["fileName"].startswith("teapot"):
            m = copy.deepcopy(m)
            if shift:
                m["instances"][0]["transforms"].append({"type": "translate", "x": shift, "y": 0, "z": -shift})
            out.append(m)
    return out


def check_edit(doc_a, doc_b, cfg=(160, 90, 2, 8), repeat=1):
    a, b = Loaded(doc_a, *cfg), Loaded(doc_b, *cfg)
    g = a.upload()
    try:
        for _ in range(repeat):
            edit(g, b)
        assert_same_as_fresh(g, b, ray_set(b.camera))
    finally:
        g.close()
        a.free()
        b.free()


@pytest.mark.gpu
def test_many_instances_all_moved():
    """About 20k sphere instances of 40 objects and the teapot instances, all moved: the builder runs through many levels, and the
    ray offset of each sphere object comes from its last instance."""
    pos = spread(20000, 1)
    moved = pos + np.round(np.random.default_rng(2).normal(0.0, 15.0, pos.shape), 3)
    check_edit(sphere_scene(pos, groups=40, meshes=teapots(), radius=2.0),
               sphere_scene(moved, groups=40, meshes=teapots(60.0), radius=2.0))


@pytest.mark.gpu
def test_single_instance_top_level_is_a_leaf():
    check_edit(sphere_scene(spread(1, 3), radius=60.0), sphere_scene(spread(1, 4), radius=60.0))


@pytest.mark.gpu
def test_coincident_instances_take_the_median_fallback():
    pos = spread(40, 5)
    same = np.repeat(pos[:1], 40, axis=0)
    check_edit(sphere_scene(pos, groups=4), sphere_scene(same, groups=4))


@pytest.mark.gpu
def test_spreading_coincident_instances_grows_the_top_level():
    """12 coincident instances upload as one leaf (no pair nodes); spread out they need 11 internal nodes."""
    pos = spread(12, 6)
    check_edit(sphere_scene(np.repeat(pos[:1], 12, axis=0), groups=3), sphere_scene(pos, groups=3))


@pytest.mark.gpu
def test_repeated_edit_is_idempotent():
    check_edit(sphere_scene(spread(300, 7), groups=6, meshes=teapots()), sphere_scene(spread(300, 8), groups=6, meshes=teapots(40.0)),
               repeat=3)


# ---- GPU: interactive use, staging, rejections -------------------------------------------------------------------------------

@pytest.mark.gpu
def test_camera_move_after_a_stopped_render():
    """Arm, start an asynchronous render, stop it, move the camera, clear the stop and the framebuffer, render in full: the frame is
    the fresh scene's wherever the stop landed."""
    doc = scene_json("hdr")
    moved = copy.deepcopy(doc)
    moved["camera"]["transforms"][1]["degrees"] += 3
    W, H, spp, b, mp = GOLDEN_FRAMES["hdr"]
    a, bb = Loaded(doc, W, H, spp, b), Loaded(moved, W, H, spp, b)
    fresh = bb.upload(max_paths=mp)
    want = full(fresh)
    fresh.close()
    g = a.upload(max_paths=mp)
    try:
        g.enable_stop()
        g.clear()
        g.render_tile(0, 0, g.W, g.H, flags=crgpu.FLAG_ASYNC)
        g.request_stop()
        g.set_camera(bb.camera)
        g.clear_stop()
        g.clear()
        st = g.render_tile(0, 0, g.W, g.H)
        assert st["stopped"] is False
        assert g.read().tobytes() == want.tobytes()
    finally:
        g.close()
        a.free()
        bb.free()


STAGED = r"""
import sys
sys.path[:0] = [{pkg!r}, {tests!r}]
import test_gpu_scene_edit as T
doc = T.scene_json("hdr")
a, b = T.Loaded(doc, 320, 240, 2, 32), T.Loaded(T.edited(doc, T.STEP["hdr"]), 320, 240, 2, 32)
g = a.upload()
T.edit(g, b)
T.assert_same_as_fresh(g, b, T.ray_set(b.camera, n=70000))
g.close()
print("staged ok")
"""


@pytest.mark.gpu
def test_edited_frame_with_staged_top_nodes():
    """CRGPU_TRACE_STAGE=128 (read at prepare time) stages 32 top-level pairs; an edit rewrites that prefix."""
    scene_json("hdr")
    env = dict(os.environ, CRGPU_TRACE_STAGE="128")
    code = STAGED.format(pkg=os.path.join(ROOT, "c-ray_b200"), tests=os.path.join(ROOT, "tests"))
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0 and "staged ok" in r.stdout, r.stdout[-3000:]


@pytest.mark.gpu
def test_rejected_edits_leave_the_scene_unchanged():
    doc = scene_json("hdr")
    W, H, spp = SMALL
    a = Loaded(doc, W, H, spp, BOUNCES["hdr"])
    other = Loaded(doc, W // 2, H, spp, BOUNCES["hdr"])
    g = a.upload()
    L = crgpu.lib()
    try:
        before = full(g)
        inst = a.instances.copy()
        assert L.crgpu_scene_set_instances(g.handle, inst.ctypes.data, len(inst) - 1) == -3
        k = int(np.flatnonzero(inst["kind"] == 0)[0])
        bad = inst.copy()
        bad["kind"][k] = 1
        bad["A"][:, 3] += 1.0
        assert L.crgpu_scene_set_instances(g.handle, bad.ctypes.data, len(bad)) == -3
        bad = inst.copy()
        bad["object"][k] += 1
        assert L.crgpu_scene_set_instances(g.handle, bad.ctypes.data, len(bad)) == -3
        assert L.crgpu_scene_set_camera(g.handle, C.byref(other.camera)) == -3
        assert full(g).tobytes() == before.tobytes()
    finally:
        g.close()
        a.free()
        other.free()
