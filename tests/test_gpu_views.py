"""Rendering several views of a resident GPU scene in one call (crgpu_scene_set_views / crgpu_render_views, include/crgpu.h).

The target is exact: each view of a views call ends with the bits a single-camera render of its camera gives (crgpu_scene_set_camera,
then crgpu_render_tiles over the same tile set and passes) on a second upload of the scene, whatever the view count, the path budget,
the pieces, the pass split, the path order or a stop in between.  Cameras come from edited JSON (crscene.load_json_buf): moved and
turned, and one with another aperture and focal distance (depth of field).

CPU: argument checks of the new entry points.  GPU: everything else.
"""
import copy
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

import crgpu
import crscene
import oracle_lib as O
from conftest import GOLDEN, ROOT

DIGESTS = os.path.join(GOLDEN, "shade_frames.sha256.json")
REFDIR = os.path.join(ROOT, "oracle", "_ref")
# name -> (W, H, spp, bounces); 0 = the scene's own value.  The bundled scenes at their frame bounce limits.
SCENES = {"g_single": (0, 0, 0, 0), "g_nodes": (0, 0, 0, 0), "g_f4": (0, 0, 0, 0),
          "hdr": (240, 135, 4, 32), "venus": (240, 135, 4, 25), "refraction": (240, 135, 2, 512)}
# the configurations of tests/golden/shade_frames.sha256.json (W, H, spp, bounces, max paths in flight; 0 = the default)
GOLDEN_FRAMES = {"g_nodes": (0, 0, 0, 0, 0), "g_f4": (0, 0, 0, 0, 0), "hdr": (240, 135, 16, 32, 240 * 135 * 4),
                 "refraction": (240, 135, 8, 512, 0)}
STEP = {"hdr": 0.02, "venus": 20.0, "refraction": 20.0}
# one sphere: the cameras only depend on the camera object and the image size
MINI = {"ambientColor": {"down": [1, 1, 1], "up": [0.5, 0.7, 1.0]}, "meshes": [],
        "primitives": [{"type": "sphere", "radius": 1.0, "color": [0.7, 0.6, 0.5],
                        "instances": [{"transforms": [{"type": "translate", "Z": -5}]}]}]}


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


# ---- CPU -----------------------------------------------------------------------------------------------------------------------

def test_entry_points_reject_null_arguments():
    L = crgpu.lib()
    cams = (crgpu.Camera * 2)()
    n = C.c_uint32(0)
    rect = np.array([0, 0, 1, 1], dtype=np.int32)
    buf = np.zeros(16, dtype=np.float32)
    assert L.crgpu_scene_set_views(None, None, 1) == -3
    assert L.crgpu_scene_set_views(None, cams, 2) == -3
    assert L.crgpu_scene_view_count(None, C.byref(n)) == -3
    assert L.crgpu_render_views(None, 0, 1, rect.ctypes.data, 1, 0, 1, 0, None) == -3
    assert L.crgpu_view_clear(None, 0) == -3
    assert L.crgpu_view_read(None, 0, buf.ctypes.data) == -3
    assert L.crgpu_view_to_srgb8(None, 0, buf.ctypes.data) == -3


def test_no_scene_to_give_views_without_a_device():
    """Without a GPU no scene exists to give views to: creating one fails loudly (CRGPU_ERR_NO_DEVICE), never on the CPU."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    with pytest.raises(crgpu.CrgpuError):
        crgpu.GpuScene(os.path.join(GOLDEN, "g_single.crscene")).set_views([crgpu.Camera()])


# ---- helpers ---------------------------------------------------------------------------------------------------------------------

def scene_doc(name):
    path = os.path.join(GOLDEN, name + ".json")
    if not os.path.exists(path):
        path = os.path.join(REFDIR, "input", name + ".json")
    if not os.path.exists(path):
        pytest.skip(f"{name}.json not available")
    return json.load(open(path))


def scene_path(name, tmp):
    if name.startswith("g_"):
        return os.path.join(GOLDEN, name + ".crscene")
    p = O.bundled_scene(name, str(tmp))
    if not p:
        pytest.skip(f"{name} not available")
    return p


def upload(name, tmp, cfg=None, max_paths=None):
    W, H, spp, b = cfg or SCENES[name]
    path = scene_path(name, tmp)
    g = crgpu.GpuScene(path, W, H, spp, b, max_paths=max_paths)
    g.camera = scene_camera(path, W, H)
    return g


def scene_camera(path, W, H):
    """the camera a flat scene uploads with at W x H (0 = its own size)"""
    L = crgpu.lib()
    flat = crgpu.FlatScene()
    assert L.crscene_load(C.byref(flat), os.fsencode(path)) == 0
    try:
        L.crscene_set_config(C.byref(flat), W, H, 0, 0)
        return crgpu.Camera.from_buffer_copy(flat.camera)
    finally:
        L.crscene_free(C.byref(flat))


def cameras(name, g, n):
    """View 0: the scene's camera; view k >= 1: the JSON camera moved by k steps and turned by 2k degrees, view 1 also with
    another aperture and focal distance.  `name` is a scene's name or its JSON document."""
    doc = scene_doc(name) if isinstance(name, str) else name
    step = STEP.get(name, 0.05) if isinstance(name, str) else 0.05
    out = [crgpu.Camera.from_buffer_copy(g.camera)]
    for k in range(1, n):
        cam = copy.deepcopy(doc["camera"])
        turned = False
        for tr in cam.get("transforms", []):
            if tr["type"] == "translate":
                for a in ("x", "y", "z"):
                    if a in tr:
                        tr[a] = tr[a] + step * k * (1 if a != "y" else 0.5)
            elif tr["type"].startswith("rotate"):
                tr["degrees"] = tr.get("degrees", 0) + 2 * k
                turned = True
        if not turned:
            cam.setdefault("transforms", []).append({"type": "rotateY", "degrees": 2 * k})
        if k == 1:
            cam["fstops"] = 2.0
            cam["focalDistance"] = 1.5 * cam.get("focalDistance", 1.0)
        d = {"renderer": dict(doc["renderer"], width=g.W, height=g.H), "camera": cam, "scene": MINI}
        flat = crscene.load_json_buf(json.dumps(d))
        try:
            crgpu.lib().crscene_set_config(C.byref(flat), g.W, g.H, 0, 0)
            out.append(crgpu.Camera.from_buffer_copy(flat.camera))
        finally:
            crscene.free(flat)
    return out


def single(h, cam, rects, pass_begin=0, pass_count=None, flags=0):
    """a single-camera render of `cam` on the second upload h, from a cleared framebuffer"""
    h.set_camera(cam)
    h.clear()
    st = h.render_tiles(rects, pass_begin, pass_count, flags)
    return h.read().copy(), st


def views(g):
    return [g.view_read(v).copy() for v in range(g.view_count())]


def grid(W, H, tw=37, th=29):
    """a tile list with edge tiles: pixel counts that are not multiples of the pass-group pixel block, tiles not aligned to 8x4"""
    return [(x, y, min(x + tw, W), min(y + th, H)) for y in range(0, H, th) for x in range(0, W, tw)]


COUNTERS = ("node_pairs", "tri_tests", "sphere_tests", "inst_visits")


# ---- GPU -------------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SCENES))
def test_each_view_is_its_single_render(name, tmp_path):
    """V = 1, 2, 7, 33 views: each view's framebuffer bytes are a single-camera render's, and stats.paths, rays and (FLAG_COUNT)
    P/T/S/I are the sums of the single renders."""
    g, h = upload(name, tmp_path), upload(name, tmp_path)
    try:
        cams = cameras(name, g, 33)
        full = [(0, 0, g.W, g.H)]
        ref = {}
        for v, cam in enumerate(cams):
            img, st = single(h, cam, full)
            _, stc = single(h, cam, full, 0, 1, crgpu.FLAG_COUNT)
            ref[v] = (img, st, stc)
        for V in (1, 2, 7, 33):
            g.set_views(cams[:V])
            assert g.view_count() == V
            for v in range(V):
                g.view_clear(v)
            st = g.render_views(full)
            for v in range(V):
                assert g.view_read(v).tobytes() == ref[v][0].tobytes(), (V, v)
            assert st["paths"] == V * g.W * g.H * g.samples == sum(ref[v][1]["paths"] for v in range(V))
            assert st["rays"] == sum(ref[v][1]["rays"] for v in range(V)), V
            for v in range(V):
                g.view_clear(v)
            stc = g.render_views(full, pass_count=1, flags=crgpu.FLAG_COUNT)
            for k in ("paths", "rays") + COUNTERS:
                assert stc[k] == sum(ref[v][2][k] for v in range(V)), (V, k)
        h.write(g.view_read(6))                      # the sRGB8 of a view is crgpu_framebuffer_to_srgb8's of the same floats
        assert g.view_srgb8(6).tobytes() == h.srgb8().tobytes()
    finally:
        g.close()
        h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GOLDEN_FRAMES))
def test_scene_camera_gives_the_committed_frames(name, tmp_path):
    """The scene's own camera rendered as view 1 of three through render_views gives the committed digest at its configuration."""
    W, H, spp, b, mp = GOLDEN_FRAMES[name]
    g = upload(name, tmp_path, (W, H, spp, b), max_paths=mp or None)
    try:
        cams = cameras(name, g, 3)
        g.set_views([cams[1], cams[0], cams[2]])
        g.render_views([(0, 0, g.W, g.H)])
        want = json.load(open(DIGESTS))[name]
        assert digest(g.view_read(1)) == want
        assert digest(g.view_read(0)) != want
    finally:
        g.close()


@pytest.mark.gpu
def test_a_subset_of_views_leaves_the_others(tmp_path):
    """Passes [0, 2) in all 7 views, then passes [2, spp) in views [2, 5): every other view keeps its bytes (view 0 included), and
    views 2..4 are the single renders of all passes."""
    g, h = upload("hdr", tmp_path, (240, 135, 6, 32)), upload("hdr", tmp_path, (240, 135, 6, 32))
    try:
        cams = cameras("hdr", g, 7)
        g.set_views(cams)
        rects = grid(g.W, g.H)
        g.render_views(rects, pass_count=2)
        before = views(g)
        g.render_views(rects, first=2, count=3, pass_begin=2)
        after = views(g)
        for v in (0, 1, 5, 6):
            assert after[v].tobytes() == before[v].tobytes(), v
        for v in (2, 3, 4):
            assert after[v].tobytes() == single(h, cams[v], rects)[0].tobytes(), v
    finally:
        g.close()
        h.close()


@pytest.mark.gpu
def test_budgets_pieces_and_pass_splits_do_not_change_the_views(tmp_path):
    """One unsplit call against: several views per piece, one view per piece, views cut into pieces, and passes [0, k) + [k, spp)."""
    g = upload("hdr", tmp_path, (240, 135, 6, 32))
    try:
        cams = cameras("hdr", g, 7)
        g.set_views(cams)
        rects = grid(g.W, g.H)
        npix = g.W * g.H

        def run(max_paths, split=None):
            g.set_max_paths(max_paths)
            for v in range(7):
                g.view_clear(v)
            if split is None:
                g.render_views(rects)
            else:
                g.render_views(rects, pass_count=split)
                g.render_views(rects, pass_begin=split)
            return [digest(x) for x in views(g)]

        want = run(7 * npix * g.samples)
        assert run(4 * npix) == want                 # two pieces, of 4 and 3 views, one pass per batch
        assert run(npix) == want                     # one view per piece
        assert run(5000) == want                     # views cut inside, pieces across view boundaries
        assert run(7 * npix * g.samples, 2) == want
        assert run(5000, 5) == want
    finally:
        g.close()


_VIEWS_CODE = r"""
import hashlib, json, sys
sys.path[:0] = sys.argv[1:3]
import numpy as np, crgpu
def h(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
out = {}
for name, path, W, H, spp, b, cams in json.loads(sys.argv[3]):
    g = crgpu.GpuScene(path, W, H, spp, b)
    W, H, spp = g.W, g.H, g.samples
    g.set_views([crgpu.Camera.from_buffer_copy(bytes.fromhex(c)) for c in cams])
    V = len(cams)
    def dig(tag):
        out[name + "/" + tag] = [h(g.view_read(v)) for v in range(V)]
        for v in range(V):
            g.view_clear(v)
    g.render_views([(0, 0, W, H)])
    dig("frame")
    rects = [(x, y, min(x + 37, W), min(y + 29, H)) for y in range(0, H, 29) for x in range(0, W, 37)]
    g.render_views(rects, first=1)
    dig("tiles")
    g.set_max_paths(5000)
    g.render_views(rects, pass_count=min(5, spp))
    dig("pieces")
    g.set_max_paths(max(1024, W * H * 3))
    g.enable_stop()
    g.request_stop()
    st = g.render_views(rects)
    assert st["stopped"] and g.progress() == (0, False)
    g.clear_stop()
    g.render_views(rects, pass_count=spp // 2)
    g.render_views(rects, pass_begin=spp // 2)
    assert g.progress() == (spp, False)
    dig("resumed")
    g.close()
print("FRAMES " + json.dumps(out))
"""


def _view_frames(env, jobs):
    e = {k: v for k, v in os.environ.items() if not k.startswith("CRGPU_")}
    e.update(env)
    r = subprocess.run([sys.executable, "-c", _VIEWS_CODE, os.path.join(ROOT, "c-ray_b200"), os.path.join(ROOT, "tests"), json.dumps(jobs)],
                       env=e, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("FRAMES ")]
    assert r.returncode == 0 and lines, r.stdout[-2000:]
    return json.loads(lines[-1][7:])


@pytest.mark.gpu
def test_every_path_order_renders_the_default_views(tmp_path):
    """Every CRGPU_PATH_ORDER gives the default order's views: whole frames, a tile list with edge tiles, pieces across views, and
    an armed call stopped and resumed, on g_nodes and on hdr at 240x135, 8 spp."""
    jobs = []
    for name, cfg in (("g_nodes", (0, 0, 0, 0)), ("hdr", (240, 135, 8, 32))):
        g = upload(name, tmp_path, cfg)
        cams = [bytes(c).hex() for c in cameras(name, g, 5)]
        jobs.append([name, scene_path(name, tmp_path), *cfg, cams])
        g.close()
    base = _view_frames({}, jobs)
    assert len(base) == 4 * len(jobs)
    bad = []
    for order in range(8):
        got = _view_frames({"CRGPU_PATH_ORDER": str(order)}, jobs)
        bad += [(order, k) for k in base if got[k] != base[k]]
    assert not bad, bad


@pytest.mark.gpu
def test_stop_from_another_thread_and_resume(tmp_path):
    """A stop requested while a views call renders ends it at a pass boundary: every view then holds passes [0, committed) exactly,
    and resuming at the committed pass gives the unarmed call's bits."""
    cfg = (240, 135, 32, 32)
    g, h = upload("hdr", tmp_path, cfg), upload("hdr", tmp_path, cfg)
    try:
        cams = cameras("hdr", g, 7)
        rects = [(0, 0, g.W, g.H)]
        npix = g.W * g.H
        h.set_views(cams)
        h.set_max_paths(7 * npix * 2)
        h.render_views(rects)
        want = views(h)
        g.set_views(cams)
        g.set_max_paths(7 * npix * 2)                # 16 pass batches over the two wave sets
        g.enable_stop()
        done = threading.Event()

        def stopper():
            while not done.is_set():
                if g.progress()[0] > 0:
                    g.request_stop()
                    return
                time.sleep(0.0005)
        th = threading.Thread(target=stopper)
        th.start()
        try:
            st = g.render_views(rects)
        finally:
            done.set()
            th.join()
        committed = g.progress()[0]
        assert st["stopped"] and 0 < committed < g.samples, (st, committed)
        assert st["paths"] == 7 * npix * committed
        part = views(g)
        for v in range(7):
            assert part[v].tobytes() == single(h, cams[v], rects, 0, committed)[0].tobytes(), v
        g.clear_stop()
        st = g.render_views(rects, pass_begin=committed)
        assert not st["stopped"] and g.progress() == (g.samples, False)
        assert [x.tobytes() for x in views(g)] == [x.tobytes() for x in want]
    finally:
        g.close()
        h.close()


@pytest.mark.gpu
def test_snapshot_stays_pending_during_a_views_call(tmp_path):
    g = upload("hdr", tmp_path, (240, 135, 32, 32))
    try:
        cams = cameras("hdr", g, 7)
        g.set_views(cams)
        g.set_max_paths(7 * g.W * g.H * 2)
        g.enable_stop()
        g.render_views([(0, 0, g.W, g.H)], flags=crgpu.FLAG_ASYNC)
        g.request_snapshot()
        polls = 0
        while g.progress()[1]:
            r = g.take_snapshot()
            if g.progress()[1]:           # still in flight after the take: it must have been pending
                assert r is None
                polls += 1
        assert polls > 0
        g.get_stats()
        img, done = g.take_snapshot()
        assert done == g.samples and img.tobytes() == g.view_srgb8(0).tobytes()
    finally:
        g.close()


@pytest.mark.gpu
@pytest.mark.skipif(any(k.startswith("CRGPU_") for k in os.environ), reason="the schedule is that of the default knobs")
@pytest.mark.parametrize("armed", [False, True])
def test_launch_count_follows_the_schedule(armed):
    """The launch schedule of tests/test_gpu_launch_schedule.py, taken over the call's (view, pixel) set: pieces are ranges of the
    view-major numbering."""
    import test_gpu_launch_schedule as LS
    W, H, SPP, B = LS.W, LS.H, LS.SPP, LS.BOUNCES
    g = crgpu.GpuScene(os.path.join(GOLDEN, "g_legacy.crscene"), W, H, SPP, B, force_bounces=B)
    try:
        V = 3
        cams = [scene_camera(os.path.join(GOLDEN, "g_legacy.crscene"), W, H)] * V
        g.set_views(cams)
        if armed:
            g.enable_stop()
        for mp in (1 << 20, 4 * W * H, 1024, 5000):
            total = V * W * H
            parts = [min(mp, total - p) for p in range(0, total, mp)]
            if not armed:
                want = sum(LS.batches(p, mp, SPP, True) * LS.per_batch(B, False, False) for p in parts)
            elif len(parts) == 1:
                want = LS.batches(parts[0], mp, SPP, True) * (LS.per_batch(B, False, True) + 1) + 2
            else:
                step = max(1, mp // max(parts))
                want = 2
                for pb in range(0, SPP, step):
                    n = min(step, SPP - pb)
                    want += sum(LS.batches(p, mp, n, True) * LS.per_batch(B, False, True) for p in parts) + 1
            g.set_max_paths(mp)
            g.get_stats()
            g.render_views([(0, 0, W, H)], flags=crgpu.FLAG_ASYNC)
            st = g.get_stats()
            assert st["kernel_launches"] == want, (mp, st)
            assert st["paths"] == total * SPP
    finally:
        g.close()


def _recoloured(doc):
    """the first material colour given as three numbers, changed (the material count stays)"""
    d = copy.deepcopy(doc)

    def walk(o):
        if isinstance(o, dict):
            for k, v in o.items():
                if k == "color" and isinstance(v, list) and len(v) == 3:
                    o[k] = [0.9, 0.25, 0.1]
                    return True
                if k == "color" and isinstance(v, dict) and set(v) >= {"r", "g", "b"}:
                    v.update(r=0.9, g=0.25, b=0.1)
                    return True
                if walk(v):
                    return True
        elif isinstance(o, list):
            return any(walk(x) for x in o)
        return False
    assert walk(d["scene"])
    return d


@pytest.mark.gpu
def test_edits_compose_with_views(tmp_path):
    """After set_views, each of set_instances, set_instance_list, set_meshes and set_shading leaves every view equal to a single
    render of the same edit on the second upload."""
    import test_gpu_scene_edit as SE
    doc = SE.scene_json("hdr")
    W, H, spp, b = 240, 135, 4, 32
    a, moved = SE.Loaded(doc, W, H, spp, b), SE.Loaded(SE.edited(doc, STEP["hdr"]), W, H, spp, b)
    shaded = SE.Loaded(_recoloured(doc), W, H, spp, b)
    g, h = a.upload(), a.upload()
    g.camera = a.camera
    try:
        cams = cameras("hdr", g, 5)
        g.set_views(cams)
        rects = grid(W, H)
        mesh = int(np.nonzero(moved.instances["kind"] == 1)[0][-1])
        mesh = int(moved.instances["object"][mesh])
        steps = [("instances", lambda s: s.set_instances(moved.instances)),
                 ("instance_list", lambda s: s.set_instance_list(moved.instances[:-1])),
                 ("meshes", lambda s: s.set_meshes(moved.flat, [mesh])),
                 ("shading", lambda s: s.set_shading(shaded.flat))]
        for what, fn in steps:
            fn(g)
            fn(h)
            assert g.view_count() == 5
            for v in range(5):
                g.view_clear(v)
            g.render_views(rects)
            for v in range(5):
                assert g.view_read(v).tobytes() == single(h, cams[v], rects)[0].tobytes(), (what, v)
    finally:
        g.close()
        h.close()
        a.free()
        moved.free()
        shaded.free()


@pytest.mark.gpu
def test_set_camera_moves_view_zero_only(tmp_path):
    g, h = upload("hdr", tmp_path), upload("hdr", tmp_path)
    try:
        cams = cameras("hdr", g, 5)
        g.set_views(cams[:4])
        rects = [(0, 0, g.W, g.H)]
        g.render_views(rects)
        before = views(g)
        g.set_camera(cams[4])
        assert g.view_count() == 4
        assert [x.tobytes() for x in views(g)] == [x.tobytes() for x in before]      # an edit never touches the pixels
        for v in range(4):
            g.view_clear(v)
        g.render_views(rects)
        after = views(g)
        assert after[0].tobytes() == single(h, cams[4], rects)[0].tobytes()
        for v in (1, 2, 3):
            assert after[v].tobytes() == before[v].tobytes(), v
    finally:
        g.close()
        h.close()


@pytest.mark.gpu
def test_shrinking_and_growing_keep_surviving_views(tmp_path):
    g = upload("hdr", tmp_path)
    try:
        cams = cameras("hdr", g, 7)
        g.set_views(cams[:5])
        g.render_views([(0, 0, g.W, g.H)])
        before = views(g)
        assert all(x.any() for x in before)
        g.set_views(cams[:3])
        assert g.view_count() == 3
        assert [x.tobytes() for x in views(g)] == [x.tobytes() for x in before[:3]]
        g.set_views(cams[:7])                        # grows past the block: views 0..2 move, 3..6 start zeroed
        got = views(g)
        assert [x.tobytes() for x in got[:3]] == [x.tobytes() for x in before[:3]]
        assert all(not x.any() for x in got[3:])
        g.set_views(cams[:2])
        g.set_views(cams[:4])                        # regrows inside the block: views 2, 3 start zeroed again
        got = views(g)
        assert [x.tobytes() for x in got[:2]] == [x.tobytes() for x in before[:2]]
        assert all(not x.any() for x in got[2:])
    finally:
        g.close()


@pytest.mark.gpu
def test_refusals_leave_every_view_unchanged(tmp_path):
    g = upload("hdr", tmp_path)
    try:
        L = crgpu.lib()
        cams = cameras("hdr", g, 4)
        g.set_views(cams)
        g.render_views([(0, 0, g.W, g.H)], pass_count=1)
        before = views(g)
        wrong = crgpu.Camera.from_buffer_copy(cams[2])
        wrong.width = g.W + 1
        arr = (crgpu.Camera * 4)(cams[0], cams[1], wrong, cams[3])
        assert L.crgpu_scene_set_views(g.handle, arr, 4) == -3
        assert L.crgpu_scene_set_views(g.handle, arr, 0) == -3
        big = (crgpu.Camera * 1)(cams[0])
        assert L.crgpu_scene_set_views(g.handle, big, 65537) == -3
        rect = np.array([0, 0, g.W, g.H], dtype=np.int32)
        for first, count in ((4, 1), (2, 3), (0, 0), (0, 5), (0xffffffff, 2)):
            assert L.crgpu_render_views(g.handle, first, count, rect.ctypes.data, 1, 0, 1, 0, None) == -3, (first, count)
        outside = np.array([0, 0, g.W + 1, g.H, 5, 5, 4, 9], dtype=np.int32)
        assert L.crgpu_render_views(g.handle, 0, 4, outside.ctypes.data, 1, 0, 1, 0, None) == -3
        assert L.crgpu_render_views(g.handle, 0, 4, outside[4:].ctypes.data, 1, 0, 1, 0, None) == -3
        assert L.crgpu_render_views(g.handle, 0, 4, rect.ctypes.data, 0, 0, 1, 0, None) == -3
        assert L.crgpu_view_read(g.handle, 4, before[0].ctypes.data) == -3
        assert L.crgpu_view_clear(g.handle, 4) == -3
        assert g.view_count() == 4
        assert [x.tobytes() for x in views(g)] == [x.tobytes() for x in before]
    finally:
        g.close()
