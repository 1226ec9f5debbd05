"""Changing the image size, sample count and bounce limit of a resident GPU scene between renders (crgpu_scene_set_render,
include/crgpu.h).

The target is exact: after the call the scene renders, traces and shades the bits of a fresh scene of the same content given those
settings (crscene_set_config, then crgpu_scene_create: crgpu_prepare + crgpu_scene_create_prepared), whatever edits came before or
after it, across views, framebuffer contents, an armed render with stop and snapshots, and the launch schedule.  Every frame is
compared as fp32 bytes.

CPU: argument checks and the Python wrapper.  GPU: everything else.
"""
import ctypes as C
import os
import threading
import time

import numpy as np
import pytest

import crgpu
import test_gpu_scene_edit as SE
from conftest import GOLDEN
from test_gpu_add_objects import grown
from test_gpu_views import _recoloured, cameras, grid, single, views

BAD_ARGUMENT, NOMEM = -3, -5
BASE = (96, 54, 4, 32)                       # W, H, spp, bounces every scene is uploaded at
# each setting alone (size up, size down, 1 x N, N x 1, not a multiple of the tile size; samples up and down; bounces 0, 1 and
# above the uploaded limit), all four together, and back to the uploaded settings, one call after the other on one scene
STEPS = [(160, 90, 4, 32), (48, 27, 4, 32), (1, 40, 4, 32), (40, 1, 4, 32), (37, 23, 4, 32), (96, 54, 7, 32), (96, 54, 2, 32),
         (96, 54, 4, 0), (96, 54, 4, 1), (96, 54, 4, 40), (120, 68, 3, 5), BASE]


# ---- CPU -----------------------------------------------------------------------------------------------------------------------

def test_null_scene_is_refused():
    L = crgpu.lib()
    cams = (crgpu.Camera * 2)()
    assert L.crgpu_scene_set_render(None, 8, 8, 1, 1, None, 1) == BAD_ARGUMENT
    assert L.crgpu_scene_set_render(None, 8, 8, 1, 1, cams, 2) == BAD_ARGUMENT


class _Recorder:
    """stands in for libcrgpu.so: records crgpu_scene_set_render's arguments, and has a view list of `views`"""

    def __init__(self, views):
        self.calls, self.views = [], views

    def crgpu_scene_view_count(self, handle, count):
        count._obj.value = self.views
        return 0

    def crgpu_scene_set_render(self, *args):
        self.calls.append(args)
        return 0


def test_wrapper_passes_its_arguments_as_declared(monkeypatch):
    L = crgpu.lib()
    P, U = C.c_void_p, C.c_uint32
    assert L.crgpu_scene_set_render.argtypes == [P, U, U, U, U, P, U]
    assert L.crgpu_scene_set_render.restype == C.c_int
    rec = _Recorder(3)
    monkeypatch.setattr(crgpu, "_lib", rec)
    g = crgpu.GpuScene.__new__(crgpu.GpuScene)
    g.handle = C.c_void_p(1234)
    cams = [crgpu.Camera(width=33, height=17, sensor_x=float(k)) for k in range(3)]
    g.set_render(33, 17, 9, 0, cams)
    h, w, hh, spp, b, arr, n = rec.calls[-1]
    assert (h.value, w, hh, spp, b, n) == (1234, 33, 17, 9, 0, 3)
    assert [bytes(c) for c in arr] == [bytes(c) for c in cams]
    assert (g.W, g.H, g.samples, g.bounces) == (33, 17, 9, 0)
    g.set_render(33, 17, 2, 5)                       # cameras kept: NULL and the scene's view count
    assert rec.calls[-1][1:] == (33, 17, 2, 5, None, 3)
    assert (g.W, g.H, g.samples, g.bounces) == (33, 17, 2, 5)
    g.handle = None


# ---- helpers ---------------------------------------------------------------------------------------------------------------------

class Src:
    """A flat scene uploaded fresh at any render settings: crscene_set_config, then crgpu_scene_create.  The bounce limit is set
    directly, so that 0 can be asked for (crscene_set_config keeps the value for 0)."""

    def __init__(self, flat, release):
        self.flat, self.release = flat, release

    @classmethod
    def golden(cls, name):
        L = crgpu.lib()
        flat = crgpu.FlatScene()
        assert L.crscene_load(C.byref(flat), os.fsencode(os.path.join(GOLDEN, name + ".crscene"))) == 0
        return cls(flat, lambda: L.crscene_free(C.byref(flat)))

    @classmethod
    def doc(cls, doc):
        x = SE.Loaded(doc, *BASE)
        return cls(x.flat, x.free)

    def camera(self, cfg):
        W, H, spp, b = cfg
        crgpu.lib().crscene_set_config(C.byref(self.flat), W, H, spp, 0)
        self.flat.prefs.bounces = b
        return crgpu.Camera.from_buffer_copy(self.flat.camera)

    def instances(self):
        import crscene
        return crscene.arrays(self.flat)["instances"]

    def upload(self, cfg=BASE, max_paths=None):
        cam = self.camera(cfg)
        g = crgpu.GpuScene.__new__(crgpu.GpuScene)
        g.handle = C.c_void_p()
        crgpu._check(crgpu.lib().crgpu_scene_create(C.byref(self.flat), 0, C.byref(g.handle)), "crgpu_scene_create")
        g.W, g.H, g.samples, g.bounces = cfg
        g.camera = cam
        if max_paths:
            g.set_max_paths(max_paths)
        return g

    def free(self):
        self.release()


def sources(name):
    return Src.doc(SE.scene_json(name)) if name == "hdr" else Src.golden(name)


def frame(g):
    g.clear()
    g.render_tile(0, 0, g.W, g.H)
    return g.read().copy()


def split(g, rects):
    """a tile set over two pass ranges, from a cleared framebuffer"""
    g.clear()
    k = g.samples // 2
    g.render_tiles(rects, 0, k)
    g.render_tiles(rects, k)
    return g.read().copy()


def traced(g):
    rec, _perm, misses, st = g.trace_rays(SE.ray_set(g.camera, 4096), count=1)
    return rec.tobytes(), misses, tuple(st[k] for k in ("node_pairs", "tri_tests", "sphere_tests", "inst_visits"))


def assert_same(g, fresh, what):
    assert frame(g).tobytes() == frame(fresh).tobytes(), f"{what}: frame"
    assert traced(g) == traced(fresh), f"{what}: ray records or P/T/S/I"


def set_render(g, src, cfg):
    """g.set_render to cfg with src's camera at cfg's size"""
    g.camera = src.camera(cfg)
    g.set_render(*cfg, [g.camera])


# ---- GPU: the settings -----------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", ["hdr", "g_nodes", "g_f4"])
def test_each_setting_renders_as_the_fresh_scene(name):
    src = sources(name)
    g = src.upload()
    try:
        for cfg in STEPS:
            set_render(g, src, cfg)
            fresh = src.upload(cfg)
            try:
                assert frame(g).tobytes() == frame(fresh).tobytes(), cfg
                rects = grid(g.W, g.H, 23, 17)
                assert split(g, rects).tobytes() == split(fresh, rects).tobytes(), cfg
            finally:
                fresh.close()
        d, w, h = C.c_int(), C.c_int(), C.c_int()
        crgpu._check(crgpu.lib().crgpu_scene_info(g.handle, C.byref(d), C.byref(w), C.byref(h)), "crgpu_scene_info")
        assert (w.value, h.value) == BASE[:2]
    finally:
        g.close()
        src.free()


@pytest.mark.gpu
def test_zero_bounces_is_black():
    src = sources("hdr")
    g = src.upload()
    try:
        set_render(g, src, (96, 54, 4, 0))
        assert not frame(g).any()
    finally:
        g.close()
        src.free()


# ---- GPU: composition with the other edits -------------------------------------------------------------------------------------

NEW = (120, 68, 3, 9)


def _edits(doc):
    """the unedited scene, the moved one, every source to free, and name -> (edit(g, cfg), the fresh reference at cfg)"""
    moved = Src.doc(SE.edited(doc, SE.STEP["hdr"]))
    shaded = Src.doc(_recoloured(doc))
    bigger = Src.doc(grown("hdr", doc))
    a = Src.doc(doc)
    mi = moved.instances()
    mesh = int(mi["object"][int(np.nonzero(mi["kind"] == 1)[0][-1])])

    def on_a(fn):
        def ref(cfg):
            r = a.upload(cfg)
            fn(r, cfg)
            return r
        return ref

    def camera(g, cfg):
        g.camera = moved.camera(cfg)
        g.set_camera(g.camera)

    def instances(g, cfg):
        camera(g, cfg)
        g.set_instances(moved.instances())
    E = {"camera": (camera, on_a(camera)),
         "instances": (instances, moved.upload),
         "instance_list": (lambda g, cfg: g.set_instance_list(mi[:-1]), on_a(lambda g, cfg: g.set_instance_list(mi[:-1]))),
         "meshes": (lambda g, cfg: g.set_meshes(moved.flat, [mesh]), on_a(lambda g, cfg: g.set_meshes(moved.flat, [mesh]))),
         "shading": (lambda g, cfg: g.set_shading(shaded.flat), shaded.upload),
         "add_objects": (lambda g, cfg: g.add_objects(bigger.flat), bigger.upload)}
    return a, moved, [moved, shaded, bigger, a], E


@pytest.mark.gpu
@pytest.mark.parametrize("settings_first", [False, True])
@pytest.mark.parametrize("what", ["camera", "instances", "instance_list", "meshes", "shading", "add_objects"])
def test_settings_compose_with_every_edit(what, settings_first):
    """settings then the edit, or the edit then settings: the fresh scene of the edited content at the new settings"""
    doc = SE.scene_json("hdr")
    a, moved, srcs, E = _edits(doc)
    edit, ref = E[what]
    g = a.upload()
    try:
        if settings_first:
            set_render(g, a, NEW)
            edit(g, NEW)
        else:
            edit(g, BASE)
            g.camera = (moved if what in ("camera", "instances") else a).camera(NEW)
            g.set_render(*NEW, [g.camera])
        fresh = ref(NEW)
        try:
            assert_same(g, fresh, what)
        finally:
            fresh.close()
    finally:
        g.close()
        for s in srcs:
            s.free()


# ---- GPU: views ----------------------------------------------------------------------------------------------------------------

class _At:
    """what test_gpu_views.cameras reads of a scene: its size and camera"""

    def __init__(self, src, cfg):
        self.W, self.H = cfg[:2]
        self.camera = src.camera(cfg)


@pytest.mark.gpu
def test_views_after_a_size_change():
    src = sources("hdr")
    g = src.upload()
    new = (160, 90, 4, 12)
    h = src.upload(new)
    try:
        g.set_views(cameras("hdr", _At(src, BASE), 4))
        g.render_views([(0, 0, g.W, g.H)])
        cams = cameras("hdr", _At(src, new), 4)
        g.set_render(*new, cams)
        assert g.view_count() == 4
        assert all(v.shape == (new[1], new[0], 3) and not v.any() for v in views(g))
        rects = grid(g.W, g.H)
        g.render_views(rects)
        for v in range(4):
            assert g.view_read(v).tobytes() == single(h, cams[v], rects)[0].tobytes(), v
        more = cameras("hdr", _At(src, new), 6)          # the view list still grows and shrinks at the new size
        g.set_views(more)
        got = views(g)
        g.render_views(rects, first=4)
        for v in (4, 5):
            assert g.view_read(v).tobytes() == single(h, more[v], rects)[0].tobytes(), v
        assert [x.tobytes() for x in views(g)[:4]] == [x.tobytes() for x in got[:4]]
    finally:
        g.close()
        h.close()
        src.free()


@pytest.mark.gpu
def test_same_size_keeps_every_view_and_camera():
    src = sources("hdr")
    g = src.upload()
    new = (BASE[0], BASE[1], 6, 7)
    h = src.upload(new)
    try:
        cams = cameras("hdr", _At(src, BASE), 3)
        g.set_views(cams)
        g.render_views([(0, 0, g.W, g.H)], pass_count=2)
        before = views(g)
        ptr = g.device_ptr()
        g.set_render(*new)                           # cameras kept
        assert [x.tobytes() for x in views(g)] == [x.tobytes() for x in before]
        assert g.device_ptr() == ptr
        g.render_views([(0, 0, g.W, g.H)], pass_begin=2)
        for v in range(3):                           # passes [2, 6) added to the kept contents, under the kept camera
            h.set_camera(cams[v])
            h.write(before[v])
            h.render_tiles([(0, 0, h.W, h.H)], 2)
            assert g.view_read(v).tobytes() == h.read().tobytes(), v
    finally:
        g.close()
        h.close()
        src.free()


# ---- GPU: framebuffer state ----------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_same_size_continues_on_the_old_contents():
    """set_camera, passes [0, 2), then samples and bounces change: passes [2, 5) add to the old contents as a fresh scene given them"""
    src = sources("hdr")
    g = src.upload()
    new = (BASE[0], BASE[1], 5, 6)
    h = src.upload(new)
    try:
        moved = cameras("hdr", _At(src, BASE), 2)[1]
        g.set_camera(moved)
        g.render_tile(0, 0, g.W, g.H, 0, 2)
        old = g.read().copy()
        g.set_render(*new)
        assert g.read().tobytes() == old.tobytes()
        g.render_tile(0, 0, g.W, g.H, 2)
        h.set_camera(moved)
        h.write(old)
        h.render_tile(0, 0, h.W, h.H, 2)
        assert g.read().tobytes() == h.read().tobytes()
    finally:
        g.close()
        h.close()
        src.free()


@pytest.mark.gpu
def test_new_size_reads_zeros_and_reports_the_new_size():
    src = sources("g_nodes")
    g = src.upload()
    try:
        g.set_views([g.camera] * 3)
        g.render_views([(0, 0, g.W, g.H)])
        g.srgb8()                                    # the lazy sRGB8 staging buffer exists at the old size
        for cfg in ((200, 150, 2, 4), (17, 9, 2, 4)):
            cam = src.camera(cfg)
            g.set_render(*cfg, [cam] * 3)
            W, H = cfg[:2]
            assert all(v.shape == (H, W, 3) and not v.any() for v in views(g))
            assert g.device_ptr()[1] == W * H * 3 * 4
            d, w, h = C.c_int(), C.c_int(), C.c_int()
            crgpu._check(crgpu.lib().crgpu_scene_info(g.handle, C.byref(d), C.byref(w), C.byref(h)), "crgpu_scene_info")
            assert (w.value, h.value) == (W, H)
            assert g.srgb8().shape == (H, W, 3) and not g.srgb8().any()
            assert not g.view_srgb8(2).any()
            rc = crgpu.lib().crgpu_render_tile(g.handle, 0, 0, W + 1, H, 0, 1, 0, None)
            assert rc == BAD_ARGUMENT
    finally:
        g.close()
        src.free()


# ---- GPU: armed scene ------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_stop_and_resume_after_a_size_change():
    src = sources("hdr")
    new = (240, 135, 32, 32)
    g, h = src.upload(), src.upload(new)
    try:
        npix = new[0] * new[1]
        g.enable_stop()
        g.render_tile(0, 0, g.W, g.H)
        set_render(g, src, new)
        for s in (g, h):
            s.set_max_paths(npix * 2)
        want = frame(h)
        done = threading.Event()

        def stopper():                               # progress still shows the earlier call's passes until this call is in flight
            while not done.is_set():
                if g.progress()[1] and g.progress()[0] > 0:
                    g.request_stop()
                    return
                time.sleep(0.0005)
        th = threading.Thread(target=stopper)
        th.start()
        try:
            st = g.render_tile(0, 0, g.W, g.H)
        finally:
            done.set()
            th.join()
        committed = g.progress()[0]
        assert st["stopped"] and 0 < committed < g.samples, (st, committed)
        h.clear()
        h.render_tile(0, 0, h.W, h.H, 0, committed)
        assert g.read().tobytes() == h.read().tobytes()
        g.clear_stop()
        st = g.render_tile(0, 0, g.W, g.H, committed)
        assert not st["stopped"] and g.progress() == (g.samples, False)
        assert g.read().tobytes() == want.tobytes()
    finally:
        g.close()
        h.close()
        src.free()


@pytest.mark.gpu
def test_snapshots_across_a_size_change():
    """An image staged at the old size is dropped; a request pending across the change is served at the new size, as the fresh
    scene's sRGB8 image of the same passes."""
    src = sources("hdr")
    new = (160, 90, 8, 32)
    g, h = src.upload(), src.upload(new)
    try:
        g.enable_stop()
        g.request_snapshot()
        g.render_tile(0, 0, g.W, g.H)                # stages the snapshot at the old size
        before = g.progress()
        set_render(g, src, new)
        assert g.progress() == before                # progress untouched
        img, done = g.take_snapshot()                # nothing staged, no call in flight: the (zeroed) framebuffer
        assert img.shape == (new[1], new[0], 3) and not img.any() and done == before[0]

        g.request_snapshot()                         # pending across a second size change
        new = (200, 120, 8, 32)
        h.close()
        h = src.upload(new)
        set_render(g, src, new)
        for s in (g, h):
            s.set_max_paths(new[0] * new[1] * 2)
        g.render_tile(0, 0, g.W, g.H)
        img, done = g.take_snapshot()
        assert img.shape == (new[1], new[0], 3) and 0 < done <= g.samples
        h.clear()
        h.render_tile(0, 0, h.W, h.H, 0, done)
        assert img.tobytes() == h.view_srgb8(0).tobytes()
    finally:
        g.close()
        h.close()
        src.free()


# ---- GPU: test entry points and launch schedule ----------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", ["hdr", "g_nodes"])
def test_entry_points_at_the_new_settings(name):
    src = sources(name)
    new = (150, 70, 5, 3)
    g, h = src.upload(), src.upload(new)
    try:
        set_render(g, src, new)
        rng = np.random.default_rng(3)
        xyp = np.stack([rng.integers(0, new[0], 512), rng.integers(0, new[1], 512), rng.integers(0, new[2], 512)], 1)
        assert g.trace_kat(xyp).tobytes() == h.trace_kat(xyp).tobytes()
        assert traced(g) == traced(h)
        rays = SE.ray_set(g.camera, 2048)
        st = np.zeros(len(rays), crgpu.PATH_STATE_DTYPE)
        st["o"], st["d"], st["weight"] = rays[:, :3], rays[:, 3:], 1.0
        st["rng"] = rng.integers(0, 1 << 63, len(rays), dtype=np.uint64)
        for depth in range(new[3]):
            a, b = g.shade_rays(st, depth, new[3]), h.shade_rays(st, depth, new[3])
            assert a[2] == b[2], depth
            for f in ("rec", "alive", "dir_key", "next"):        # the compaction slot is taken in atomic order
                assert a[0][f].tobytes() == b[0][f].tobytes(), (depth, f)
    finally:
        g.close()
        h.close()
        src.free()


@pytest.mark.gpu
@pytest.mark.parametrize("armed", [False, True])
def test_launch_count_is_the_fresh_scenes(armed):
    src = sources("g_nodes")
    new = (70, 44, 6, 5)
    g, h = src.upload(), src.upload(new)
    try:
        set_render(g, src, new)
        for s in (g, h):
            if armed:
                s.enable_stop()
        for mp in (1 << 20, 4 * new[0] * new[1], 1024, 5000):
            got = []
            for s in (g, h):
                s.set_max_paths(mp)
                s.get_stats()
                s.render_tiles(grid(s.W, s.H), flags=crgpu.FLAG_ASYNC)
                got.append(s.get_stats())
            assert got[0]["kernel_launches"] == got[1]["kernel_launches"], mp
            assert got[0]["paths"] == got[1]["paths"] == new[0] * new[1] * new[2]
    finally:
        g.close()
        h.close()
        src.free()


# ---- GPU: refusals ---------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_refusals_leave_the_scene_unchanged():
    src = sources("hdr")
    g, h = src.upload(), src.upload()
    try:
        L = crgpu.lib()
        cams = cameras("hdr", _At(src, BASE), 3)
        g.set_views(cams)
        h.set_views(cams)
        g.enable_stop()
        g.render_views([(0, 0, g.W, g.H)], pass_count=1)
        before, ptr, prog = views(g), g.device_ptr(), g.progress()
        W, H, spp, b = BASE
        new = cameras("hdr", _At(src, (64, 40, 4, 32)), 3)
        wrong = crgpu.Camera.from_buffer_copy(new[2])
        wrong.height = 41

        def arr(cs):
            return (crgpu.Camera * len(cs))(*cs)
        refusals = [(0, 40, 4, 32, arr(new), 3), (64, 0, 4, 32, arr(new), 3), (64, 40, 0, 32, arr(new), 3),
                    (64, 40, 4, 32, arr(new), 2), (64, 40, 4, 32, arr(new[:2]), 2), (64, 40, 4, 32, arr(new + new[:1]), 4),
                    (64, 40, 4, 32, arr(new[:2] + [wrong]), 3), (64, 40, 4, 32, None, 3), (W, H, spp, b, arr(new), 3),
                    (W, H, 0, b, None, 3), (W, H, spp, b, None, 2)]
        for args in refusals:
            assert L.crgpu_scene_set_render(g.handle, *args) == BAD_ARGUMENT, args[:4]
            assert [x.tobytes() for x in views(g)] == [x.tobytes() for x in before], args[:4]
            assert g.device_ptr() == ptr and g.progress() == prog and g.view_count() == 3
        # more framebuffer than the device holds: refused before anything changes
        huge = crgpu.Camera.from_buffer_copy(new[0])
        huge.width = huge.height = 1 << 20
        assert L.crgpu_scene_set_render(g.handle, 1 << 20, 1 << 20, 4, 32, arr([huge] * 3), 3) == NOMEM
        assert [x.tobytes() for x in views(g)] == [x.tobytes() for x in before]
        assert g.device_ptr() == ptr and g.progress() == prog
        for s in (g, h):                             # the cameras and settings are the ones before the calls
            for v in range(3):
                s.view_clear(v)
            s.render_views(grid(W, H))
        assert [x.tobytes() for x in views(g)] == [x.tobytes() for x in views(h)]
    finally:
        g.close()
        h.close()
        src.free()
