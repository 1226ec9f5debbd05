"""ctypes binding of libcrgpu.so (include/crgpu.h) — the same C ABI a cgo/JNI/C host would bind.

Python is plumbing only (tests, bench, multi-GPU launch); nothing here computes pixels.  The library
has no CPU fallback: if it is missing or no CUDA device is present, every call raises.
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libcrgpu.so")

FLAG_COUNT = 0x1
FLAG_TIME_KERNELS = 0x2
FLAG_ASYNC = 0x4
STOPPED = 1          # CRGPU_STOPPED: an armed render call ended at a pass boundary because a stop was requested
PENDING = 2          # CRGPU_PENDING: the snapshot asked for has not been staged yet


class Prefs(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("image_width", "image_height", "sample_count", "bounces",
                                          "tile_width", "tile_height", "tile_order", "thread_count")]


class Camera(C.Structure):
    _fields_ = [("sensor_x", C.c_float), ("sensor_y", C.c_float), ("aperture", C.c_float),
                ("focal_distance", C.c_float), ("forward", C.c_float * 3), ("right", C.c_float * 3),
                ("up", C.c_float * 3), ("width", C.c_int32), ("height", C.c_int32), ("pad", C.c_uint32),
                ("A", C.c_float * 16)]


class FlatScene(C.Structure):
    """struct crs_scene (include/crscene.h)"""
    _fields_ = [("prefs", Prefs), ("camera", Camera), ("background", C.c_int32), ("top_bvh", C.c_uint32),
                ("instance_count", C.c_uint32), ("sphere_count", C.c_uint32), ("mesh_count", C.c_uint32),
                ("material_count", C.c_uint32), ("node_count", C.c_uint32), ("texture_count", C.c_uint32),
                ("bvh_count", C.c_uint32), ("bvh_node_count", C.c_uint32), ("prim_index_count", C.c_uint32),
                ("poly_count", C.c_uint32), ("vertex_count", C.c_uint32), ("normal_count", C.c_uint32),
                ("texcoord_count", C.c_uint32), ("texdata_bytes", C.c_uint64)] + \
               [(n, C.c_void_p) for n in ("instances", "spheres", "meshes", "materials", "nodes", "textures",
                                          "bvhs", "bvh_nodes", "prim_indices", "polys", "vertices", "normals",
                                          "texcoords", "texdata", "owner")]


class Stats(C.Structure):
    """struct crgpu_stats"""
    _fields_ = [(n, C.c_uint64) for n in ("paths", "rays", "node_pairs", "tri_tests", "sphere_tests",
                                          "inst_visits", "kernel_launches")] + \
               [(n, C.c_float) for n in ("trace_ms", "shade_ms", "total_ms", "pad")]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_ if n != "pad"}


class Adaptive(C.Structure):
    """struct crgpu_adaptive: the rule of an adaptive round (crgpu_adaptive_round)"""
    _fields_ = [("min_passes", C.c_uint32), ("round_passes", C.c_uint32), ("pass_end", C.c_uint32), ("threshold", C.c_float),
                ("floor", C.c_float)]


# struct crgpu_adaptive_record: a pixel's adaptive record (crgpu_adaptive_write / crgpu_adaptive_records); bit 31 of n is ADAPTIVE_DONE
ADAPT_RECORD_DTYPE = np.dtype([("n", "<u4"), ("mean", "<f4"), ("m2", "<f4"), ("err", "<f4")])
assert ADAPT_RECORD_DTYPE.itemsize == 16
ADAPTIVE_DONE = 0x80000000


class TraceOpts(C.Structure):
    """struct crgpu_trace_opts: the launch variant of the traversal kernel (crgpu_trace_rays)"""
    _fields_ = [(n, C.c_int32) for n in ("count", "minb", "defer", "refill", "burst", "inst_min")] + [("order", C.c_void_p)]


# struct crgpu_ray_record
RAY_RECORD_DTYPE = np.dtype([("t", "<f4"), ("u", "<f4"), ("v", "<f4"), ("inst", "<i4"), ("poly", "<i4"), ("key", "<u4"),
                             ("prim", "<u4"), ("pad", "<u4")])
assert RAY_RECORD_DTYPE.itemsize == 32
# the frame path's defaults (crg_trace_knobs_env); burst is 4 when leaves are deferred
TRACE_DEFAULTS = dict(count=0, minb=4, defer=0, refill=16, burst=3, inst_min=4)

# struct crgpu_path_state / crgpu_shade_result (crgpu_shade_rays); the path state is struct cro_path_state of the oracle
PATH_STATE_DTYPE = np.dtype([("o", "<f4", 3), ("d", "<f4", 3), ("weight", "<f4", 3), ("has_l", "<u4"), ("rng", "<u8"),
                             ("L", "<f4", 3), ("pad", "<u4")])
assert PATH_STATE_DTYPE.itemsize == 64
SHADE_RESULT_DTYPE = np.dtype([("rec", RAY_RECORD_DTYPE), ("alive", "<i4"), ("slot", "<u4"), ("dir_key", "<u4"), ("pad", "<u4"),
                               ("next", PATH_STATE_DTYPE)])
assert SHADE_RESULT_DTYPE.itemsize == 112
# the frame path's K3 defaults (crg_shade_knobs_env)
SHADE_DEFAULTS = dict(minb=2, split=1, prefetch=0, dirmode=0, complete_interpreter=0, tail=0, generic_only=0)
LIBM = ["sin", "cos", "tan", "log", "log10", "atan2", "acos", "asin", "pow", "pow5", "sincos_sin", "sincos_cos"]


class ShadeOpts(C.Structure):
    """struct crgpu_shade_opts"""
    _fields_ = [(n, C.c_int32) for n in ("minb", "split", "prefetch", "dirmode", "complete_interpreter", "tail", "depth", "max_depth",
                                         "generic_only")]

_lib = None


def lib():
    """Load libcrgpu.so; fail loudly when the CUDA extension has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing — build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(there is no CPU fallback for the hot path)")
        L = C.CDLL(LIB_PATH)
        P = C.c_void_p
        L.crgpu_last_error.restype = C.c_char_p
        L.crgpu_device_count.argtypes = [C.POINTER(C.c_int)]
        L.crgpu_scene_create.argtypes = [C.POINTER(FlatScene), C.c_int, C.POINTER(P)]
        L.crgpu_scene_destroy.argtypes = [P]
        L.crgpu_set_max_paths_in_flight.argtypes = [P, C.c_uint64]
        L.crgpu_render_tile.argtypes = [P] + [C.c_int] * 6 + [C.c_uint, C.POINTER(Stats)]
        L.crgpu_render_tiles.argtypes = [P, P, C.c_int, C.c_int, C.c_int, C.c_uint, C.POINTER(Stats)]
        L.crgpu_set_stream.argtypes = [P, P]
        L.crgpu_get_stats.argtypes = [P, C.POINTER(Stats)]
        L.crgpu_use_own_stream.argtypes = [P]
        L.crgpu_framebuffer_clear.argtypes = [P]
        L.crgpu_framebuffer_read.argtypes = [P, P] + [C.c_int] * 4
        L.crgpu_framebuffer_write.argtypes = [P, P] + [C.c_int] * 4
        L.crgpu_framebuffer_to_srgb8.argtypes = [P, P]
        L.crgpu_framebuffer_device_ptr.argtypes = [P, C.POINTER(P), C.POINTER(C.c_size_t)]
        L.crgpu_trace_kat.argtypes = [P, P, C.c_int, P]
        L.crgpu_trace_rays.argtypes = [P, P, C.c_uint32, C.POINTER(TraceOpts), P, P, C.POINTER(C.c_uint32), C.POINTER(Stats)]
        L.crgpu_shade_rays.argtypes = [P, P, C.c_uint32, C.POINTER(ShadeOpts), P, P, C.POINTER(C.c_uint32), P]
        L.crgpu_libm_eval.argtypes = [C.c_int, C.c_int, P, P, P, C.c_uint32]
        L.crgpu_path_order_map.argtypes = [C.c_int, C.c_uint32, C.c_uint32, P, P, P, C.c_uint32, C.c_uint32, P]
        L.crgpu_prepared_background.argtypes = [P, C.POINTER(C.c_uint32)]
        L.crgpu_scene_create_prepared.argtypes = [P, C.c_int, C.POINTER(P)]
        L.crgpu_scene_info.argtypes = [P, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.crgpu_device_trim.argtypes = [C.c_int]
        L.crgpu_stop_enable.argtypes = [P, C.c_int]
        L.crgpu_request_stop.argtypes = [P]
        L.crgpu_clear_stop.argtypes = [P]
        L.crgpu_progress.argtypes = [P, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.crgpu_scene_set_camera.argtypes = [P, C.POINTER(Camera)]
        L.crgpu_scene_set_instances.argtypes = [P, P, C.c_uint32]
        L.crscene_load.argtypes = [C.POINTER(FlatScene), C.c_char_p]
        L.crscene_free.argtypes = [C.POINTER(FlatScene)]
        L.crscene_set_config.argtypes = [C.POINTER(FlatScene)] + [C.c_int] * 4
        for f in ("crgpu_device_count", "crgpu_scene_create", "crgpu_scene_destroy", "crgpu_set_max_paths_in_flight",
                  "crgpu_render_tile", "crgpu_render_tiles", "crgpu_set_stream", "crgpu_use_own_stream", "crgpu_get_stats", "crgpu_framebuffer_clear", "crgpu_framebuffer_read", "crgpu_framebuffer_write",
                  "crgpu_framebuffer_to_srgb8", "crgpu_framebuffer_device_ptr", "crgpu_trace_kat", "crgpu_trace_rays", "crscene_load",
                  "crgpu_shade_rays", "crgpu_libm_eval", "crgpu_path_order_map", "crgpu_prepared_background",
                  "crgpu_scene_create_prepared", "crgpu_scene_info", "crgpu_device_trim",
                  "crgpu_stop_enable", "crgpu_request_stop", "crgpu_clear_stop", "crgpu_progress",

                  "crgpu_scene_set_camera", "crgpu_scene_set_instances", "crscene_set_config"):
            getattr(L, f).restype = C.c_int
        if hasattr(L, "crgpu_take_snapshot"):      # absent from libraries built before snapshots (tools/driver_check.py compares builds)
            L.crgpu_request_snapshot.argtypes = [P]
            L.crgpu_take_snapshot.argtypes = [P, P, C.POINTER(C.c_int)]
            L.crgpu_request_snapshot.restype = L.crgpu_take_snapshot.restype = C.c_int
        if hasattr(L, "crgpu_scene_set_meshes"):   # absent from libraries built before mesh edits
            L.crgpu_scene_set_meshes.argtypes = [P, C.POINTER(FlatScene), P, C.c_uint32]
            L.crgpu_scene_set_meshes.restype = C.c_int
        if hasattr(L, "crgpu_scene_set_instance_list"):   # absent from libraries built before instance-list edits
            L.crgpu_scene_set_instance_list.argtypes = [P, P, C.c_uint32]
            L.crgpu_scene_set_instance_list.restype = C.c_int
        if hasattr(L, "crgpu_scene_set_shading"):  # absent from libraries built before shading edits
            L.crgpu_scene_set_shading.argtypes = [P, C.POINTER(FlatScene)]
            L.crgpu_scene_shading.argtypes = [P, P, P, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_int)]
            L.crgpu_scene_set_shading.restype = L.crgpu_scene_shading.restype = C.c_int
        if hasattr(L, "crgpu_scene_add_objects"):  # absent from libraries built before object adds
            L.crgpu_scene_add_objects.argtypes = [P, C.POINTER(FlatScene)]
            L.crgpu_scene_add_objects.restype = C.c_int
        if hasattr(L, "crgpu_render_views"):      # absent from libraries built before views
            L.crgpu_scene_set_views.argtypes = [P, P, C.c_uint32]
            L.crgpu_scene_view_count.argtypes = [P, C.POINTER(C.c_uint32)]
            L.crgpu_render_views.argtypes = [P, C.c_uint32, C.c_uint32, P, C.c_int, C.c_int, C.c_int, C.c_uint, C.POINTER(Stats)]
            L.crgpu_view_clear.argtypes = [P, C.c_uint32]
            L.crgpu_view_read.argtypes = [P, C.c_uint32, P]
            L.crgpu_view_to_srgb8.argtypes = [P, C.c_uint32, P]
            for f in ("crgpu_scene_set_views", "crgpu_scene_view_count", "crgpu_render_views", "crgpu_view_clear", "crgpu_view_read",
                      "crgpu_view_to_srgb8"):
                getattr(L, f).restype = C.c_int
        if hasattr(L, "crgpu_scene_set_render"):  # absent from libraries built before render-settings edits
            L.crgpu_scene_set_render.argtypes = [P] + [C.c_uint32] * 4 + [P, C.c_uint32]
            L.crgpu_scene_set_render.restype = C.c_int
        if hasattr(L, "crgpu_adaptive_round"):    # absent from libraries built before adaptive rounds
            L.crgpu_adaptive_reset.argtypes = [P]
            L.crgpu_adaptive_round.argtypes = [P, P, C.c_int, C.POINTER(Adaptive), C.c_uint, C.POINTER(Stats), C.POINTER(C.c_uint32),
                                               C.POINTER(C.c_int), C.POINTER(C.c_int)]
            L.crgpu_adaptive_read.argtypes = [P, P, P]
            for f in ("crgpu_adaptive_reset", "crgpu_adaptive_round", "crgpu_adaptive_read"):
                getattr(L, f).restype = C.c_int
        if hasattr(L, "crgpu_adaptive_select"):   # absent from libraries built before the adaptive kernels' test entry points
            L.crgpu_accumulate_samples.argtypes = [P, P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, P, P]
            L.crgpu_adaptive_write.argtypes = [P, P]
            L.crgpu_adaptive_records.argtypes = [P, P]
            L.crgpu_adaptive_select.argtypes = [P, P, C.c_int, C.POINTER(Adaptive), P, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32),
                                                C.POINTER(C.c_uint32)]
            for f in ("crgpu_accumulate_samples", "crgpu_adaptive_write", "crgpu_adaptive_records", "crgpu_adaptive_select"):
                getattr(L, f).restype = C.c_int
        _lib = L
    return _lib


class CrgpuError(RuntimeError):
    pass


def _check(rc, what):
    if rc != 0:
        raise CrgpuError(f"{what} failed ({rc}): {lib().crgpu_last_error().decode(errors='replace')}")


def device_count():
    n = C.c_int(0)
    _check(lib().crgpu_device_count(C.byref(n)), "crgpu_device_count")
    return n.value


class GpuScene:
    """A scene resident on one GPU (crgpu_scene) plus its device framebuffer."""

    def __init__(self, crscene_path, width=0, height=0, samples=0, bounces=0, device=0, max_paths=None, force_bounces=None, prepared=None):
        L = lib()
        if prepared is not None:
            # a crgpu_prepared* owned by someone else (e.g. crhost.Renderer.prepared()): upload only
            self.handle = C.c_void_p()
            _check(L.crgpu_scene_create_prepared(C.c_void_p(prepared), device, C.byref(self.handle)), "crgpu_scene_create_prepared")
            d, w, h = C.c_int(), C.c_int(), C.c_int()
            _check(L.crgpu_scene_info(self.handle, C.byref(d), C.byref(w), C.byref(h)), "crgpu_scene_info")
            self.W, self.H, self.samples, self.bounces = w.value, h.value, samples, bounces
            if max_paths:
                _check(L.crgpu_set_max_paths_in_flight(self.handle, int(max_paths)), "crgpu_set_max_paths_in_flight")
            return
        if str(crscene_path).lower().endswith(".json"):
            # a c-ray JSON scene: parsed + BVH-built on the host by libcrloader.so (include/crloader.h)
            import crscene
            self.flat = crscene.load_json(crscene_path)
        else:
            self.flat = FlatScene()
            rc = L.crscene_load(C.byref(self.flat), os.fsencode(crscene_path))
            if rc != 0:
                raise CrgpuError(f"crscene_load({crscene_path}) failed: {rc}")
        L.crscene_set_config(C.byref(self.flat), width, height, samples, bounces)     # 0 = keep the scene's value
        if force_bounces is not None:
            self.flat.prefs.bounces = force_bounces                                       # (so that 0 itself can be requested)
        self.W, self.H = self.flat.prefs.image_width, self.flat.prefs.image_height
        self.samples, self.bounces = self.flat.prefs.sample_count, self.flat.prefs.bounces
        self.handle = C.c_void_p()
        try:
            _check(L.crgpu_scene_create(C.byref(self.flat), device, C.byref(self.handle)), "crgpu_scene_create")
        finally:
            L.crscene_free(C.byref(self.flat))
        if max_paths:
            _check(L.crgpu_set_max_paths_in_flight(self.handle, int(max_paths)), "crgpu_set_max_paths_in_flight")

    def render_tile(self, x0, y0, x1, y1, pass_begin=0, pass_count=None, flags=0):
        """Returns the call's stats (None with FLAG_ASYNC); on an armed scene the dict has "stopped": whether the call ended early."""
        st = Stats()
        if pass_count is None:
            pass_count = self.samples - pass_begin
        rc = lib().crgpu_render_tile(self.handle, x0, y0, x1, y1, pass_begin, pass_count, flags, C.byref(st))
        return self._render_result(rc, flags, st, "crgpu_render_tile")

    def render_tiles(self, rects, pass_begin=0, pass_count=None, flags=0):
        """Render a union of tiles [(x0, y0, x1, y1), ...] as ONE wavefront (the result as for render_tile)."""
        st = Stats()
        if pass_count is None:
            pass_count = self.samples - pass_begin
        arr = np.ascontiguousarray(rects, dtype=np.int32).reshape(-1, 4)
        rc = lib().crgpu_render_tiles(self.handle, arr.ctypes.data, len(arr), pass_begin, pass_count, flags, C.byref(st))
        return self._render_result(rc, flags, st, "crgpu_render_tiles")

    def _render_result(self, rc, flags, st, what):
        if rc != STOPPED:
            _check(rc, what)
        if flags & FLAG_ASYNC:
            return None
        d = st.as_dict()
        if getattr(self, "armed", False):
            d["stopped"] = rc == STOPPED
        return d

    def enable_stop(self, on=True):
        """Arm (or disarm) the scene: its render calls can then be stopped at a pass boundary (crgpu_stop_enable)."""
        _check(lib().crgpu_stop_enable(self.handle, 1 if on else 0), "crgpu_stop_enable")
        self.armed = bool(on)

    def request_stop(self):
        """Ask the call in flight (and every later call, until clear_stop) to end at the next pass boundary; any thread may call it."""
        _check(lib().crgpu_request_stop(self.handle), "crgpu_request_stop")

    def clear_stop(self):
        _check(lib().crgpu_clear_stop(self.handle), "crgpu_clear_stop")

    def progress(self):
        """(committed pass index of the call in flight or of the last one, whether a call is in flight), without synchronising."""
        done, busy = C.c_int(0), C.c_int(0)
        _check(lib().crgpu_progress(self.handle, C.byref(done), C.byref(busy)), "crgpu_progress")
        return done.value, bool(busy.value)

    def request_snapshot(self):
        """Ask the next publish step of the call in flight to stage the image (crgpu_request_snapshot); any thread may call it."""
        _check(lib().crgpu_request_snapshot(self.handle), "crgpu_request_snapshot")

    def take_snapshot(self):
        """(uint8 [H, W, 3] sRGB image, passes_done) once the requested image is staged, or with no call in flight the framebuffer
        as it is; None while the snapshot is pending.  Never waits for the render."""
        out = np.empty((self.H, self.W, 3), dtype=np.uint8)
        done = C.c_int(0)
        rc = lib().crgpu_take_snapshot(self.handle, out.ctypes.data, C.byref(done))
        if rc == PENDING:
            return None
        _check(rc, "crgpu_take_snapshot")
        return out, done.value

    def set_camera(self, camera):
        """Move the camera of the resident scene (crgpu_scene_set_camera): a Camera of the scene's image size, taken bit for bit."""
        _check(lib().crgpu_scene_set_camera(self.handle, C.byref(camera)), "crgpu_scene_set_camera")

    def set_instances(self, instances):
        """Re-place every instance (crgpu_scene_set_instances): an array of struct crs_instance (crscene.INSTANCE) with the uploaded
        count, kinds and objects; A and Ainv are taken bit for bit and the top-level BVH is rebuilt on the device."""
        import crscene
        arr = np.ascontiguousarray(instances, dtype=crscene.INSTANCE)
        _check(lib().crgpu_scene_set_instances(self.handle, arr.ctypes.data, len(arr)), "crgpu_scene_set_instances")

    def set_instance_list(self, instances):
        """Replace the whole instance list (crgpu_scene_set_instance_list): an array of struct crs_instance (crscene.INSTANCE) of any
        length up to 4,194,304, each a sphere or mesh the scene was uploaded with; A and Ainv are taken bit for bit and the top-level
        BVH is rebuilt on the device."""
        import crscene
        arr = np.ascontiguousarray(instances, dtype=crscene.INSTANCE)
        _check(lib().crgpu_scene_set_instance_list(self.handle, arr.ctypes.data if len(arr) else None, len(arr)),
               "crgpu_scene_set_instance_list")

    def set_meshes(self, flat, meshes):
        """Deform meshes of the resident scene (crgpu_scene_set_meshes): each mesh index in `meshes` takes its polys and the
        vertices, normals and texcoords they index from the FlatScene `flat` (same topology as uploaded), and its BVH, triangles and
        shading records, the instance boxes and the top level are rebuilt on the device."""
        idx = np.ascontiguousarray(meshes, dtype=np.uint32).reshape(-1)
        _check(lib().crgpu_scene_set_meshes(self.handle, C.byref(flat), idx.ctypes.data if len(idx) else None, len(idx)),
               "crgpu_scene_set_meshes")

    def set_shading(self, flat):
        """Replace the materials, node graph, textures, texel data and background of the resident scene with those of the FlatScene
        `flat` (crgpu_scene_set_shading): same material count, everything else of `flat` is ignored."""
        _check(lib().crgpu_scene_set_shading(self.handle, C.byref(flat)), "crgpu_scene_set_shading")

    def add_objects(self, flat):
        """Put new meshes and spheres into the resident scene (crgpu_scene_add_objects): the FlatScene `flat` is the grown scene as a
        whole, its first meshes and spheres the scene's own; the new meshes' BVHs are built on the device, and flat's shading and
        instance list replace the scene's."""
        _check(lib().crgpu_scene_add_objects(self.handle, C.byref(flat)), "crgpu_scene_add_objects")

    def shading(self):
        """How the shading kernels sample the live scene (crgpu_scene_shading): dict of kinds and flags (uint32 per material, as
        crgpu_prepared_materials gives them), background_kind and complete_interpreter."""
        n, bg, x = C.c_uint32(0), C.c_uint32(0), C.c_int(0)
        _check(lib().crgpu_scene_shading(self.handle, None, None, 0, C.byref(n), C.byref(bg), C.byref(x)), "crgpu_scene_shading")
        kinds, flags = np.zeros(n.value, np.uint32), np.zeros(n.value, np.uint32)
        _check(lib().crgpu_scene_shading(self.handle, kinds.ctypes.data, flags.ctypes.data, n.value, None, None, None), "crgpu_scene_shading")
        return {"kinds": kinds, "flags": flags, "background_kind": bg.value, "complete_interpreter": bool(x.value)}

    def set_views(self, cameras):
        """Replace the view list (crgpu_scene_set_views): a sequence of Camera of the scene's image size, taken bit for bit; the first
        becomes the scene camera.  Surviving views keep their framebuffers, new views start zeroed."""
        arr = (Camera * len(cameras))(*cameras)
        _check(lib().crgpu_scene_set_views(self.handle, arr, len(cameras)), "crgpu_scene_set_views")

    def set_render(self, width, height, samples, bounces, cameras=None):
        """Change image size, sample count and bounce limit (crgpu_scene_set_render): `cameras` is a sequence of Camera of the new
        size, one per view (the first becomes the scene camera), or None to keep every camera when the size stays.  A new size
        gives every view a new zeroed framebuffer; an unchanged size touches none."""
        if cameras is None:
            arr, n = None, self.view_count()
        else:
            arr, n = (Camera * len(cameras))(*cameras), len(cameras)
        _check(lib().crgpu_scene_set_render(self.handle, width, height, samples, bounces, arr, n), "crgpu_scene_set_render")
        self.W, self.H, self.samples, self.bounces = width, height, samples, bounces

    def adaptive_reset(self):
        """Give every pixel of view 0 a fresh adaptive record: 0 passes, err +inf, not done (crgpu_adaptive_reset)."""
        _check(lib().crgpu_adaptive_reset(self.handle), "crgpu_adaptive_reset")

    def adaptive_round(self, rects, min_passes, round_passes, threshold, floor, pass_end=None, flags=0):
        """One adaptive round over the tile set [(x0, y0, x1, y1), ...] (crgpu_adaptive_round).  Returns a dict: the call's stats (none
        with FLAG_ASYNC), "active", "pass_begin", "pass_end" (the passes [pass_begin, pass_end) rendered for the active pixels) and, on
        an armed scene, "stopped"."""
        st = Stats()
        a = Adaptive(min_passes, round_passes, self.samples if pass_end is None else pass_end, threshold, floor)
        arr = np.ascontiguousarray(rects, dtype=np.int32).reshape(-1, 4)
        active, pb, pe = C.c_uint32(0), C.c_int(0), C.c_int(0)
        rc = lib().crgpu_adaptive_round(self.handle, arr.ctypes.data, len(arr), C.byref(a), flags, C.byref(st), C.byref(active), C.byref(pb),
                                        C.byref(pe))
        d = self._render_result(rc, flags, st, "crgpu_adaptive_round") or {}
        d.update(active=active.value, pass_begin=pb.value, pass_end=pe.value)
        return d

    def adaptive_read(self):
        """(passes uint32 [H, W], err float32 [H, W]) of every pixel, in the framebuffer layout (as read() gives the image)."""
        n = np.empty((self.H, self.W), dtype=np.uint32)
        err = np.empty((self.H, self.W), dtype=np.float32)
        _check(lib().crgpu_adaptive_read(self.handle, n.ctypes.data, err.ctypes.data), "crgpu_adaptive_read")
        return n, err

    def render_adaptive(self, rects, min_passes, round_passes, threshold, floor, pass_end=None):
        """Adaptive rounds over the tile set until no pixel is active, or until an armed round is stopped (synchronous).  Does not
        reset: call adaptive_reset (and clear) first for a new frame.  Returns the stats summed over the rounds, with "rounds" and, on
        an armed scene, "stopped"."""
        total = {n: 0 for n, _ in Stats._fields_ if n != "pad"}
        total["rounds"] = 0
        while True:
            d = self.adaptive_round(rects, min_passes, round_passes, threshold, floor, pass_end)
            for k in Stats._fields_:
                if k[0] != "pad":
                    total[k[0]] += d[k[0]]
            if d["active"] == 0:
                break
            total["rounds"] += 1
            if d.get("stopped"):
                total["stopped"] = True
                return total
        if getattr(self, "armed", False):
            total["stopped"] = False
        return total

    def adaptive_records(self):
        """Every pixel's whole record (ADAPT_RECORD_DTYPE [H, W], the framebuffer layout) (crgpu_adaptive_records)."""
        out = np.empty((self.H, self.W), dtype=ADAPT_RECORD_DTYPE)
        _check(lib().crgpu_adaptive_records(self.handle, out.ctypes.data), "crgpu_adaptive_records")
        return out

    def adaptive_write(self, recs):
        """Load every pixel's record from ADAPT_RECORD_DTYPE [H, W] (crgpu_adaptive_write)."""
        recs = np.ascontiguousarray(recs, dtype=ADAPT_RECORD_DTYPE)
        assert recs.shape == (self.H, self.W)
        _check(lib().crgpu_adaptive_write(self.handle, recs.ctypes.data), "crgpu_adaptive_write")

    def adaptive_select(self, rects, min_passes, round_passes, threshold, floor, pass_end=None):
        """A round's select, scan and compaction without its render (crgpu_adaptive_select): (active list uint32 x | y << 16, least
        count, largest count)."""
        a = Adaptive(min_passes, round_passes, self.samples if pass_end is None else pass_end, threshold, floor)
        arr = np.ascontiguousarray(rects, dtype=np.int32).reshape(-1, 4)
        npix = int(((arr[:, 2] - arr[:, 0]).astype(np.int64) * (arr[:, 3] - arr[:, 1])).sum())
        active = np.empty(max(npix, 1), dtype=np.uint32)
        count, lo, hi = C.c_uint32(0), C.c_uint32(0), C.c_uint32(0)
        _check(lib().crgpu_adaptive_select(self.handle, arr.ctypes.data, len(arr), C.byref(a), active.ctypes.data, C.byref(count),
                                           C.byref(lo), C.byref(hi)), "crgpu_adaptive_select")
        return active[:count.value].copy(), lo.value, hi.value

    def accumulate_samples(self, rects, pass_begin, L, order=-1, adaptive=False):
        """K5 on given radiance (crgpu_accumulate_samples): L is float32 [npix, passes, 4] in the tile set's list order, added to the
        framebuffer as passes [pass_begin, +passes) under path order `order` (-1: the process's); with `adaptive` the records take
        them too.  Returns the tile set's pixel list (uint32 x | y << 16)."""
        arr = np.ascontiguousarray(rects, dtype=np.int32).reshape(-1, 4)
        L = np.ascontiguousarray(L, dtype=np.float32)
        npix = int(((arr[:, 2] - arr[:, 0]).astype(np.int64) * (arr[:, 3] - arr[:, 1])).sum())
        assert L.ndim == 3 and L.shape[0] == npix and L.shape[2] == 4
        pixels = np.empty(max(npix, 1), dtype=np.uint32)
        _check(lib().crgpu_accumulate_samples(self.handle, arr.ctypes.data, len(arr), pass_begin, L.shape[1], order, 1 if adaptive else 0,
                                              L.ctypes.data, pixels.ctypes.data), "crgpu_accumulate_samples")
        return pixels[:npix]

    def view_count(self):
        n = C.c_uint32(0)
        _check(lib().crgpu_scene_view_count(self.handle, C.byref(n)), "crgpu_scene_view_count")
        return n.value

    def render_views(self, rects, first=0, count=None, pass_begin=0, pass_count=None, flags=0):
        """Render the tile set [(x0, y0, x1, y1), ...] in views [first, first + count) as ONE wavefront (crgpu_render_views); each
        view ends as render_tiles would leave it under its own camera.  The result as for render_tile."""
        st = Stats()
        if count is None:
            count = self.view_count() - first
        if pass_count is None:
            pass_count = self.samples - pass_begin
        arr = np.ascontiguousarray(rects, dtype=np.int32).reshape(-1, 4)
        rc = lib().crgpu_render_views(self.handle, first, count, arr.ctypes.data, len(arr), pass_begin, pass_count, flags, C.byref(st))
        return self._render_result(rc, flags, st, "crgpu_render_views")

    def view_read(self, view):
        """float32 [H, W, 3] framebuffer of one view (the framebuffer layout, as read() gives view 0)."""
        out = np.empty((self.H, self.W, 3), dtype=np.float32)
        _check(lib().crgpu_view_read(self.handle, view, out.ctypes.data), "crgpu_view_read")
        return out

    def view_srgb8(self, view):
        out = np.empty((self.H, self.W, 3), dtype=np.uint8)
        _check(lib().crgpu_view_to_srgb8(self.handle, view, out.ctypes.data), "crgpu_view_to_srgb8")
        return out

    def view_clear(self, view):
        _check(lib().crgpu_view_clear(self.handle, view), "crgpu_view_clear")

    def set_stream(self, cuda_stream_ptr):
        """Enqueue on a caller-owned cudaStream_t (int pointer, e.g. torch.cuda.current_stream().cuda_stream)."""
        _check(lib().crgpu_set_stream(self.handle, C.c_void_p(cuda_stream_ptr)), "crgpu_set_stream")

    def use_own_stream(self):
        _check(lib().crgpu_use_own_stream(self.handle), "crgpu_use_own_stream")

    def get_stats(self):
        st = Stats()
        _check(lib().crgpu_get_stats(self.handle, C.byref(st)), "crgpu_get_stats")
        return st.as_dict()

    def render_frame(self, flags=0, tile=None):
        """Whole frame; tile=(tw,th) walks the reference's tile grid, else row bands sized to the path budget."""
        total = None
        if tile:
            rects = [(x, y, min(x + tile[0], self.W), min(y + tile[1], self.H))
                     for y in range(0, self.H, tile[1]) for x in range(0, self.W, tile[0])]
        else:
            rects = [(0, 0, self.W, self.H)]
        for r in rects:
            st = self.render_tile(*r, flags=flags)
            if total is None:
                total = st
            else:
                for k in total:
                    total[k] += st[k]
        return total

    def clear(self):
        _check(lib().crgpu_framebuffer_clear(self.handle), "crgpu_framebuffer_clear")

    def read(self, out=None):
        if out is None:
            out = np.empty((self.H, self.W, 3), dtype=np.float32)
        _check(lib().crgpu_framebuffer_read(self.handle, out.ctypes.data, 0, 0, 0, 0), "crgpu_framebuffer_read")
        return out

    def write(self, rgb):
        rgb = np.ascontiguousarray(rgb, dtype=np.float32)
        assert rgb.shape == (self.H, self.W, 3)
        _check(lib().crgpu_framebuffer_write(self.handle, rgb.ctypes.data, 0, 0, 0, 0), "crgpu_framebuffer_write")

    def srgb8(self):
        out = np.empty((self.H, self.W, 3), dtype=np.uint8)
        _check(lib().crgpu_framebuffer_to_srgb8(self.handle, out.ctypes.data), "crgpu_framebuffer_to_srgb8")
        return out

    def device_ptr(self):
        p, n = C.c_void_p(), C.c_size_t()
        _check(lib().crgpu_framebuffer_device_ptr(self.handle, C.byref(p), C.byref(n)), "crgpu_framebuffer_device_ptr")
        return p.value, n.value

    def trace_kat(self, xyp):
        xyp = np.ascontiguousarray(xyp, dtype=np.int32).reshape(-1, 3)
        out = np.zeros(len(xyp) * 160, dtype=np.uint8)
        _check(lib().crgpu_trace_kat(self.handle, xyp.ctypes.data, len(xyp), out.ctypes.data), "crgpu_trace_kat")
        return out

    def trace_rays(self, rays, order=None, **knobs):
        """Closest hits of rays (n x 6 float32: origin, direction) through the frame's traversal kernel and bucket sort.
        knobs: count, minb, defer, refill, burst, inst_min (TRACE_DEFAULTS); order: a permutation K2 takes the rays in.
        Returns (records, perm, misses, stats)."""
        rays = np.ascontiguousarray(rays, dtype=np.float32).reshape(-1, 6)
        n = len(rays)
        k = dict(TRACE_DEFAULTS)
        if knobs.get("defer"):
            k["burst"] = 4
        k.update(knobs)
        opts = TraceOpts(**{f: int(k[f]) for f in TRACE_DEFAULTS})
        if order is not None:
            order = np.ascontiguousarray(order, dtype=np.uint32)
            assert order.shape == (n,)
            opts.order = order.ctypes.data
        rec = np.zeros(n, dtype=RAY_RECORD_DTYPE)
        perm = np.zeros(n, dtype=np.uint32)
        misses = C.c_uint32(0)
        st = Stats()
        _check(lib().crgpu_trace_rays(self.handle, rays.ctypes.data, n, C.byref(opts), rec.ctypes.data, perm.ctypes.data,
                                      C.byref(misses), C.byref(st)), "crgpu_trace_rays")
        return rec, perm, misses.value, st.as_dict()

    def shade_rays(self, states, depth, max_depth, **opts):
        """One bounce of path states (PATH_STATE_DTYPE) through the frame's K2 -> K4 -> K3 (-> K4b), or the tail kernel (tail=1).
        opts: minb, split, prefetch, dirmode, complete_interpreter, tail, generic_only (SHADE_DEFAULTS).
        Returns (results (SHADE_RESULT_DTYPE, one per state), perm2 of the survivors, survivors, origin-box slot (12 x u32))."""
        states = np.ascontiguousarray(states, dtype=PATH_STATE_DTYPE)
        n = len(states)
        k = dict(SHADE_DEFAULTS)
        k.update(opts)
        o = ShadeOpts(depth=int(depth), max_depth=int(max_depth), **{f: int(k[f]) for f in SHADE_DEFAULTS})
        res = np.zeros(n, dtype=SHADE_RESULT_DTYPE)
        perm2 = np.zeros(n, dtype=np.uint32)
        box = np.zeros(12, dtype=np.uint32)
        surv = C.c_uint32(0)
        _check(lib().crgpu_shade_rays(self.handle, states.ctypes.data, n, C.byref(o), res.ctypes.data, perm2.ctypes.data,
                                      C.byref(surv), box.ctypes.data), "crgpu_shade_rays")
        return res, perm2[:surv.value], surv.value, box

    def set_max_paths(self, n):
        _check(lib().crgpu_set_max_paths_in_flight(self.handle, int(n)), "crgpu_set_max_paths_in_flight")

    def close(self):
        if self.handle:
            lib().crgpu_scene_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def libm_eval(fn, x, y=None, device=0):
    """The device's fp64 libm stand-in `fn` (a name of LIBM) over float32 arrays x (and y: atan2's x, pow's exponent)."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    y = np.zeros_like(x) if y is None else np.ascontiguousarray(y, dtype=np.float32)
    out = np.zeros_like(x)
    _check(lib().crgpu_libm_eval(device, LIBM.index(fn), x.ctypes.data, y.ctypes.data, out.ctypes.data, len(x)), "crgpu_libm_eval")
    return out


class RankGather:
    """libcrgpu_nccl.so through ctypes: the tile gather of a one-process-per-GPU job on an EXISTING communicator (crgpu_comm*,
    e.g. crhost.Renderer.comm()).  Loaded after libcrgpu.so (its symbols) — and after torch when torch is in the process, so
    that both bind the one libnccl.so.2 already mapped."""

    def __init__(self, comm_ptr):
        lib()
        C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
        self.L = C.CDLL(os.path.join(HERE, "libcrgpu_nccl.so"))
        P = C.c_void_p
        self.L.crgpu_comm_gather_tiles_rank.argtypes = [P, P, P, P, C.c_int, C.c_int]
        self.L.crgpu_comm_set_stream.argtypes = [P, P, C.c_int]
        self.comm = C.c_void_p(comm_ptr)

    def set_stream(self, cuda_stream_ptr):
        if self.L.crgpu_comm_set_stream(self.comm, C.c_void_p(cuda_stream_ptr), 0) != 0:
            raise CrgpuError("crgpu_comm_set_stream failed")

    def use_own_stream(self):
        if self.L.crgpu_comm_set_stream(self.comm, None, 1) != 0:
            raise CrgpuError("crgpu_comm_set_stream failed")

    def gather(self, scene, rects, owner, root=0):
        rects = np.ascontiguousarray(rects, dtype=np.int32).reshape(-1, 4)
        owner = np.ascontiguousarray(owner, dtype=np.int32)
        rc = self.L.crgpu_comm_gather_tiles_rank(self.comm, scene.handle, rects.ctypes.data, owner.ctypes.data, len(rects), root)
        if rc != 0:
            raise CrgpuError(f"crgpu_comm_gather_tiles_rank failed ({rc})")
