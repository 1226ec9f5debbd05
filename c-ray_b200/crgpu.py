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
                  "crgpu_shade_rays", "crgpu_libm_eval", "crgpu_prepared_background",
                  "crgpu_scene_create_prepared", "crgpu_scene_info", "crgpu_device_trim",
                  "crgpu_stop_enable", "crgpu_request_stop", "crgpu_clear_stop", "crgpu_progress",

                  "crgpu_scene_set_camera", "crgpu_scene_set_instances", "crscene_set_config"):
            getattr(L, f).restype = C.c_int
        if hasattr(L, "crgpu_take_snapshot"):      # absent from libraries built before snapshots (tools/driver_check.py compares builds)
            L.crgpu_request_snapshot.argtypes = [P]
            L.crgpu_take_snapshot.argtypes = [P, P, C.POINTER(C.c_int)]
            L.crgpu_request_snapshot.restype = L.crgpu_take_snapshot.restype = C.c_int
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
