"""ctypes view of oracle/libcray_oracle.so (the CPU restatement) — test infrastructure only."""
import ctypes as C
import os
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILT = os.path.join(ROOT, "scenes", "_built")
REF_DIGESTS = os.path.join(ROOT, "tests", "golden", "ref_frames.sha256.json")


def frame_digest(img):
    """SHA-256 of an fp32 framebuffer's bytes: how a frame is compared bit for bit with a stored reference frame."""
    import hashlib
    return hashlib.sha256(np.ascontiguousarray(img, dtype=np.float32).tobytes()).hexdigest()


def reference_digest(name, W, H, spp, b):
    """SHA-256 of the framebuffer the unmodified reference (strict build) rendered for input/<name>.json at W x H x spp, b bounces
    (tests/golden/ref_frames.sha256.json, recorded from the reference's own renders)."""
    import json
    return json.load(open(REF_DIGESTS))[f"ref_{name}_{W}x{H}x{spp}_b{b}"]


def bundled_scene(name, tmpdir):
    """A bundled input/<name>.json scene as a flat .crscene: scenes/_built/<name>.crscene (the reference loader's export) where it
    was built, else flattened by this repository's loader from oracle/_ref/input/<name>.json into tmpdir (tests/test_loader.py
    shows the two are the same bytes).  None when neither is present."""
    scene = os.path.join(BUILT, name + ".crscene")
    if os.path.exists(scene):
        return scene
    refdir = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.exists(os.path.join(refdir, "input", name + ".json")):
        return None
    import crgpu
    import crscene
    cwd = os.getcwd()
    os.chdir(refdir)                       # node-graph texture paths are relative to the reference's working directory
    try:
        flat = crscene.load_json(os.path.join("input", name + ".json"))
    finally:
        os.chdir(cwd)
    scene = os.path.join(str(tmpdir), name + ".crscene")
    L = crgpu.lib()
    L.crscene_save.argtypes = [C.POINTER(crgpu.FlatScene), C.c_char_p]
    rc = L.crscene_save(C.byref(flat), scene.encode())
    crscene.free(flat)
    if rc != 0:
        raise RuntimeError(f"crscene_save({scene}) failed ({rc})")
    return scene


class Prefs(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("image_width", "image_height", "sample_count", "bounces",
                                          "tile_width", "tile_height", "tile_order", "thread_count")]


class Camera(C.Structure):
    _fields_ = [("sensor_x", C.c_float), ("sensor_y", C.c_float), ("aperture", C.c_float),
                ("focal_distance", C.c_float), ("forward", C.c_float * 3), ("right", C.c_float * 3),
                ("up", C.c_float * 3), ("width", C.c_int32), ("height", C.c_int32), ("pad", C.c_uint32),
                ("A", C.c_float * 16)]


class Scene(C.Structure):
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


class Counters(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("paths", "rays", "node_pairs", "tri_tests", "sphere_tests",
                                          "inst_visits", "draws", "max_depth", "max_stack", "max_pairs_ray")]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


HIT_KAT_DTYPE = np.dtype([("x", "<i4"), ("y", "<i4"), ("pixIdx", "<i4"), ("instIndex", "<i4"), ("polyIndex", "<i4"),
                          ("o", "<f4", 3), ("d", "<f4", 3), ("distance", "<f4"), ("uv", "<f4", 2),
                          ("hitPoint", "<f4", 3), ("normal", "<f4", 3), ("emission", "<f4", 3),
                          ("out", "<f4", 3), ("color", "<f4", 4), ("nextDraw", "<f4"), ("pad", "<f4", 9)])
assert HIT_KAT_DTYPE.itemsize == 160

# struct cro_ray_record: one closest-hit record per ray (cro_closest_hit)
RAY_RECORD_DTYPE = np.dtype([("t", "<f4"), ("u", "<f4"), ("v", "<f4"), ("inst", "<i4"), ("poly", "<i4"), ("material", "<i4")])
assert RAY_RECORD_DTYPE.itemsize == 24
SEM_REFERENCE, SEM_DEVICE = 0, 1
# struct cro_path_state / cro_step_result (cro_path_step)
PATH_STATE_DTYPE = np.dtype([("o", "<f4", 3), ("d", "<f4", 3), ("weight", "<f4", 3), ("has_l", "<u4"), ("rng", "<u8"),
                             ("L", "<f4", 3), ("pad", "<u4")])
assert PATH_STATE_DTYPE.itemsize == 64
STEP_RESULT_DTYPE = np.dtype([("rec", RAY_RECORD_DTYPE), ("alive", "<i4"), ("flag", "<u4"), ("next", PATH_STATE_DTYPE)])
assert STEP_RESULT_DTYPE.itemsize == 96
LIBM = ["sin", "cos", "tan", "log", "log10", "atan2", "acos", "asin", "pow", "pow5"]

_lib = None


def lib():
    global _lib
    if _lib is None:
        path = os.path.join(ROOT, "oracle", "libcray_oracle.so")
        if not os.path.exists(path):
            raise RuntimeError("oracle/libcray_oracle.so missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
        L = C.CDLL(path)
        L.crscene_load.argtypes = [C.POINTER(Scene), C.c_char_p]
        L.crscene_load.restype = C.c_int
        L.crscene_free.argtypes = [C.POINTER(Scene)]
        L.crscene_set_config.argtypes = [C.POINTER(Scene)] + [C.c_int] * 4
        L.cro_render.argtypes = [C.POINTER(Scene)] + [C.c_int] * 6 + [C.c_void_p, C.c_int, C.POINTER(Counters)]
        L.cro_render.restype = C.c_int
        L.cro_sampler_kat.argtypes = [C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_void_p]
        L.cro_trace_kat.argtypes = [C.POINTER(Scene), C.c_int, C.c_int, C.c_int, C.c_void_p]
        L.cro_to_srgb8.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        L.cro_closest_hit.argtypes = [C.POINTER(Scene), C.c_size_t, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.POINTER(Counters)]
        L.cro_closest_hit.restype = C.c_int
        L.cro_trace_region.argtypes = [C.POINTER(Scene)] + [C.c_int] * 6 + [C.c_void_p, C.c_size_t]
        L.cro_trace_region.restype = C.c_size_t
        L.cro_render_sem.argtypes = [C.POINTER(Scene)] + [C.c_int] * 6 + [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.POINTER(Counters)]
        L.cro_render_sem.restype = C.c_int
        L.cro_camera_states.argtypes = [C.POINTER(Scene)] + [C.c_int] * 7 + [C.c_void_p]
        L.cro_path_step.argtypes = [C.POINTER(Scene), C.c_size_t, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
        L.cro_path_step.restype = C.c_int
        L.cro_libm.argtypes = [C.c_int, C.c_int, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.cro_libm.restype = C.c_int
        _lib = L
    return _lib


class OracleScene:
    def __init__(self, path, width=0, height=0, samples=0, bounces=0):
        self.s = Scene()
        rc = lib().crscene_load(C.byref(self.s), path.encode())
        if rc != 0:
            raise RuntimeError(f"crscene_load({path}) failed: {rc}")
        lib().crscene_set_config(C.byref(self.s), width, height, samples, bounces)
        self.W = self.s.prefs.image_width
        self.H = self.s.prefs.image_height

    def render(self, threads=8, tile=None, passes=None, rgb=None, count=False):
        """Full frame (or tile=(x0,y0,x1,y1), passes=(begin,count)); returns fp32 (H,W,3) y-flipped like renderBuffer."""
        if rgb is None:
            rgb = np.zeros((self.H, self.W, 3), dtype=np.float32)
        x0, y0, x1, y1 = tile if tile else (0, 0, self.W, self.H)
        pb, pc = passes if passes else (0, self.s.prefs.sample_count)
        ctr = Counters()
        lib().cro_render(C.byref(self.s), x0, y0, x1, y1, pb, pc, rgb.ctypes.data, threads,
                         C.byref(ctr) if count else None)
        return (rgb, ctr.as_dict()) if count else rgb

    def trace_kat(self, x, y, p):
        out = np.zeros(1, dtype=HIT_KAT_DTYPE)
        lib().cro_trace_kat(C.byref(self.s), x, y, p, out.ctypes.data)
        return out[0]

    def closest_hit(self, rays, semantics=SEM_DEVICE, threads=None):
        """Closest-hit records of rays (n x 6 float32: origin, direction) and the batch's counters (P/T/S/I, rays)."""
        rays = np.ascontiguousarray(rays, dtype=np.float32).reshape(-1, 6)
        out = np.zeros(len(rays), dtype=RAY_RECORD_DTYPE)
        ctr = Counters()
        rc = lib().cro_closest_hit(C.byref(self.s), len(rays), rays.ctypes.data, semantics, threads or os.cpu_count() or 1,
                                   out.ctypes.data, C.byref(ctr))
        if rc != 0:
            raise RuntimeError(f"cro_closest_hit failed ({rc})")
        return out, ctr.as_dict()

    def path_rays(self, x0, y0, x1, y1, passes=(0, 1), cap=64 << 20):
        """Every ray of every bounce of the paths of a region (cro_trace_region), n x 6 float32, in path order."""
        buf = np.zeros(cap, dtype=np.uint8)
        n = lib().cro_trace_region(C.byref(self.s), x0, y0, x1, y1, passes[0], passes[1], buf.ctypes.data, cap)
        assert n + 4096 < cap, "trace buffer too small for the region"
        rays, pos = [], 0
        while pos < n:
            ev = int(buf[pos + 8:pos + 12].view(np.uint32)[0])
            rays.append(buf[pos + 12:pos + 36].view(np.float32))
            pos += 36 + ev
        return np.array(rays, dtype=np.float32).reshape(-1, 6)

    def render_sem(self, semantics, threads=None, tile=None, passes=None):
        """Full frame (or a tile / pass range) in the given semantics: (fp32 (H,W,3) frame, per-pixel count of flagged samples)."""
        rgb = np.zeros((self.H, self.W, 3), dtype=np.float32)
        flagged = np.zeros((self.H, self.W), dtype=np.uint32)
        x0, y0, x1, y1 = tile if tile else (0, 0, self.W, self.H)
        pb, pc = passes if passes else (0, self.s.prefs.sample_count)
        rc = lib().cro_render_sem(C.byref(self.s), x0, y0, x1, y1, pb, pc, rgb.ctypes.data, threads or os.cpu_count() or 1,
                                  semantics, flagged.ctypes.data, None)
        if rc != 0:
            raise RuntimeError(f"cro_render_sem failed ({rc})")
        return rgb, flagged

    def camera_states(self, x0, y0, x1, y1, passes=None, semantics=SEM_DEVICE):
        """Path states of the camera rays of a region: pixels row-major (y up), passes innermost (pad = near-tie flag)."""
        pb, pc = passes if passes else (0, self.s.prefs.sample_count)
        out = np.zeros((y1 - y0) * (x1 - x0) * pc, dtype=PATH_STATE_DTYPE)
        lib().cro_camera_states(C.byref(self.s), x0, y0, x1, y1, pb, pc, semantics, out.ctypes.data)
        return out

    def path_step(self, states, depth, max_depth=None, bounces=1, semantics=SEM_DEVICE, threads=None):
        """`bounces` passes of pathTrace's loop body from bounce `depth` (STEP_RESULT_DTYPE per state)."""
        states = np.ascontiguousarray(states, dtype=PATH_STATE_DTYPE)
        out = np.zeros(len(states), dtype=STEP_RESULT_DTYPE)
        md = self.s.prefs.bounces if max_depth is None else max_depth
        rc = lib().cro_path_step(C.byref(self.s), len(states), states.ctypes.data, depth, md, bounces, semantics,
                                 threads or os.cpu_count() or 1, out.ctypes.data)
        if rc != 0:
            raise RuntimeError(f"cro_path_step failed ({rc})")
        return out

    def close(self):
        lib().crscene_free(C.byref(self.s))


def libm(fn, semantics, x, y=None):
    """An oracle libm call over float32 arrays: (results, near-tie flags)."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    y = np.zeros_like(x) if y is None else np.ascontiguousarray(y, dtype=np.float32)
    out = np.zeros_like(x)
    flag = np.zeros(len(x), dtype=np.uint8)
    rc = lib().cro_libm(LIBM.index(fn), semantics, len(x), x.ctypes.data, y.ctypes.data, out.ctypes.data, flag.ctypes.data)
    assert rc == 0
    return out, flag.astype(bool)


def sampler_kat(pix, p, maxp, n):
    out = np.zeros(n, dtype=np.float32)
    lib().cro_sampler_kat(pix, p, maxp, n, out.ctypes.data)
    return out
