"""numpy view of the flat scene (include/crscene.h) and ctypes binding of the scene loader (include/crloader.h).

`load_json(path)` runs libcrloader.so (c-ray_b200/host/loader/, plain C: JSON + OBJ/MTL + PNG/HDR + BVH build) and
returns a FlatScene that `crgpu.GpuScene.from_flat` can upload; `arrays(scene)` exposes the 14 arrays as structured
numpy arrays (copies), which is what tests/test_loader.py compares against the reference's exported scenes.
"""
import ctypes as C
import os

import numpy as np

from crgpu import FlatScene

HERE = os.path.dirname(os.path.abspath(__file__))
LOADER_PATH = os.path.join(HERE, "libcrloader.so")

INSTANCE = np.dtype([("A", "<f4", 16), ("Ainv", "<f4", 16), ("kind", "<u4"), ("object", "<u4"), ("pad", "<u4", 2)])
SPHERE = np.dtype([("radius", "<f4"), ("ray_offset", "<f4"), ("material", "<u4"), ("pad", "<u4")])
MESH = np.dtype([("poly_offset", "<u4"), ("poly_count", "<u4"), ("material_offset", "<u4"), ("material_count", "<u4"),
                 ("texcoord_count", "<u4"), ("bvh", "<u4"), ("ray_offset", "<f4"), ("pad", "<u4")])
MATERIAL = np.dtype([("emission", "<f4", 4), ("IOR", "<f4"), ("bsdf", "<i4"), ("pad", "<u4", 2)])
NODE = np.dtype([("kind", "<i4"), ("in", "<i4", 3), ("f", "<f4", 8), ("tex", "<i4"), ("options", "<u4"), ("pad", "<u4", 2)])
TEXTURE = np.dtype([("width", "<u4"), ("height", "<u4"), ("channels", "<u4"), ("is_float", "<u4"), ("has_alpha", "<u4"),
                    ("pad", "<u4"), ("data_offset", "<u8")])
BVH = np.dtype([("node_offset", "<u4"), ("node_count", "<u4"), ("prim_offset", "<u4"), ("prim_count", "<u4")])
BVH_NODE = np.dtype([("bounds", "<f4", 6), ("first", "<u4"), ("count_leaf", "<u4")])
POLY = np.dtype([("v", "<i4", 3), ("n", "<i4", 3), ("t", "<i4", 3), ("material", "<u4"), ("has_normals", "<u4")])
assert (INSTANCE.itemsize, SPHERE.itemsize, MESH.itemsize, MATERIAL.itemsize, NODE.itemsize, TEXTURE.itemsize,
        BVH.itemsize, BVH_NODE.itemsize, POLY.itemsize) == (144, 16, 32, 32, 64, 32, 16, 32, 44)

LEAF_BIT = 1 << 30
COUNT_MASK = LEAF_BIT - 1

_SECTIONS = [("instances", INSTANCE, "instance_count", 1), ("spheres", SPHERE, "sphere_count", 1),
             ("meshes", MESH, "mesh_count", 1), ("materials", MATERIAL, "material_count", 1),
             ("nodes", NODE, "node_count", 1), ("textures", TEXTURE, "texture_count", 1), ("bvhs", BVH, "bvh_count", 1),
             ("bvh_nodes", BVH_NODE, "bvh_node_count", 1), ("prim_indices", np.dtype("<i4"), "prim_index_count", 1),
             ("polys", POLY, "poly_count", 1), ("vertices", np.dtype("<f4"), "vertex_count", 3),
             ("normals", np.dtype("<f4"), "normal_count", 3), ("texcoords", np.dtype("<f4"), "texcoord_count", 2),
             ("texdata", np.dtype("u1"), "texdata_bytes", 1)]


def arrays(scene):
    """dict name -> numpy copy of each array of a FlatScene (vertices/normals as (n,3), texcoords as (n,2))."""
    out = {}
    for name, dtype, count_field, width in _SECTIONS:
        n = int(getattr(scene, count_field)) * width
        ptr = getattr(scene, name)
        if n == 0 or not ptr:
            a = np.zeros(0, dtype=dtype)
        else:
            a = np.frombuffer(C.string_at(ptr, n * dtype.itemsize), dtype=dtype).copy()
        out[name] = a.reshape(-1, width) if width > 1 else a
    return out


def write_back(scene, name, values):
    """Write `values` over the FlatScene array `name` ("vertices", "normals", "texcoords" or "polys") in place, from its first
    element: `arrays` returns copies, so an edited copy goes back this way (e.g. before crgpu.GpuScene.set_meshes).  The scene must
    own writable arrays, as load_json and load_json_buf return (crscene_load maps its file read-only)."""
    table = {n: (dtype, count_field, width) for n, dtype, count_field, width in _SECTIONS}
    if name not in ("vertices", "normals", "texcoords", "polys"):
        raise ValueError(f"write_back: {name!r} is not vertices, normals, texcoords or polys")
    dtype, count_field, width = table[name]
    a = np.ascontiguousarray(values, dtype=dtype).reshape(-1)
    n = int(getattr(scene, count_field)) * width
    if len(a) > n:
        raise ValueError(f"write_back: {len(a)} elements of {name}, the scene has {n}")
    if len(a):
        C.memmove(getattr(scene, name), a.ctypes.data, a.nbytes)


_loader = None


def loader():
    global _loader
    if _loader is None:
        if not os.path.exists(LOADER_PATH):
            raise RuntimeError(f"{LOADER_PATH} is missing — build it with `python -c 'import __graft_entry__ as g; g.build()'`")
        L = C.CDLL(LOADER_PATH)
        L.crloader_load_json.argtypes = [C.POINTER(FlatScene), C.c_char_p]
        L.crloader_load_json.restype = C.c_int
        L.crloader_load_json_buf.argtypes = [C.POINTER(FlatScene), C.c_char_p, C.c_char_p, C.c_void_p]
        L.crloader_load_json_buf.restype = C.c_int
        L.crloader_last_error.restype = C.c_char_p
        _loader = L
    return _loader


_libc = C.CDLL(None)
_libc.free.argtypes = [C.c_void_p]


def load_json(path):
    """Parse a c-ray JSON scene (+ its assets) into a FlatScene.  Raises RuntimeError with the loader's message."""
    s = FlatScene()
    rc = loader().crloader_load_json(C.byref(s), os.fsencode(path))
    if rc != 0:
        raise RuntimeError(f"crloader_load_json({path}) failed ({rc}): {loader().crloader_last_error().decode()}")
    return s


def load_json_buf(text, asset_path=None):
    """Parse c-ray JSON text already in memory into a FlatScene (crloader_load_json_buf); mesh and HDR names are resolved against
    asset_path (a directory; None = the working directory)."""
    if asset_path is not None:
        asset_path = os.path.join(os.fsdecode(asset_path), "")
    s = FlatScene()
    rc = loader().crloader_load_json_buf(C.byref(s), text.encode() if isinstance(text, str) else text,
                                         None if asset_path is None else os.fsencode(asset_path), None)
    if rc != 0:
        raise RuntimeError(f"crloader_load_json_buf failed ({rc}): {loader().crloader_last_error().decode()}")
    return s


def free(scene):
    """Release a FlatScene returned by load_json."""
    if scene.owner:
        _libc.free(scene.owner)
        scene.owner = None


def prim_boxes(vertices, polys):
    """(bboxes n x 6, centers n x 3) of a mesh's triangles exactly as the loader computes them (cr_sceneload.c poly_bbox <- reference
    bvh.c:283-291): the min/max MACROS (a < b ? a : b — ties return the second operand, which decides the sign of a zero) and the
    centre (v0 + v1 + v2) * (1/3) in fp32."""
    V = np.ascontiguousarray(vertices, dtype=np.float32).reshape(-1, 3)
    v0, v1, v2 = V[polys["v"][:, 0]], V[polys["v"][:, 1]], V[polys["v"][:, 2]]
    mn = lambda a, b: np.where(a < b, a, b)
    mx = lambda a, b: np.where(a > b, a, b)
    bb = np.concatenate([mn(v0, mn(v1, v2)), mx(v0, mx(v1, v2))], axis=1).astype(np.float32)
    ct = ((v0 + v1).astype(np.float32) + v2).astype(np.float32) * np.float32(1.0 / 3.0)
    return np.ascontiguousarray(bb), np.ascontiguousarray(ct.astype(np.float32))


def _build(fn, bboxes, centers, *extra):
    bb = np.ascontiguousarray(bboxes, dtype=np.float32).reshape(-1, 6)
    ct = np.ascontiguousarray(centers, dtype=np.float32).reshape(-1, 3)
    n = len(bb)
    nodes = np.zeros(max(2 * n, 1), dtype=BVH_NODE)
    prims = np.zeros(max(n, 1), dtype=np.int32)
    cnt = C.c_uint32(0)
    rc = fn(bb.ctypes.data_as(C.c_void_p), ct.ctypes.data_as(C.c_void_p), C.c_uint32(n), *extra,
            nodes.ctypes.data_as(C.c_void_p), C.byref(cnt), prims.ctypes.data_as(C.c_void_p))
    return rc, nodes[:cnt.value].copy(), prims[:n].copy()


def build_bvh(bboxes, centers):
    """crloader_build_bvh: the host binned-SAH builder on its own -> (nodes BVH_NODE[], prims int32[])."""
    L = loader()
    L.crloader_build_bvh.restype = C.c_int
    rc, nodes, prims = _build(L.crloader_build_bvh, bboxes, centers)
    if rc != 0:
        raise RuntimeError(f"crloader_build_bvh failed ({rc}): " + L.crloader_last_error().decode(errors="replace"))
    return nodes, prims


def build_bvh_gpu(bboxes, centers, device=0):
    """crgpu_bvh_build (SURVEY 8 f1): the same tree built on the device."""
    import crgpu
    G = crgpu.lib()
    G.crgpu_bvh_build.restype = C.c_int
    rc, nodes, prims = _build(G.crgpu_bvh_build, bboxes, centers, C.c_int(device))
    if rc != 0:
        raise crgpu.CrgpuError(f"crgpu_bvh_build failed ({rc}): " + G.crgpu_last_error().decode(errors="replace"))
    return nodes, prims
