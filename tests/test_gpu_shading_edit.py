"""Editing the materials and the background of a resident GPU scene (crgpu_scene_set_shading / crgpu_scene_shading, include/crgpu.h).

The target is exact: a scene A edited with the shading of a scene B renders the same bits as B loaded fresh, when B differs from A
only in its materials, node graph, textures, texel data and background.  B is either A's flat arrays with new shading arrays
(Shading), which keeps the geometry identical by construction, or the JSON loaded again with other materials (the geometry arrays are
then compared).  Edited == fresh means: the same framebuffer, the same trace_kat records (they hold the bsdf sample), the same
shade_rays results over a fixed set of path states (K3 hit and miss launches and the tail kernel), and crgpu_scene_shading of the
edited scene equal to crgpu_prepared_materials / crgpu_prepared_background of a fresh prepare of B.

CPU: argument checks, and the validation and fold against the stub CUDA runtime (tests/stub/shading_harness.c).  GPU: the rest.
"""
import copy
import ctypes as C
import hashlib
import json
import os
import random
import subprocess

import numpy as np
import pytest

import crgpu
import crscene
from conftest import GOLDEN, ROOT
from test_gpu_scene_edit import DIGESTS, GOLDEN_FRAMES, SMALL, STEP, Loaded, digest, edited, full, ray_set, scene_json

PKG = os.path.join(ROOT, "c-ray_b200")
GEOMETRY = ("instances", "spheres", "meshes", "bvhs", "bvh_nodes", "prim_indices", "polys", "vertices", "normals", "texcoords")
GOLDEN_JSON = ["g_single", "g_legacy", "g_nodes", "g_meshmat", "g_f4"]
BOUNCES = {"hdr": 32, "venus": 25, "refraction": 512}

# node kinds (include/crscene.h enum crs_node_kind)
DIFFUSE, METAL, GLASS, PLASTIC, MIX, ADD, TRANSPARENT, EMISSIVE, BACKGROUND = 1, 2, 3, 4, 5, 6, 7, 8, 9
C_CONST, C_IMAGE, C_CHECKER, C_GRADIENT = 32, 33, 34, 35
V_CONST, V_GRAYSCALE, V_MATH = 64, 65, 67
BG_NONE, BG_CONSTANT, BG_IMAGE, BG_GRADIENT = 0, 1, 2, 3
FLAT_COL_IMG = 4
BAD_ARGUMENT, UNSUPPORTED = -3, -4


def _lib():
    L = crgpu.lib()
    P = C.c_void_p
    L.crgpu_prepare.argtypes = [C.POINTER(crgpu.FlatScene), C.POINTER(P)]
    L.crgpu_prepare.restype = C.c_int
    L.crgpu_prepared_free.argtypes = [P]
    L.crgpu_prepared_free.restype = None
    L.crgpu_prepared_materials.argtypes = [P, P, P, C.c_uint32, C.POINTER(C.c_uint32)]
    L.crgpu_prepared_slab.argtypes = [P, C.POINTER(P), C.POINTER(C.c_size_t)]
    L.crscene_save.argtypes = [C.POINTER(crgpu.FlatScene), C.c_char_p]
    return L


# ---- building shading variants ---------------------------------------------------------------------------------------------------

class Shading:
    """The shading arrays of a flat scene as numpy copies, to edit; .flat() gives a FlatScene with the prefs, camera and geometry of
    `base` (which must outlive it) and these arrays."""

    def __init__(self, base):
        A = crscene.arrays(base)
        self.base = base
        self.materials, self.nodes, self.textures, self.texdata = (A[k].copy() for k in ("materials", "nodes", "textures", "texdata"))
        self.background = int(base.background)
        self._keep = []

    def copy(self):
        s = Shading.__new__(Shading)
        s.base, s.background, s._keep = self.base, self.background, []
        s.materials, s.nodes, s.textures, s.texdata = self.materials.copy(), self.nodes.copy(), self.textures.copy(), self.texdata.copy()
        return s

    def node(self, kind, ins=(), f=(), tex=-1, options=0):
        n = np.zeros(1, dtype=crscene.NODE)
        n["kind"] = kind
        n["in"][0] = list(ins) + [-1] * (3 - len(ins))
        n["f"][0, :len(f)] = f
        n["tex"] = tex
        n["options"] = options
        self.nodes = np.concatenate([self.nodes, n])
        return len(self.nodes) - 1

    def color(self, r, g, b, a=1.0):
        return self.node(C_CONST, f=(r, g, b, a))

    def value(self, v):
        return self.node(V_CONST, f=(v,))

    def texture(self, w, h, ch, is_float=False, seed=0):
        data = np.random.default_rng(seed).random(w * h * ch, dtype=np.float32)
        raw = data.tobytes() if is_float else (data * 255).astype(np.uint8).tobytes()
        t = np.zeros(1, dtype=crscene.TEXTURE)
        t["width"], t["height"], t["channels"], t["is_float"], t["has_alpha"] = w, h, ch, int(is_float), int(not is_float and ch > 3)
        pad = -len(self.texdata) % 16                           # the loader's layout: every texture 16-byte aligned (float texels are read as floats)
        t["data_offset"] = len(self.texdata) + pad
        self.texdata = np.concatenate([self.texdata, np.zeros(pad, np.uint8), np.frombuffer(raw, dtype=np.uint8)])
        self.textures = np.concatenate([self.textures, t])
        return len(self.textures) - 1

    def background_node(self, color, strength=None, offset=0.0):
        s = self.value(1.0) if strength is None else strength
        self.background = self.node(BACKGROUND, (color, s, self.value(offset)))
        return self.background

    def flat(self):
        f = crgpu.FlatScene.from_buffer_copy(self.base)
        f.owner = None
        for name, arr, count in (("materials", self.materials, "material_count"), ("nodes", self.nodes, "node_count"),
                                 ("textures", self.textures, "texture_count"), ("texdata", self.texdata, "texdata_bytes")):
            a = np.ascontiguousarray(arr)
            self._keep.append(a)
            setattr(f, name, a.ctypes.data if len(a) else None)
            setattr(f, count, len(a))
        f.background = self.background
        self._keep.append(f)
        return f


def leaf_color(sh, m):
    """Index of the constant colour node a flat material's leaf reads (None when it has none)."""
    n = sh.nodes
    root = int(sh.materials["bsdf"][m])
    leaf = int(n["in"][root][1]) if n["kind"][root] == MIX else root
    col = int(n["in"][leaf][0])
    if n["kind"][leaf] == PLASTIC:
        col = int(n["in"][int(n["in"][leaf][2])][0])
    return col if col >= 0 and n["kind"][col] == C_CONST else None


def load_golden(name, spp=4, bounces=8):
    here = os.getcwd()
    os.chdir(GOLDEN)
    try:
        flat = crscene.load_json(name + ".json")
    finally:
        os.chdir(here)
    crgpu.lib().crscene_set_config(C.byref(flat), 0, 0, spp, bounces)
    return flat


def upload(flat):
    g = crgpu.GpuScene.__new__(crgpu.GpuScene)
    g.handle = C.c_void_p()
    crgpu._check(crgpu.lib().crgpu_scene_create(C.byref(flat), 0, C.byref(g.handle)), "crgpu_scene_create")
    g.W, g.H, g.samples, g.bounces = flat.prefs.image_width, flat.prefs.image_height, flat.prefs.sample_count, flat.prefs.bounces
    return g


def prepared_shading(flat):
    """(crgpu_prepare's code, kinds, flags, background kind) of a flat scene."""
    L = _lib()
    p = C.c_void_p()
    rc = L.crgpu_prepare(C.byref(flat), C.byref(p))
    if rc:
        return rc, None, None, None
    n = C.c_uint32(0)
    L.crgpu_prepared_materials(p, None, None, 0, C.byref(n))
    kinds, flags = np.zeros(n.value, np.uint32), np.zeros(n.value, np.uint32)
    L.crgpu_prepared_materials(p, kinds.ctypes.data, flags.ctypes.data, n.value, None)
    bg = C.c_uint32(0)
    L.crgpu_prepared_background(p, C.byref(bg))
    L.crgpu_prepared_free(p)
    return 0, kinds, flags, bg.value


def set_shading_rc(g, flat):
    return crgpu.lib().crgpu_scene_set_shading(g.handle, C.byref(flat))


def assert_same_geometry(a, b):
    A, B = crscene.arrays(a), crscene.arrays(b)
    for k in GEOMETRY:
        assert A[k].tobytes() == B[k].tobytes(), f"{k} differ: the variant is not a shading-only edit"
    assert a.material_count == b.material_count


# ---- observing a scene ---------------------------------------------------------------------------------------------------------

def path_states(g, cam, n=4096, seed=11):
    rays = ray_set(cam, n=n, seed=seed)
    st = np.zeros(n, dtype=crgpu.PATH_STATE_DTYPE)
    st["o"], st["d"] = rays[:, :3], rays[:, 3:]
    st["weight"] = 1.0
    st["rng"] = np.random.default_rng(seed).integers(0, 2 ** 63, n, dtype=np.uint64)
    return st


def observe(g, cam):
    """frame, trace_kat records, and shade_rays of a fixed state set at bounces 0 and 1 (K2 -> K4 -> K3) and through the tail kernel"""
    rng = np.random.default_rng(5)
    xyp = np.stack([rng.integers(0, g.W, 512), rng.integers(0, g.H, 512), rng.integers(0, max(1, g.samples), 512)], axis=1)
    out = {"frame": full(g).tobytes(), "kat": g.trace_kat(xyp).tobytes()}
    states = path_states(g, cam)
    for depth, opts in ((0, {}), (1, {}), (1, {"complete_interpreter": 1}), (0, {"tail": 1})):
        res, _perm2, surv, _ = g.shade_rays(states, depth, 8, **opts)
        # the compaction slots (and so perm2) follow the order of K3's atomics; everything else of a state is deterministic: its
        # record, whether it lives on, its direction key, its next state, and L where it holds radiance
        alive = res["alive"] != 0
        has_l = ~alive | (res["next"]["has_l"] != 0)
        nxt = np.zeros_like(res["next"])
        nxt[alive] = res["next"][alive]
        nxt["L"] = np.where(has_l[:, None], res["next"]["L"], np.float32(0))
        out[f"shade{depth}{sorted(opts.items())}"] = (res["rec"].tobytes(), res["alive"].tobytes(), res["dir_key"].tobytes(),
                                                      nxt.tobytes(), surv)
    return out


def assert_same_as_fresh(g, flat_b, cam=None):
    """g (edited) renders, samples and shades exactly as a fresh upload of flat_b, and reports its shading as flat_b's prepare does"""
    cam = cam or crgpu.Camera.from_buffer_copy(flat_b.camera)
    fresh = upload(flat_b)
    try:
        want, want_sh = observe(fresh, cam), fresh.shading()
    finally:
        fresh.close()
    got, sh = observe(g, cam), g.shading()
    for k in want:
        assert got[k] == want[k], f"edited scene differs from the fresh one in {k}"
    rc, kinds, flags, bg = prepared_shading(flat_b)
    assert rc == 0
    assert np.array_equal(sh["kinds"], kinds) and np.array_equal(sh["flags"], flags) and sh["background_kind"] == bg
    assert sh["complete_interpreter"] == want_sh["complete_interpreter"]
    return got


# ---- CPU ---------------------------------------------------------------------------------------------------------------------------

def test_set_shading_rejects_null_arguments():
    L = crgpu.lib()
    flat = crgpu.FlatScene()
    n, bg, x = C.c_uint32(), C.c_uint32(), C.c_int()
    kinds = np.zeros(4, np.uint32)
    assert L.crgpu_scene_set_shading(None, None) == -3
    assert L.crgpu_scene_set_shading(None, C.byref(flat)) == -3
    assert L.crgpu_scene_shading(None, None, None, 0, None, None, None) == -3
    assert L.crgpu_scene_shading(None, kinds.ctypes.data, kinds.ctypes.data, 4, C.byref(n), C.byref(bg), C.byref(x)) == -3


def test_no_shading_edit_without_a_device():
    """Without a GPU no scene exists to edit: creating one fails loudly (CRGPU_ERR_NO_DEVICE), never on the CPU."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    L = crgpu.lib()
    flat = crgpu.FlatScene()
    assert L.crscene_load(C.byref(flat), os.path.join(GOLDEN, "g_single.crscene").encode()) == 0
    h = C.c_void_p()
    assert L.crgpu_scene_create(C.byref(flat), 0, C.byref(h)) == -1
    with pytest.raises(crgpu.CrgpuError):
        crgpu.GpuScene(os.path.join(GOLDEN, "g_single.crscene")).set_shading(flat)
    L.crscene_free(C.byref(flat))


@pytest.fixture(scope="module")
def stub_harness(tmp_path_factory):
    objs = [os.path.join(PKG, "build", n) for n in ("crgpu_api.o", "crgpu_trace.o", "crgpu_shade.o")]
    if not all(os.path.exists(o) for o in objs):
        pytest.skip("c-ray_b200/build/*.o not present (built by nvcc in build())")
    d = tmp_path_factory.mktemp("shading_stub")
    exe = str(d / "shading_harness")
    stub = os.path.join(ROOT, "tests", "stub")
    subprocess.run(["gcc", "-O2", "-c", "-o", str(d / "stub.o"), os.path.join(stub, "cudart_stub.c")], check=True)
    subprocess.run(["gcc", "-O2", "-c", "-I" + os.path.join(ROOT, "include"), "-o", str(d / "h.o"), os.path.join(stub, "shading_harness.c")], check=True)
    subprocess.run(["gcc", "-O2", "-c", "-o", str(d / "io.o"), os.path.join(PKG, "host", "crscene_io.c")], check=True)
    subprocess.run(["g++", "-o", exe, str(d / "h.o")] + objs + [str(d / "io.o"), str(d / "stub.o"), "-lpthread"], check=True)
    return exe, d


def run_stub(stub_harness, a_path, sh):
    exe, d = stub_harness
    b_path = str(d / "b.crscene")
    assert _lib().crscene_save(C.byref(sh.flat()), b_path.encode()) == 0
    r = subprocess.run([exe, a_path, b_path], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=60)
    assert r.returncode == 0, r.stdout
    out = {}
    for line in r.stdout.splitlines():
        key, _, rest = line.partition(" ")
        out[key] = rest
    out["prepare"] = int(out["prepare"].split("=")[1])
    out["set"] = int(out["set"].split("=")[1].split()[0])
    return out


def variants(sh):
    """(name, Shading, expected code) over the golden scene whose shading is sh: accepted edits and every refusal"""
    out = []
    v = sh.copy()
    v.materials["bsdf"][0] = v.node(DIFFUSE, (v.node(C_CHECKER, (v.color(1, 0, 0), v.color(0, 0, 1), v.value(4.0))),))
    v.materials["emission"][0, :3] = (2.0, 1.0, 0.5)
    out.append(("generic", v, 0))
    v = sh.copy()
    v.materials["bsdf"][0] = v.node(METAL, (v.color(0.5, 0.5, 0.5), v.node(V_MATH, (v.value(0.1), v.value(0.2)), options=0)))
    out.append(("xnode", v, 0))
    v = sh.copy()
    v.materials["bsdf"][0] = v.node(DIFFUSE, (v.node(C_IMAGE, tex=v.texture(4, 4, 3)),))
    v.background_node(v.node(C_IMAGE, tex=v.texture(8, 4, 3, True)), offset=30.0)
    out.append(("image", v, 0))
    v = sh.copy()
    v.background_node(v.node(C_GRADIENT, f=(1, 1, 1, 1, 0.5, 0.7, 1, 1)), strength=v.node(V_GRAYSCALE, (v.color(0.5, 0.5, 0.5),)))
    out.append(("composed_background", v, 0))
    v = sh.copy()
    v.textures, v.texdata = v.textures[:0], v.texdata[:0]
    v.nodes["tex"][v.nodes["kind"] == C_IMAGE] = -1
    out.append(("no_textures", v, 0))
    # refusals
    v = sh.copy()
    v.background = len(v.nodes) + 5
    out.append(("background_out_of_range", v, UNSUPPORTED))
    v = sh.copy()
    v.background = v.node(DIFFUSE, (v.color(1, 1, 1),))
    out.append(("background_not_background", v, UNSUPPORTED))
    v = sh.copy()
    v.materials["bsdf"][0] = len(v.nodes) + 1
    out.append(("bsdf_out_of_range", v, UNSUPPORTED))
    v = sh.copy()
    c = v.color(0.5, 0.5, 0.5)
    for _ in range(4):                                          # every checker -> grayscale -> colour step costs a level
        c = v.node(C_CHECKER, (v.color(1, 1, 1), v.color(0, 0, 0), v.node(V_GRAYSCALE, (c,))))
    v.materials["bsdf"][0] = v.node(DIFFUSE, (c,))
    out.append(("colour_too_deep", v, UNSUPPORTED))
    v = sh.copy()
    d = v.node(DIFFUSE, (v.color(0.5, 0.5, 0.5),))
    a = d
    for _ in range(3):
        a = v.node(ADD, (a, d))
    v.materials["bsdf"][0] = a
    out.append(("add_too_deep", v, UNSUPPORTED))
    v = sh.copy()
    v.texture(4, 4, 3)
    v.textures["width"][-1] = 0
    out.append(("texture_zero_width", v, BAD_ARGUMENT))
    v = sh.copy()
    v.texture(4, 4, 3)
    v.textures["data_offset"][-1] = len(v.texdata) - 8
    out.append(("texture_outside_texdata", v, BAD_ARGUMENT))
    v = sh.copy()
    v.materials["bsdf"][0] = v.node(DIFFUSE, (v.node(C_IMAGE, tex=len(v.textures)),))
    out.append(("image_index_out_of_range", v, BAD_ARGUMENT))
    return out


@pytest.mark.parametrize("name", GOLDEN_JSON)
def test_stub_edits_match_prepare(stub_harness, name):
    """Against the stub runtime: every refusal returns crgpu_prepare's code and leaves the scene's shading as it was; every accepted
    edit leaves crgpu_scene_shading equal to B's prepared queries and to a scene created fresh from B."""
    base = load_golden(name)
    exe, d = stub_harness
    a_path = str(d / "a.crscene")
    sh = Shading(base)
    try:
        assert _lib().crscene_save(C.byref(sh.flat()), a_path.encode()) == 0
        for what, v, code in variants(sh):
            out = run_stub(stub_harness, a_path, v)
            assert out["prepare"] == code, (what, out)
            assert out["set"] == code, (what, out)
            if code:
                assert out["edited"] == out["before"], what
            else:
                assert out["edited"] == out["fresh"], what
                n, bg, x, *kf = out["edited"].split()
                assert out["prepared"] == " ".join([n, bg] + kf), what
                if what == "xnode":
                    assert x == "x=1"
        more = sh.copy()
        more.materials = np.concatenate([more.materials, more.materials[:1]])
        out = run_stub(stub_harness, a_path, more)
        assert out["set"] == BAD_ARGUMENT and out["edited"] == out["before"]
    finally:
        crscene.free(base)


# ---- GPU: golden scenes ------------------------------------------------------------------------------------------------------------

def first_flat(sh, kinds):
    return next(i for i, k in enumerate(kinds) if k and leaf_color(sh, i) is not None)


@pytest.mark.gpu
@pytest.mark.parametrize("name", GOLDEN_JSON)
def test_golden_shading_edits(name):
    """One scene through a sequence of edits, each compared with the fresh scene: a flat material recoloured, flat -> generic (a
    checker colour, a mix) and back, emission on and off, image <-> constant colour, the background through constant, gradient,
    image and an interpreted composition, and an X-only node switching the complete interpreter on and off again."""
    base = load_golden(name)
    a = Shading(base)
    A = a.flat()
    g = upload(A)
    try:
        want_a = observe(g, crgpu.Camera.from_buffer_copy(A.camera))
        kinds0 = g.shading()["kinds"]
        x0 = g.shading()["complete_interpreter"]
        m = first_flat(a, kinds0)

        def step(v, check=None):
            f = v.flat()
            g.set_shading(f)
            got = assert_same_as_fresh(g, f)
            if check:
                check(g.shading())
            return got

        v = a.copy()
        col = leaf_color(v, m)
        v.nodes["f"][col, :3] = v.nodes["f"][col, :3][::-1] * np.float32(0.5) + np.float32(0.25)
        got = step(v, lambda s: s["kinds"][m] == kinds0[m] or pytest.fail("recoloured material is no longer flat"))
        assert got["frame"] != want_a["frame"]
        v = a.copy()
        v.materials["bsdf"][m] = v.node(DIFFUSE, (v.node(C_CHECKER, (v.color(1, 0.2, 0), v.color(0, 0.2, 1), v.value(3.0))),))
        step(v, lambda s: s["kinds"][m] == 0 or pytest.fail("checker material still flat"))
        v = a.copy()
        v.materials["bsdf"][m] = v.node(MIX, (v.node(DIFFUSE, (v.color(0.9, 0.1, 0.1),)), v.node(METAL, (v.color(0.8, 0.8, 0.8), v.value(0.2))),
                                              v.value(0.3)))
        step(v, lambda s: s["kinds"][m] == 0 or pytest.fail("mix material still flat"))
        g.set_shading(A)
        assert observe(g, crgpu.Camera.from_buffer_copy(A.camera)) == want_a
        v = a.copy()
        v.materials["emission"][m, :3] = (3.0, 2.0, 1.0)
        step(v)
        v.materials["emission"][m, :3] = 0.0
        step(v)
        v = a.copy()
        v.materials["bsdf"][m] = v.node(DIFFUSE, (v.node(C_IMAGE, tex=v.texture(8, 8, 3, seed=2)),))
        step(v, lambda s: s["flags"][m] & FLAT_COL_IMG or pytest.fail("image colour not folded as one"))
        v.materials["bsdf"][m] = v.node(DIFFUSE, (v.color(0.3, 0.6, 0.9),))
        step(v, lambda s: not s["flags"][m] & FLAT_COL_IMG or pytest.fail("constant colour folded as an image"))
        for kind, make in ((BG_CONSTANT, lambda v: v.color(0.2, 0.4, 0.8)), (BG_GRADIENT, lambda v: v.node(C_GRADIENT, f=(1, 0.9, 0.8, 1, 0.2, 0.3, 1, 1))),
                           (BG_IMAGE, lambda v: v.node(C_IMAGE, tex=v.texture(16, 8, 3, True, seed=3)))):
            v = a.copy()
            v.background_node(make(v), offset=45.0)
            step(v, lambda s: s["background_kind"] == kind or pytest.fail(f"background kind {s['background_kind']}, want {kind}"))
        v = a.copy()
        v.background_node(v.node(C_GRADIENT, f=(1, 1, 1, 1, 0.5, 0.7, 1, 1)), strength=v.node(V_GRAYSCALE, (v.color(0.6, 0.6, 0.6),)))
        step(v, lambda s: s["background_kind"] == BG_NONE or pytest.fail("composed background folded"))
        v = a.copy()
        v.materials["bsdf"][m] = v.node(METAL, (v.color(0.7, 0.7, 0.7), v.node(V_MATH, (v.value(0.05), v.value(0.1)), options=0)))
        step(v, lambda s: s["complete_interpreter"] or pytest.fail("X-only node did not select the complete interpreter"))
        g.set_shading(A)
        assert g.shading()["complete_interpreter"] == x0
        assert observe(g, crgpu.Camera.from_buffer_copy(A.camera)) == want_a
    finally:
        g.close()
        crscene.free(base)


@pytest.mark.gpu
def test_texture_tables_grow_and_shrink():
    """Textures added (0 -> 3) and removed (3 -> 0), texel data larger than the previous block, the same count with other sizes."""
    base = load_golden("g_single")
    a = Shading(base)
    assert len(a.textures) == 0
    A = a.flat()
    g = upload(A)
    try:
        def with_textures(sizes, seed):
            v = a.copy()
            ts = [v.texture(w, h, ch, fl, seed + i) for i, (w, h, ch, fl) in enumerate(sizes)]
            for i in range(len(v.materials)):
                v.materials["bsdf"][i] = v.node(DIFFUSE, (v.node(C_IMAGE, tex=ts[i % (len(ts) - 1)]),))
            v.background_node(v.node(C_IMAGE, tex=ts[-1]))
            return v

        three = with_textures([(4, 4, 3, False), (5, 3, 4, False), (8, 4, 3, True)], 1)
        g.set_shading(three.flat())
        assert_same_as_fresh(g, three.flat())
        g.set_shading(A)
        assert_same_as_fresh(g, A)
        big = with_textures([(64, 64, 4, False), (33, 17, 1, False), (512, 256, 3, True)], 2)
        g.set_shading(three.flat())
        g.set_shading(big.flat())
        assert_same_as_fresh(g, big.flat())
        other = with_textures([(7, 9, 3, False), (2, 2, 4, False), (64, 32, 3, True)], 3)
        g.set_shading(other.flat())
        assert_same_as_fresh(g, other.flat())
    finally:
        g.close()
        crscene.free(base)


@pytest.mark.gpu
def test_refused_edits_leave_the_scene_unchanged():
    base = load_golden("g_nodes")
    a = Shading(base)
    A = a.flat()
    g = upload(A)
    try:
        cam = crgpu.Camera.from_buffer_copy(A.camera)
        before = observe(g, cam)
        sh0 = g.shading()
        more = a.copy()
        more.materials = np.concatenate([more.materials, more.materials[:1]])
        assert set_shading_rc(g, more.flat()) == BAD_ARGUMENT
        refused = [(w, v, c) for w, v, c in variants(a) if c]
        assert len(refused) == 8
        for what, v, code in refused:
            f = v.flat()
            assert prepared_shading(f)[0] == code, what
            assert set_shading_rc(g, f) == code, what
        assert observe(g, cam) == before
        sh = g.shading()
        assert all(np.array_equal(sh[k], sh0[k]) if isinstance(sh[k], np.ndarray) else sh[k] == sh0[k] for k in sh)
    finally:
        g.close()
        crscene.free(base)


# ---- GPU: bundled scenes ---------------------------------------------------------------------------------------------------------

def recolour_doc(name, doc=None):
    """The bundled scene's JSON (or `doc`, an edited copy of it) with other materials and, for hdr, the other HDR environment at
    another offset."""
    d = copy.deepcopy(scene_json(name) if doc is None else doc)
    s = d["scene"]
    if name == "hdr":
        s["ambientColor"]["hdr"] = "HDRs/rooitou_park_1k.hdr"
        s["ambientColor"]["offset"] = 120
        p = s["primitives"]
        p[0]["bsdf"], p[3]["bsdf"] = p[3]["bsdf"], p[0]["bsdf"]
        p[1]["bsdf"], p[2]["bsdf"] = "glass", "plastic"
        p[1]["color"] = {"r": 0.2, "g": 0.9, "b": 0.4}
        for q in p:
            if q["bsdf"] == "emissive":
                q["intensity"] = q["intensity"] * 0.5
    else:
        for i, m in enumerate(s["meshes"]):
            m["bsdf"] = ["metal", "plastic", "glass", "lambertian"][i % 4]
            m["roughness"] = 0.1 * (i % 3)
        p = s["primitives"]
        p[0]["color"] = {"r": 0.3, "g": 0.6, "b": 0.9}
        p[1]["bsdf"] = "metal"
    return d


def bundled_pair(name, W, H, spp, b, doc_b=None):
    a, bb = Loaded(scene_json(name), W, H, spp, b), Loaded(doc_b or recolour_doc(name), W, H, spp, b)
    assert_same_geometry(a.flat, bb.flat)
    return a, bb


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["hdr", "venus", "refraction"])
def test_bundled_shading_edit_renders_as_the_fresh_scene(name):
    W, H, spp = SMALL
    a, b = bundled_pair(name, W, H, spp, BOUNCES[name])
    g = a.upload()
    try:
        before = full(g)
        g.set_shading(b.flat)
        got = assert_same_as_fresh(g, b.flat)
        assert got["frame"] != before.tobytes()
    finally:
        g.close()
        a.free()
        b.free()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GOLDEN_FRAMES))
def test_editing_back_gives_the_committed_frames(name):
    W, H, spp, bounces, mp = GOLDEN_FRAMES[name]
    a, b = bundled_pair(name, W, H, spp, bounces)
    g = a.upload(max_paths=mp)
    try:
        g.set_shading(b.flat)
        changed = full(g)
        g.set_shading(a.flat)
        back = full(g)
        want = json.load(open(DIGESTS))[name]
        assert digest(back) == want
        assert digest(changed) != want
    finally:
        g.close()
        a.free()
        b.free()


# ---- GPU: random worlds ------------------------------------------------------------------------------------------------------------

def shading_variant(doc, d, seed):
    """The world's JSON with every material redrawn (test_loader._rand_bsdf from a second seeded rng, the same number of materials)
    and the background redrawn."""
    from test_loader import _rand_bsdf
    rng = random.Random(7000 + seed)
    images = [p for p in (os.path.join(d, "tex%d.png" % i) for i in range(3)) if os.path.exists(p)] or \
        [os.path.join(GOLDEN, "assets", n) for n in ("gray.png", "rgb.png", "rgba.png")]
    v = copy.deepcopy(doc)
    s = v["scene"]
    for ob in list(s.get("primitives", [])) + list(s.get("meshes", [])):
        if isinstance(ob.get("material"), list):
            ob["material"] = [_rand_bsdf(rng, images) for _ in ob["material"]]
        elif "material" in ob:
            ob["material"] = _rand_bsdf(rng, images)
        else:
            ob["bsdf"] = rng.choice(["lambertian", "metal", "glass", "plastic", "emissive"])
            ob["color"] = [round(rng.random(), 3) for _ in range(3)]
            ob["intensity"] = rng.choice([0.5, 3.0])
    amb = [{"down": [round(rng.random(), 3) for _ in range(3)], "up": [round(rng.random(), 3) for _ in range(3)]}, {}]
    if os.path.exists(os.path.join(d, "env.hdr")):
        amb.append({"hdr": "env.hdr", "offset": rng.choice([15, 90, -60])})
    s["ambientColor"] = rng.choice(amb)
    return v


def _world_seeds():
    from test_gpu_worlds import SEEDS
    return SEEDS


@pytest.mark.gpu
@pytest.mark.parametrize("seed", _world_seeds())
def test_world_shading_edit(seed, tmp_path):
    """A world edited with its shading variant equals the variant loaded fresh; a variant crgpu_prepare refuses is refused with the
    same code and the world keeps rendering its own bits."""
    from test_gpu_worlds import World
    w = World(str(tmp_path), seed)
    if w.refusal:
        pytest.skip(f"world {seed} is refused by the device: {w.refusal}")
    a = w.loaded()
    b = Loaded(shading_variant(w.doc, w.dir, seed), *w.cfg, cwd=w.dir, asset_path=w.dir)
    g = a.upload()
    try:
        assert_same_geometry(a.flat, b.flat)
        want_a = full(g)
        rc = prepared_shading(b.flat)[0]
        if rc:
            assert set_shading_rc(g, b.flat) == rc
            assert full(g).tobytes() == want_a.tobytes()
        else:
            g.set_shading(b.flat)
            assert_same_as_fresh(g, b.flat)
            g.set_shading(a.flat)
            assert full(g).tobytes() == want_a.tobytes()
    finally:
        g.close()
        a.free()
        b.free()


# ---- GPU: composition, a stopped render ------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("order", ["shading_first", "shading_last"])
def test_shading_edit_combined_with_the_other_edits(order):
    """Other materials, a moved camera, moved instances and deformed teapots, in either order, render as the fresh load of the JSON
    with all of them."""
    from test_gpu_mesh_edit import Assets, LoadedFrom, changed_meshes, deform_obj
    doc = scene_json("refraction")
    cfg = (*SMALL, BOUNCES["refraction"])
    assets = Assets()
    assets.write("teapot.obj", deform_obj(assets.original("teapot.obj"), seed=9))
    doc_b = edited(recolour_doc("refraction"), STEP["refraction"])
    a, b = Loaded(doc, *cfg), LoadedFrom(doc_b, assets.dir, *cfg)
    g = a.upload()
    try:
        ch = changed_meshes(a, b)
        assert ch
        if order == "shading_first":
            g.set_shading(b.flat)
        g.set_meshes(b.flat, ch)
        g.set_camera(b.camera)
        g.set_instances(b.instances)
        if order != "shading_first":
            g.set_shading(b.flat)
        assert_same_as_fresh(g, b.flat, b.camera)
    finally:
        g.close()
        a.free()
        b.free()
        assets.close()


@pytest.mark.gpu
def test_shading_edit_after_a_stopped_render():
    W, H, spp, bounces, mp = GOLDEN_FRAMES["hdr"]
    a, b = bundled_pair("hdr", W, H, spp, bounces)
    fresh = b.upload(max_paths=mp)
    want = full(fresh)
    fresh.close()
    g = a.upload(max_paths=mp)
    try:
        g.enable_stop()
        g.clear()
        g.render_tile(0, 0, g.W, g.H, flags=crgpu.FLAG_ASYNC)
        g.request_stop()
        g.set_shading(b.flat)
        g.clear_stop()
        g.clear()
        st = g.render_tile(0, 0, g.W, g.H)
        assert st["stopped"] is False
        assert g.read().tobytes() == want.tobytes()
    finally:
        g.close()
        a.free()
        b.free()


# ---- GPU: isolation and repetition ---------------------------------------------------------------------------------------------

def slab_sum(L, p):
    ptr, n = C.c_void_p(), C.c_size_t()
    assert L.crgpu_prepared_slab(p, C.byref(ptr), C.byref(n)) == 0
    return hashlib.sha256(C.string_at(ptr, n.value)).hexdigest()


@pytest.mark.gpu
def test_edit_applies_to_one_scene_only():
    """Two scenes created from one crgpu_prepared: editing one leaves the other, a scene created later, and the slab unedited."""
    base = load_golden("g_nodes")
    a = Shading(base)
    A = a.flat()
    v = a.copy()
    v.background_node(v.color(0.9, 0.3, 0.1))
    v.materials["emission"][0, :3] = 1.5
    L = _lib()
    p = C.c_void_p()
    assert L.crgpu_prepare(C.byref(A), C.byref(p)) == 0
    scenes = []
    try:
        sum0 = slab_sum(L, p)
        cfg = (A.prefs.image_width, A.prefs.image_height, A.prefs.sample_count, A.prefs.bounces)
        for _ in range(2):
            g = crgpu.GpuScene(None, *cfg, prepared=p.value)
            g.W, g.H = cfg[:2]
            scenes.append(g)
        want = full(scenes[0])
        scenes[0].set_shading(v.flat())
        assert full(scenes[0]).tobytes() != want.tobytes()
        assert full(scenes[1]).tobytes() == want.tobytes()
        late = crgpu.GpuScene(None, *cfg, prepared=p.value)
        late.W, late.H = cfg[:2]
        scenes.append(late)
        assert full(late).tobytes() == want.tobytes()
        assert slab_sum(L, p) == sum0
    finally:
        for g in scenes:
            g.close()
        L.crgpu_prepared_free(p)
        crscene.free(base)


@pytest.mark.gpu
def test_alternating_edits_stay_exact_and_do_not_leak():
    """20 edits alternating A and B (B with a 2048 x 1024 float environment, 24 MB of texels) stay exact, and the device's free
    memory does not fall from edit to edit once both blocks are in the cache."""
    import torch
    base = load_golden("g_nodes")
    a = Shading(base)
    A = a.flat()
    v = a.copy()
    v.background_node(v.node(C_IMAGE, tex=v.texture(2048, 1024, 3, True, seed=4)), offset=10.0)
    B = v.flat()
    g = upload(A)
    fresh_b = upload(B)
    try:
        want = {0: full(g).tobytes(), 1: full(fresh_b).tobytes()}
        fresh_b.close()
        torch.cuda.init()
        free = []
        for k in range(20):
            g.set_shading(B if k % 2 == 0 else A)
            assert full(g).tobytes() == want[(k + 1) % 2], f"edit {k}"
            free.append(torch.cuda.mem_get_info()[0])
        assert min(free[2:]) >= free[1], free
    finally:
        g.close()
        crscene.free(base)
