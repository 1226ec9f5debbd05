"""Deforming the meshes of a resident GPU scene (crgpu_scene_set_meshes, include/crgpu.h).

Each comparison has two sides: A is the original scene uploaded and then edited with set_meshes(B.flat, changed meshes); B is the
deformed scene loaded fresh (its JSON with a deformed copy of an OBJ, whose `v` — or `vn` / `vt` — lines alone are rewritten with
round-trip-exact floats) and uploaded.  Both must render the same bits and trace a fixed ray set (count = 1) with the same records
and P/T/S/I counts, which pins the rebuilt tree's shape, its BFS packing and the slot order.

CPU: argument checks of the new entry point.  GPU: everything else.
"""
import copy
import ctypes as C
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import crgpu
import crscene
from conftest import GOLDEN, ROOT
from test_gpu_scene_edit import (BOUNCES, DIGESTS, GOLDEN_FRAMES, REFDIR, SMALL, STEP, Loaded, assert_same_as_fresh, digest, edited,
                                 full, ray_set, scene_json, sphere_scene, traced)

BOUNCES = dict(BOUNCES, statues=30, scene=50)


# ---- CPU -----------------------------------------------------------------------------------------------------------------------

def test_set_meshes_rejects_null_arguments():
    L = crgpu.lib()
    flat = crgpu.FlatScene()
    idx = np.zeros(1, np.uint32)
    assert L.crgpu_scene_set_meshes(None, None, None, 0) == -3
    assert L.crgpu_scene_set_meshes(None, C.byref(flat), idx.ctypes.data, 1) == -3


def test_no_mesh_edit_without_a_device():
    """Without a GPU no scene exists to deform: creating one fails loudly (CRGPU_ERR_NO_DEVICE), never on the CPU."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    L = crgpu.lib()
    h = C.c_void_p()
    flat = crgpu.FlatScene()
    assert L.crscene_load(C.byref(flat), os.path.join(GOLDEN, "g_single.crscene").encode()) == 0
    assert L.crgpu_scene_create(C.byref(flat), 0, C.byref(h)) == -1
    with pytest.raises(crgpu.CrgpuError):
        crgpu.GpuScene(os.path.join(GOLDEN, "g_single.crscene")).set_meshes(flat, [0])
    L.crscene_free(C.byref(flat))


def test_write_back_round_trips():
    cwd = os.getcwd()
    os.chdir(GOLDEN)
    try:
        flat = crscene.load_json("g_meshmat.json")
    finally:
        os.chdir(cwd)
    try:
        v = crscene.arrays(flat)["vertices"]
        crscene.write_back(flat, "vertices", v * 2.0)
        assert np.array_equal(crscene.arrays(flat)["vertices"], (v * 2.0).astype(np.float32))
        polys = crscene.arrays(flat)["polys"]
        polys["material"][:] = 0
        crscene.write_back(flat, "polys", polys)
        assert crscene.arrays(flat)["polys"].tobytes() == polys.tobytes()
        with pytest.raises(ValueError):
            crscene.write_back(flat, "meshes", crscene.arrays(flat)["meshes"])
        with pytest.raises(ValueError):
            crscene.write_back(flat, "vertices", np.zeros((len(v) + 1, 3)))
    finally:
        crscene.free(flat)


# ---- helpers ---------------------------------------------------------------------------------------------------------------------

def fmt(x):
    return repr(float(np.float32(x)))


def deform_obj(text, kind="v", seed=1, amp=0.01, fn=None):
    """OBJ text with the `kind` lines ("v", "vn" or "vt") rewritten: a seeded smooth displacement of `amp` times the extent of those
    coordinates, or fn(array) -> array.  Every other line stays byte for byte."""
    lines = text.split("\n")
    rows = [i for i, ln in enumerate(lines) if ln.split(" ", 1)[0] == kind]
    vals = np.array([[float(t) for t in lines[i].split()[1:]] for i in rows], dtype=np.float32)
    if fn is not None:
        new = np.asarray(fn(vals), dtype=np.float32)
    else:
        rng = np.random.default_rng(seed)
        ext = float(np.ptp(vals, axis=0).max()) or 1.0
        k = rng.uniform(0.5, 2.0, vals.shape[1]) * 2 * np.pi / ext
        ph = rng.uniform(0, 2 * np.pi, vals.shape[1])
        d = amp * ext * np.sin(vals.astype(np.float64)[:, ::-1] * k + ph)
        new = (vals + d).astype(np.float32)
    for i, r in zip(rows, new):
        lines[i] = kind + " " + " ".join(fmt(x) for x in r)
    return "\n".join(lines)


class Assets:
    """A temporary copy of the bundled input/ directory (symbolic links) in which some OBJ files are replaced."""

    def __init__(self):
        self.dir = tempfile.mkdtemp(prefix="crgpu_mesh_edit_")
        src = os.path.join(REFDIR, "input")
        for e in os.listdir(src):
            os.symlink(os.path.join(src, e), os.path.join(self.dir, e))

    def original(self, name):
        return open(os.path.join(REFDIR, "input", name)).read()

    def write(self, name, text):
        sub = os.path.dirname(name)
        if sub and os.path.islink(os.path.join(self.dir, sub)):
            real = os.readlink(os.path.join(self.dir, sub))
            os.unlink(os.path.join(self.dir, sub))
            os.mkdir(os.path.join(self.dir, sub))
            for e in os.listdir(real):
                os.symlink(os.path.join(real, e), os.path.join(self.dir, sub, e))
        path = os.path.join(self.dir, name)
        if os.path.lexists(path):
            os.unlink(path)
        with open(path, "w") as f:
            f.write(text)

    def close(self):
        shutil.rmtree(self.dir, ignore_errors=True)


class LoadedFrom(Loaded):
    """Loaded, with assets from another directory (the textures named inside node graphs still resolve against the bundled input/)."""

    def __init__(self, doc, asset_dir, W, H, spp, b):
        cwd = os.getcwd()
        os.chdir(REFDIR)
        try:
            self.flat = crscene.load_json_buf(json.dumps(doc), asset_dir)
        finally:
            os.chdir(cwd)
        crgpu.lib().crscene_set_config(C.byref(self.flat), W, H, spp, b)
        self.cfg = (W, H, spp, b)
        self.camera = crgpu.Camera.from_buffer_copy(self.flat.camera)
        self.instances = crscene.arrays(self.flat)["instances"]


def changed_meshes(a, b):
    """Meshes whose polys, or the vertices, normals or texcoords they index, differ between the flat scenes a and b."""
    A, B = crscene.arrays(a.flat), crscene.arrays(b.flat)
    for k in ("meshes", "polys", "bvhs"):
        assert len(A[k]) == len(B[k])
    out = []
    for m, mesh in enumerate(A["meshes"]):
        sl = slice(int(mesh["poly_offset"]), int(mesh["poly_offset"] + mesh["poly_count"]))
        pa, pb = A["polys"][sl], B["polys"][sl]
        same = pa.tobytes() == pb.tobytes()
        for name, col in (("vertices", "v"), ("normals", "n"), ("texcoords", "t")):
            if name == "texcoords" and mesh["texcoord_count"] == 0:
                continue                                            # a mesh without texcoords reads none
            idx = pa[col].reshape(-1)
            idx = idx[(idx >= 0) & (idx < len(A[name]))]
            same = same and A[name][idx].tobytes() == B[name][idx].tobytes()
        if not same:
            out.append(m)
    return out


def deformed(doc, files, cfg, kind="v", seed=1, fn=None):
    """(A, B, assets, changed): doc loaded as is and with each OBJ of `files` deformed."""
    assets = Assets()
    for i, name in enumerate(files):
        assets.write(name, deform_obj(assets.original(name), kind, seed + i, fn=fn))
    a, b = Loaded(doc, *cfg), LoadedFrom(doc, assets.dir, *cfg)
    return a, b, assets, changed_meshes(a, b)


def check(doc, files, name=None, kind="v", cfg=None, seed=1, fn=None, repeat=1):
    cfg = cfg or (*SMALL, BOUNCES[name])
    a, b, assets, ch = deformed(doc, files, cfg, kind, seed, fn)
    g = a.upload()
    try:
        assert ch, "the deformation changed no mesh"
        for _ in range(repeat):
            g.set_meshes(b.flat, ch)
        assert_same_as_fresh(g, b, ray_set(b.camera))
    finally:
        g.close()
        a.free()
        b.free()
        assets.close()
    return ch


# ---- GPU: bundled scenes -----------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name,files,want", [
    ("hdr", ["venusscaled.obj"], [1]),                     # Venus, 274k triangles
    ("hdr", ["shapes/gridplane.obj"], [0]),                # the textured grid plane
    ("statues", ["venusscaled.obj"], [1]),                 # Venus under 55 instances: every instance box and ray offset changes
    ("scene", ["teapot.obj"], None),                       # a teapot with 3 instances
    ("venus", ["teapot.obj", "torus.obj"], None),          # several meshes in one call
])
def test_deformed_mesh_renders_as_the_fresh_scene(name, files, want):
    ch = check(scene_json(name), files, name)
    if want is not None:
        assert ch == want
    if name == "venus":
        assert len(ch) >= 3


@pytest.mark.gpu
def test_normal_only_edit():
    check(scene_json("hdr"), ["venusscaled.obj"], "hdr", kind="vn", fn=lambda n: n[:, [1, 2, 0]] * np.float32(0.9))


@pytest.mark.gpu
def test_uv_only_edit():
    check(scene_json("hdr"), ["shapes/gridplane.obj"], "hdr", kind="vt", fn=lambda t: t * np.float32(0.5) + np.float32(0.25))


@pytest.mark.gpu
def test_material_reassignment_within_the_mesh_range():
    """Per-poly materials changed in the flat scene (the tree does not change): the shading records and keys follow."""
    doc = scene_json("scene")
    cfg = (*SMALL, BOUNCES["scene"])
    a, b = Loaded(doc, *cfg), Loaded(doc, *cfg)
    A = crscene.arrays(a.flat)
    m = next(i for i, x in enumerate(A["meshes"]) if x["material_count"] >= 2)
    mesh = A["meshes"][m]
    polys = A["polys"].copy()
    sl = slice(int(mesh["poly_offset"]), int(mesh["poly_offset"] + mesh["poly_count"]))
    polys["material"][sl] = (polys["material"][sl] + 1) % mesh["material_count"]
    crscene.write_back(b.flat, "polys", polys)
    g = a.upload()
    try:
        assert changed_meshes(a, b) == [m]
        g.set_meshes(b.flat, [m])
        assert_same_as_fresh(g, b, ray_set(b.camera))
    finally:
        g.close()
        a.free()
        b.free()


# ---- GPU: tree shape changes on a generated mesh -------------------------------------------------------------------------------

def tri_obj(centres, size=3.0):
    """An OBJ of one triangle per centre (same shape each), with teapot.mtl's material."""
    out = ["mtllib teapot.mtl", "o gen", "vn 0.0 0.0 1.0"]
    for c in centres:
        for d in ((0.0, 0.0, 0.0), (size, 0.0, 0.0), (0.0, size, size * 0.5)):
            out.append("v " + " ".join(fmt(c[k] + d[k]) for k in range(3)))
    out.append("usemtl " + [ln.split()[1] for ln in open(os.path.join(REFDIR, "input", "teapot.mtl")) if ln.startswith("newmtl")][0])
    out += [f"f {3 * i + 1}//1 {3 * i + 2}//1 {3 * i + 3}//1" for i in range(len(centres))]
    return "\n".join(out) + "\n"


def gen_scene(objs):
    """Two sphere instances and one instance of each generated mesh, in the region of the bundled refraction scene."""
    meshes = [{"fileName": f, "bsdf": "lambertian", "instances": [{"transforms": [{"type": "translate", "x": 900.0 + 40 * i, "y": 350.0, "z": 1100.0}]}]}
              for i, f in enumerate(objs)]
    return sphere_scene(np.array([[800.0, 300.0, 1000.0], [1000.0, 400.0, 1200.0]]), meshes=meshes)


def check_gen(before, after, cfg=(160, 90, 2, 8)):
    """Each of `before` / `after`: {obj name: centres}; A loads `before`, B `after`."""
    sa, sb = Assets(), Assets()
    for n, c in before.items():
        sa.write(n, tri_obj(c))
    for n, c in after.items():
        sb.write(n, tri_obj(c))
    doc = gen_scene(sorted(before))
    a, b = LoadedFrom(doc, sa.dir, *cfg), LoadedFrom(doc, sb.dir, *cfg)
    g = a.upload()
    try:
        ch = changed_meshes(a, b)
        g.set_meshes(b.flat, ch)
        assert_same_as_fresh(g, b, ray_set(b.camera))
        return crscene.arrays(a.flat)["bvhs"], crscene.arrays(b.flat)["bvhs"]
    finally:
        g.close()
        a.free()
        b.free()
        sa.close()
        sb.close()


def spread_tris(n, seed, scale=30.0):
    return np.round(np.random.default_rng(seed).uniform(-scale, scale, (n, 3)), 3)


@pytest.mark.gpu
def test_single_leaf_mesh_grows_into_a_tree():
    """Eight same-shaped triangles at one place upload as one leaf; spread out, the tree has internal nodes in the mesh's new region."""
    ba, bb = check_gen({"gen.obj": np.zeros((8, 3))}, {"gen.obj": spread_tris(8, 1)})
    assert ba["node_count"][0] == 1 and bb["node_count"][0] > 1


@pytest.mark.gpu
def test_tree_collapses_into_a_single_leaf():
    ba, bb = check_gen({"gen.obj": spread_tris(8, 2)}, {"gen.obj": np.zeros((8, 3))})
    assert ba["node_count"][0] > 1 and bb["node_count"][0] == 1


@pytest.mark.gpu
def test_tree_with_more_internal_nodes_than_uploaded():
    """40 triangles in two tight clusters grow to 40 spread ones: more pair nodes than the upload gave the mesh."""
    clusters = np.concatenate([np.zeros((20, 3)), np.full((20, 3), 50.0)]) + spread_tris(40, 3, 0.01)
    ba, bb = check_gen({"gen.obj": clusters}, {"gen.obj": spread_tris(40, 4)})
    assert bb["node_count"][0] > ba["node_count"][0]


@pytest.mark.gpu
def test_two_meshes_edited_in_separate_calls():
    """The edit block grows on the second call; the mesh of the first call still renders as deformed."""
    doc = scene_json("hdr")
    cfg = (*SMALL, BOUNCES["hdr"])
    assets = Assets()
    assets.write("venusscaled.obj", deform_obj(assets.original("venusscaled.obj"), seed=5))
    assets.write("shapes/gridplane.obj", deform_obj(assets.original("shapes/gridplane.obj"), seed=6))
    a, b = Loaded(doc, *cfg), LoadedFrom(doc, assets.dir, *cfg)
    g = a.upload()
    try:
        assert changed_meshes(a, b) == [0, 1]
        g.set_meshes(b.flat, [1])
        g.set_meshes(b.flat, [0])
        assert_same_as_fresh(g, b, ray_set(b.camera))
    finally:
        g.close()
        a.free()
        b.free()
        assets.close()


# ---- GPU: editing back, repeating, combining ------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GOLDEN_FRAMES))
def test_editing_back_gives_the_committed_frames(name):
    doc = scene_json(name)
    W, H, spp, bounces, mp = GOLDEN_FRAMES[name]
    files = ["venusscaled.obj"] if name == "hdr" else ["teapot.obj", "torus.obj"]
    a, b, assets, ch = deformed(doc, files, (W, H, spp, bounces))
    g = a.upload(max_paths=mp)
    try:
        g.set_meshes(b.flat, ch)
        moved = full(g)
        g.set_meshes(a.flat, ch)
        back = full(g)
        want = json.load(open(DIGESTS))[name]
        assert digest(back) == want
        assert digest(moved) != want
    finally:
        g.close()
        a.free()
        b.free()
        assets.close()


@pytest.mark.gpu
def test_repeated_mesh_edit_is_idempotent():
    check(scene_json("scene"), ["teapot.obj"], "scene", repeat=3)


@pytest.mark.gpu
@pytest.mark.parametrize("order", ["meshes_first", "instances_first"])
def test_mesh_edit_combined_with_instance_edit(order):
    """Deformed teapots and moved instances, in either order, render as the fresh load of the JSON with both changes."""
    doc = scene_json("refraction")
    cfg = (*SMALL, BOUNCES["refraction"])
    assets = Assets()
    assets.write("teapot.obj", deform_obj(assets.original("teapot.obj"), seed=9))
    a, b = Loaded(doc, *cfg), LoadedFrom(edited(doc, STEP["refraction"]), assets.dir, *cfg)
    g = a.upload()
    try:
        ch = changed_meshes(a, b)
        assert ch
        if order == "meshes_first":
            g.set_meshes(b.flat, ch)
        g.set_camera(b.camera)
        g.set_instances(b.instances)
        if order != "meshes_first":
            g.set_meshes(b.flat, ch)
        assert_same_as_fresh(g, b, ray_set(b.camera))
    finally:
        g.close()
        a.free()
        b.free()
        assets.close()


@pytest.mark.gpu
def test_mesh_edit_after_a_stopped_render():
    doc = scene_json("hdr")
    W, H, spp, bounces, mp = GOLDEN_FRAMES["hdr"]
    a, b, assets, ch = deformed(doc, ["venusscaled.obj"], (W, H, spp, bounces))
    fresh = b.upload(max_paths=mp)
    want = full(fresh)
    fresh.close()
    g = a.upload(max_paths=mp)
    try:
        g.enable_stop()
        g.clear()
        g.render_tile(0, 0, g.W, g.H, flags=crgpu.FLAG_ASYNC)
        g.request_stop()
        g.set_meshes(b.flat, ch)
        g.clear_stop()
        g.clear()
        st = g.render_tile(0, 0, g.W, g.H)
        assert st["stopped"] is False
        assert g.read().tobytes() == want.tobytes()
    finally:
        g.close()
        a.free()
        b.free()
        assets.close()


# ---- GPU: staged nodes, a large mesh --------------------------------------------------------------------------------------------

STAGED = r"""
import sys
sys.path[:0] = [{pkg!r}, {tests!r}]
import test_gpu_mesh_edit as T
from test_gpu_trace import VARIANTS
doc = T.scene_json("hdr")
a, b, assets, ch = T.deformed(doc, ["venusscaled.obj", "shapes/gridplane.obj"], (320, 240, 2, 32))
g = a.upload()
fresh = b.upload()
g.set_meshes(b.flat, ch)
rays = T.ray_set(b.camera, n=70000)
for kn in VARIANTS:
    r1, r2 = g.trace_rays(rays, **kn), fresh.trace_rays(rays, **kn)
    assert r1[0].tobytes() == r2[0].tobytes(), kn
    assert r1[2] == r2[2], kn
    if kn.get("count"):
        assert T.traced(g, rays)[1:] == T.traced(fresh, rays)[1:], kn
assert T.full(g).tobytes() == T.full(fresh).tobytes()
g.close(); fresh.close(); assets.close()
print("staged ok")
"""


@pytest.mark.gpu
@pytest.mark.parametrize("stage", [128, 1024])
def test_edited_meshes_with_staged_nodes(stage):
    """CRGPU_TRACE_STAGE (read at prepare time) stages the top nodes of every BVH; a mesh edit rewrites the mesh's staged prefix."""
    scene_json("hdr")
    env = dict(os.environ, CRGPU_TRACE_STAGE=str(stage))
    code = STAGED.format(pkg=os.path.join(ROOT, "c-ray_b200"), tests=os.path.join(ROOT, "tests"))
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0 and "staged ok" in r.stdout, r.stdout[-3000:]


def grid_obj(k, z):
    """A k x k grid of quads as 2 k^2 triangles, heights z (k+1 x k+1)."""
    xs = np.arange(k + 1, dtype=np.float32) * np.float32(0.5)
    out = ["mtllib teapot.mtl", "o grid", "vn 0.0 0.0 1.0"]
    X, Y = np.meshgrid(xs, xs, indexing="ij")
    out += ["v %s %s %s" % (fmt(x), fmt(y), fmt(h)) for x, y, h in zip(X.ravel(), Y.ravel(), z.ravel())]
    out.append("usemtl " + [ln.split()[1] for ln in open(os.path.join(REFDIR, "input", "teapot.mtl")) if ln.startswith("newmtl")][0])
    i = np.arange(k)[:, None] * (k + 1) + np.arange(k)[None, :] + 1
    a, b, c, d = i.ravel(), (i + 1).ravel(), (i + k + 1).ravel(), (i + k + 2).ravel()
    out += [f"f {p}//1 {q}//1 {r}//1\nf {q}//1 {s}//1 {r}//1" for p, q, r, s in zip(a, b, c, d)]
    return "\n".join(out) + "\n"


@pytest.mark.gpu
def test_million_triangle_mesh():
    k = 708                                                     # 2 * 708^2 = 1,002,528 triangles
    xs = np.arange(k + 1) / k
    X, Y = np.meshgrid(xs, xs, indexing="ij")
    z0 = np.zeros_like(X)
    z1 = 3.0 * np.sin(6.0 * X) * np.cos(5.0 * Y)
    sa, sb = Assets(), Assets()
    sa.write("grid.obj", grid_obj(k, z0))
    sb.write("grid.obj", grid_obj(k, z1))
    doc = gen_scene(["grid.obj"])
    cfg = (64, 36, 1, 4)
    a, b = LoadedFrom(doc, sa.dir, *cfg), LoadedFrom(doc, sb.dir, *cfg)
    g = a.upload()
    fresh = b.upload()
    try:
        assert crscene.arrays(a.flat)["meshes"]["poly_count"][0] == 2 * k * k
        g.set_meshes(b.flat, [0])
        rays = ray_set(b.camera, n=50000)
        got, want = traced(g, rays), traced(fresh, rays)
        assert got[0].tobytes() == want[0].tobytes()
        assert got[1:] == want[1:]
    finally:
        g.close()
        fresh.close()
        a.free()
        b.free()
        sa.close()
        sb.close()


# ---- GPU: rejected edits, the prepared slab ----------------------------------------------------------------------------------

@pytest.mark.gpu
def test_rejected_mesh_edits_leave_the_scene_unchanged():
    doc = scene_json("hdr")
    cfg = (*SMALL, BOUNCES["hdr"])
    a, b = Loaded(doc, *cfg), Loaded(doc, *cfg)
    L = crgpu.lib()
    g = a.upload()

    def rc(meshes):
        idx = np.asarray(meshes, np.uint32)
        return L.crgpu_scene_set_meshes(g.handle, C.byref(b.flat), idx.ctypes.data, len(idx))

    try:
        before = full(g)
        B = crscene.arrays(b.flat)
        venus = B["meshes"][1]
        sl = slice(int(venus["poly_offset"]), int(venus["poly_offset"] + venus["poly_count"]))
        meshes = B["meshes"].copy()
        meshes["material_count"][1] += 1
        C.memmove(b.flat.meshes, meshes.ctypes.data, meshes.nbytes)
        assert rc([1]) == -3                                        # a changed mesh record
        C.memmove(b.flat.meshes, B["meshes"].ctypes.data, B["meshes"].nbytes)
        for col, count in (("v", len(B["vertices"])), ("t", len(B["texcoords"])), ("n", len(B["normals"]))):
            polys = B["polys"].copy()
            m = 0 if col == "t" else 1                              # the grid plane has texcoords; Venus has normals
            s0 = int(B["meshes"][m]["poly_offset"])
            polys[col][s0, 1] = count
            crscene.write_back(b.flat, "polys", polys)
            assert rc([m]) == -3, col                               # an index out of range
        polys = B["polys"].copy()
        polys["material"][sl.start] = venus["material_count"]
        crscene.write_back(b.flat, "polys", polys)
        assert rc([1]) == -3                                        # a material outside the mesh's range
        crscene.write_back(b.flat, "polys", B["polys"])
        assert rc([2]) == -3                                        # a mesh out of range
        assert rc([1, 1]) == -3                                     # a mesh listed twice
        assert full(g).tobytes() == before.tobytes()
    finally:
        g.close()
        a.free()
        b.free()


@pytest.mark.gpu
def test_collapsed_mesh_is_refused():
    """20 triangles collapsed to one point: every split sends everything left, and the tree needs more than 2n - 1 nodes."""
    assets = Assets()
    assets.write("gen.obj", tri_obj(spread_tris(20, 11)))
    doc = gen_scene(["gen.obj"])
    cfg = (160, 90, 2, 8)
    a, b = LoadedFrom(doc, assets.dir, *cfg), LoadedFrom(doc, assets.dir, *cfg)
    g = a.upload()
    try:
        before = full(g)
        V = crscene.arrays(b.flat)["vertices"].copy()
        V[:] = V[0]
        crscene.write_back(b.flat, "vertices", V)
        idx = np.zeros(1, np.uint32)
        assert crgpu.lib().crgpu_scene_set_meshes(g.handle, C.byref(b.flat), idx.ctypes.data, 1) == -4   # CRGPU_ERR_UNSUPPORTED
        assert full(g).tobytes() == before.tobytes()
    finally:
        g.close()
        a.free()
        b.free()
        assets.close()


@pytest.mark.gpu
def test_prepared_slab_stays_unedited():
    """A second scene created from the same crgpu_prepared after an edit renders the unedited frame."""
    doc = scene_json("hdr")
    cfg = (*SMALL, BOUNCES["hdr"])
    a, b, assets, ch = deformed(doc, ["venusscaled.obj"], cfg)
    L = crgpu.lib()
    L.crgpu_prepare.argtypes = [C.POINTER(crgpu.FlatScene), C.POINTER(C.c_void_p)]
    L.crgpu_prepared_free.argtypes = [C.c_void_p]
    L.crgpu_prepared_free.restype = None
    p = C.c_void_p()
    assert L.crgpu_prepare(C.byref(a.flat), C.byref(p)) == 0
    scenes = []
    try:
        W, H, spp, bounces = cfg
        for _ in range(2):
            g = crgpu.GpuScene(None, W, H, spp, bounces, prepared=p.value)
            g.W, g.H = W, H
            scenes.append(g)
        want = full(scenes[0])
        scenes[0].set_meshes(b.flat, ch)
        assert full(scenes[0]).tobytes() != want.tobytes()
        late = crgpu.GpuScene(None, W, H, spp, bounces, prepared=p.value)
        late.W, late.H = W, H
        scenes.append(late)
        assert full(late).tobytes() == want.tobytes()
        assert full(scenes[1]).tobytes() == want.tobytes()
    finally:
        for g in scenes:
            g.close()
        L.crgpu_prepared_free(p)
        a.free()
        b.free()
        assets.close()
