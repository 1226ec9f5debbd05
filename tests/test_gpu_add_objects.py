"""Adding meshes and spheres to a resident GPU scene between renders (crgpu_scene_add_objects, include/crgpu.h).

The target is exact: a scene A given a grown scene B (A's JSON with more meshes and spheres, loaded fresh) renders, traces and shades
the same bits as B uploaded fresh, including the ray records with their shading keys and the P/T/S/I counts of the instrumented
traversal.  New meshes go behind A's meshes in the JSON and new spheres behind A's spheres, which is how a grown scene extends A's
objects; the loader then moves every sphere's material behind the new meshes' materials.

CPU: argument checks of the new entry point.  GPU: everything else.
"""
import copy
import ctypes as C
import json
import os

import numpy as np
import pytest

import crgpu
import crscene
from conftest import GOLDEN
from test_gpu_instance_list import DUP, GEN, objects, scattered, translate
from test_gpu_mesh_edit import Assets, LoadedFrom, deform_obj, fmt, grid_obj
from test_gpu_scene_edit import (BOUNCES, DIGESTS, GOLDEN_FRAMES, REFDIR, SMALL, STEP, Loaded, assert_same_as_fresh, digest, full, ray_set,
                                 scene_json, sphere_scene, spread, teapots, traced)

BAD_ARGUMENT, UNSUPPORTED = -3, -4


# ---- CPU -----------------------------------------------------------------------------------------------------------------------

def test_entry_point_rejects_null_arguments():
    L = crgpu.lib()
    flat = crgpu.FlatScene()
    assert L.crgpu_scene_add_objects(None, None) == BAD_ARGUMENT
    assert L.crgpu_scene_add_objects(None, C.byref(flat)) == BAD_ARGUMENT


def test_no_scene_to_grow_without_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    with pytest.raises(crgpu.CrgpuError):
        crgpu.GpuScene(os.path.join(GOLDEN, "g_single.crscene")).add_objects(crgpu.FlatScene())


# ---- helpers ---------------------------------------------------------------------------------------------------------------------

def with_mesh(doc, entry, shift=(0.0, 0.0, 0.0), instanced=True):
    """doc with a copy of the mesh entry `entry` (a file name of doc's meshes, or a whole entry) appended, moved by shift"""
    d = copy.deepcopy(doc)
    if isinstance(entry, str):
        entry = next(m for m in d["scene"]["meshes"] if m["fileName"] == entry)
    m = copy.deepcopy(entry)
    if instanced:
        for inst in m["instances"]:
            inst["transforms"] = inst.get("transforms", []) + translate(shift)["transforms"]
    else:
        m["instances"] = []
    d["scene"]["meshes"].append(m)
    return d


def with_sphere(doc, k=0, shift=(0.0, 0.0, 0.0), radius=None, instanced=True):
    """doc with a copy of sphere primitive k appended, moved by shift"""
    d = copy.deepcopy(doc)
    p = copy.deepcopy(d["scene"]["primitives"][k])
    if radius is not None:
        p["radius"] = radius
    p["color"] = {"r": 0.3, "g": 0.9, "b": 0.4}
    p["instances"] = [{"transforms": i.get("transforms", []) + translate(shift)["transforms"]} for i in p["instances"]] if instanced else []
    d["scene"]["primitives"].append(p)
    return d


def grown(name, doc, instanced=True):
    """a bundled scene with one more OBJ mesh (a moved copy of DUP[name]) and one more sphere"""
    s = STEP[name] * 5
    return with_sphere(with_mesh(doc, DUP[name], (s, 0.0, -s), instanced), 0, (-s, s, 0.0), instanced=instanced)


def sphere_materials(x):
    return crscene.arrays(x.flat)["spheres"]["material"].copy()


def bundled_pots():
    """the refraction scene's teapot entries whose OBJ file is bundled (the loader skips the others)"""
    return [m for m in teapots() if os.path.exists(os.path.join(REFDIR, "input", m["fileName"]))]


def add(g, b):
    return crgpu.lib().crgpu_scene_add_objects(g.handle, C.byref(b.flat))


def check_add(a, b, rays=None):
    """uploads a, adds b's objects and compares with b fresh"""
    g = a.upload()
    try:
        g.add_objects(b.flat)
        assert_same_as_fresh(g, b, ray_set(b.camera) if rays is None else rays)
    finally:
        g.close()


# ---- GPU: bundled scenes -------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(DUP))
def test_bundled_scene_with_one_more_mesh_and_sphere(name):
    doc = scene_json(name)
    cfg = (*SMALL, BOUNCES[name])
    a, b = Loaded(doc, *cfg), Loaded(grown(name, doc), *cfg)
    try:
        A, B = crscene.arrays(a.flat), crscene.arrays(b.flat)
        assert len(B["meshes"]) == len(A["meshes"]) + 1 and len(B["spheres"]) == len(A["spheres"]) + 1
        assert not np.array_equal(sphere_materials(a), sphere_materials(b)[:len(A["spheres"])]), "the add must move sphere materials"
        check_add(a, b)
    finally:
        a.free()
        b.free()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GOLDEN_FRAMES))
def test_objects_without_instances_give_the_committed_frames(name):
    doc = scene_json(name)
    W, H, spp, bounces, mp = GOLDEN_FRAMES[name]
    a, b = Loaded(doc, W, H, spp, bounces), Loaded(grown(name, doc, instanced=False), W, H, spp, bounces)
    g = a.upload(max_paths=mp)
    try:
        g.add_objects(b.flat)
        assert digest(full(g)) == json.load(open(DIGESTS))[name]
    finally:
        g.close()
        a.free()
        b.free()


# ---- GPU: edge scenes ------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_sphere_only_scene_gets_its_first_mesh():
    pos = spread(30, 21)
    a, b = Loaded(sphere_scene(pos, groups=3), *GEN), Loaded(sphere_scene(pos, groups=3, meshes=teapots()[:2]), *GEN)
    try:
        assert a.flat.mesh_count == 0 and b.flat.mesh_count == 2
        check_add(a, b)
    finally:
        a.free()
        b.free()


@pytest.mark.gpu
def test_mesh_only_scene_gets_its_first_sphere():
    a, b = Loaded(sphere_scene(np.zeros((0, 3)), meshes=teapots()), *GEN), Loaded(sphere_scene(spread(2, 22), meshes=teapots()), *GEN)
    try:
        assert a.flat.sphere_count == 0 and b.flat.sphere_count == 1
        check_add(a, b)
    finally:
        a.free()
        b.free()


@pytest.mark.gpu
def test_scene_without_instances_grows():
    da = objects({})
    db = with_mesh(objects(scattered(500, 23), mesh_on=(0, 3)), teapots()[1], (40.0, 0.0, -40.0))
    a, b = Loaded(da, *GEN), Loaded(db, *GEN)
    try:
        assert len(a.instances) == 0
        check_add(a, b)
    finally:
        a.free()
        b.free()


@pytest.mark.gpu
def test_million_triangle_mesh_added_to_hdr():
    k = 708                                                     # 2 * 708^2 = 1,002,528 triangles
    xs = np.arange(k + 1) / k
    X, Y = np.meshgrid(xs, xs, indexing="ij")
    assets = Assets()
    assets.write("grid.obj", grid_obj(k, 0.3 * np.sin(6.0 * X) * np.cos(5.0 * Y)))
    doc = scene_json("hdr")
    big = with_mesh(doc, {"fileName": "grid.obj", "bsdf": "lambertian",
                          "instances": [{"transforms": [{"type": "scaleUniform", "scale": 0.002}, {"type": "translate", "x": -0.2, "y": 0.0, "z": 0.0}]}]})
    cfg = (64, 36, 1, 4)
    a, b = LoadedFrom(doc, assets.dir, *cfg), LoadedFrom(big, assets.dir, *cfg)
    g, fresh = a.upload(), b.upload()
    try:
        assert crscene.arrays(b.flat)["meshes"]["poly_count"][-1] == 2 * k * k
        g.add_objects(b.flat)
        rays = ray_set(b.camera, n=50000)
        got, want = traced(g, rays), traced(fresh, rays)
        assert got[0].tobytes() == want[0].tobytes()
        assert got[1:] == want[1:]
        assert full(g).tobytes() == full(fresh).tobytes()
    finally:
        g.close()
        fresh.close()
        a.free()
        b.free()
        assets.close()


def many_materials_obj(n_mat, per=4):
    """(OBJ, MTL): a strip of per triangles for each of n_mat materials, material i a grey of its own"""
    mtl = []
    for i in range(n_mat):
        c = 0.1 + 0.8 * i / n_mat
        mtl += [f"newmtl m{i}", f"Kd {fmt(c)} {fmt(1.0 - c)} 0.5", "illum 2", ""]
    obj = ["mtllib many.mtl", "o many", "vn 0.0 0.0 1.0"]
    faces, v = [], 0
    for i in range(n_mat):
        faces.append(f"usemtl m{i}")
        for j in range(per):
            x, y = float(i % 20), float(i // 20) + 0.2 * j
            obj += ["v " + " ".join(fmt(t) for t in p) for p in ((x, y, 0.0), (x + 0.9, y, 0.0), (x, y + 0.18, 0.1))]
            faces.append(f"f {v + 1}//1 {v + 2}//1 {v + 3}//1")
            v += 3
    return "\n".join(obj + faces) + "\n", "\n".join(mtl) + "\n"


@pytest.mark.gpu
def test_shading_keys_past_254():
    """A mesh of 300 materials: its keys saturate at 255, and the spheres' materials move past 254."""
    assets = Assets()
    obj, mtl = many_materials_obj(300)
    assets.write("many.obj", obj)
    assets.write("many.mtl", mtl)
    doc = sphere_scene(spread(40, 24), groups=4, meshes=teapots()[:1])
    doc_b = with_mesh(doc, {"fileName": "many.obj", "bsdf": "lambertian",
                            "instances": [{"transforms": [{"type": "scaleUniform", "scale": 20}, {"type": "translate", "x": 800, "y": 300, "z": 1000}]}]})
    a, b = LoadedFrom(doc, assets.dir, *GEN), LoadedFrom(doc_b, assets.dir, *GEN)
    try:
        assert crscene.arrays(b.flat)["meshes"]["material_count"][-1] == 300
        assert (sphere_materials(b) > 254).all()
        check_add(a, b)
    finally:
        a.free()
        b.free()
        assets.close()


# ---- GPU: repeated growth ------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_eight_meshes_one_per_call_then_back():
    base = objects(scattered(60, 25), mesh_on=(0,))
    docs = [base]
    pool = bundled_pots()
    for k in range(8):
        docs.append(with_mesh(docs[-1], pool[k % len(pool)], (30.0 + 25.0 * k, 10.0 * k, -20.0)))
    a = Loaded(base, *GEN)
    g = a.upload()
    try:
        for k, d in enumerate(docs[1:]):
            b = Loaded(d, *GEN)
            try:
                assert b.flat.mesh_count == a.flat.mesh_count + k + 1
                g.add_objects(b.flat)
                assert_same_as_fresh(g, b, ray_set(b.camera))
            finally:
                b.free()
        back = copy.deepcopy(docs[-1])
        for m in back["scene"]["meshes"][a.flat.mesh_count:]:
            m["instances"] = []
        b = Loaded(back, *GEN)
        try:
            g.set_instance_list(b.instances)
            assert_same_as_fresh(g, b, ray_set(b.camera))
        finally:
            b.free()
    finally:
        g.close()
        a.free()


# ---- GPU: composition --------------------------------------------------------------------------------------------------------

def comp_docs():
    """(A, B): hdr, and hdr with a moved copy of its Venus and one more sphere"""
    doc = scene_json("hdr")
    return doc, grown("hdr", doc)


@pytest.mark.gpu
def test_set_meshes_on_a_new_mesh():
    da, db = comp_docs()
    cfg = (*SMALL, BOUNCES["hdr"])
    assets = Assets()
    assets.write("torus.obj", deform_obj(assets.original("torus.obj"), seed=4))
    db = with_mesh(db, {"fileName": "torus.obj", "bsdf": "lambertian",
                        "instances": [{"transforms": [{"type": "scaleUniform", "scale": 0.05}, {"type": "translate", "x": 0.1, "y": 0.02, "z": 0.0}]}]})
    a, b, c = Loaded(da, *cfg), Loaded(db, *cfg), LoadedFrom(db, assets.dir, *cfg)
    g = a.upload()
    try:
        g.add_objects(b.flat)
        torus = b.flat.mesh_count - 1
        g.set_meshes(c.flat, [torus])
        assert_same_as_fresh(g, c, ray_set(c.camera))
    finally:
        g.close()
        for x in (a, b, c):
            x.free()
        assets.close()


@pytest.mark.gpu
def test_set_meshes_on_an_old_mesh_before_the_add():
    da, db = comp_docs()
    cfg = (*SMALL, BOUNCES["hdr"])
    assets = Assets()
    assets.write("venusscaled.obj", deform_obj(assets.original("venusscaled.obj"), seed=8))
    a, a2, b2 = Loaded(da, *cfg), LoadedFrom(da, assets.dir, *cfg), LoadedFrom(db, assets.dir, *cfg)
    g = a.upload()
    try:
        g.set_meshes(a2.flat, [1])
        g.add_objects(b2.flat)
        assert_same_as_fresh(g, b2, ray_set(b2.camera))
    finally:
        g.close()
        for x in (a, a2, b2):
            x.free()
        assets.close()


def more_instances(doc):
    """doc with a second instance of its last mesh and of its last sphere"""
    d = copy.deepcopy(doc)
    for obj in (d["scene"]["meshes"][-1], d["scene"]["primitives"][-1]):
        extra = copy.deepcopy(obj["instances"][0])
        extra["transforms"] = extra.get("transforms", []) + translate((0.03, 0.0, 0.02))["transforms"]
        obj["instances"].append(extra)
    return d


def moved_instances(doc):
    d = copy.deepcopy(doc)
    for obj in (d["scene"]["meshes"][-1], d["scene"]["primitives"][-1]):
        for inst in obj["instances"]:
            inst["transforms"] = inst.get("transforms", []) + translate((0.0, 0.01, 0.0))["transforms"]
    return d


@pytest.mark.gpu
@pytest.mark.parametrize("list_first", [False, True])
def test_instance_edits_with_the_new_objects(list_first):
    """add, then set_instance_list with more instances of the new objects and set_instances moving them; or a list edit of the old
    objects before the add"""
    da, db = comp_docs()
    cfg = (*SMALL, BOUNCES["hdr"])
    dc = more_instances(db)
    a, b, c, d = Loaded(da, *cfg), Loaded(db, *cfg), Loaded(dc, *cfg), Loaded(moved_instances(dc), *cfg)
    g = a.upload()
    try:
        if list_first:
            short = copy.deepcopy(da)
            short["scene"]["primitives"][1]["instances"] = []
            s = Loaded(short, *cfg)
            g.set_instance_list(s.instances)
            s.free()
            g.add_objects(b.flat)
            assert_same_as_fresh(g, b, ray_set(b.camera))
        else:
            g.add_objects(b.flat)
            g.set_instance_list(c.instances)
            assert_same_as_fresh(g, c, ray_set(c.camera))
            g.set_instances(d.instances)
            assert_same_as_fresh(g, d, ray_set(d.camera))
    finally:
        g.close()
        for x in (a, b, c, d):
            x.free()


@pytest.mark.gpu
@pytest.mark.parametrize("shading_first", [False, True])
def test_set_shading_and_camera(shading_first):
    """set_shading at the grown count and set_camera after the add; or set_shading at the old count before it"""
    da, db = comp_docs()
    cfg = (*SMALL, BOUNCES["hdr"])
    dc = copy.deepcopy(db)
    for prim in dc["scene"]["primitives"]:
        prim["color"] = {"r": 0.9, "g": 0.2, "b": 0.1}
    tr = next(t for t in dc["camera"]["transforms"] if t["type"] == "translate")
    for k in ("x", "y", "z"):
        if k in tr:
            tr[k] += STEP["hdr"]
    a, b, c = Loaded(da, *cfg), Loaded(db, *cfg), Loaded(dc, *cfg)
    g = a.upload()
    try:
        if shading_first:
            recol = copy.deepcopy(da)
            for prim in recol["scene"]["primitives"]:
                prim["color"] = {"r": 0.1, "g": 0.1, "b": 0.9}
            r = Loaded(recol, *cfg)
            g.set_shading(r.flat)
            r.free()
            g.add_objects(b.flat)
            assert_same_as_fresh(g, b, ray_set(b.camera))
        else:
            g.add_objects(b.flat)
            assert g.shading()["kinds"].shape == (b.flat.material_count,)
            g.set_shading(c.flat)
            g.set_camera(c.camera)
            assert_same_as_fresh(g, c, ray_set(c.camera))
    finally:
        g.close()
        for x in (a, b, c):
            x.free()


@pytest.mark.gpu
def test_render_views_after_the_add():
    da, db = comp_docs()
    W, H, spp = SMALL
    cfg = (W, H, spp, BOUNCES["hdr"])
    a, b = Loaded(da, *cfg), Loaded(db, *cfg)
    cams = []
    for k in range(3):
        c = crgpu.Camera.from_buffer_copy(b.camera)
        c.A[3] += np.float32(0.01 * k)
        cams.append(c)
    g, fresh = a.upload(), b.upload()
    try:
        g.set_views(cams)
        g.add_objects(b.flat)
        for v in range(3):
            g.view_clear(v)
        g.render_views([(0, 0, W, H)])
        for v in range(3):
            fresh.set_camera(cams[v])
            assert g.view_read(v).tobytes() == full(fresh).tobytes(), f"view {v}"
    finally:
        g.close()
        fresh.close()
        a.free()
        b.free()


@pytest.mark.gpu
def test_stopped_and_resumed_render_after_the_add():
    da, db = comp_docs()
    W, H, spp, bounces, mp = GOLDEN_FRAMES["hdr"]
    a, b = Loaded(da, W, H, spp, bounces), Loaded(db, W, H, spp, bounces)
    fresh = b.upload(max_paths=mp)
    want = full(fresh)
    fresh.close()
    g = a.upload(max_paths=mp)
    try:
        g.enable_stop()
        g.add_objects(b.flat)
        g.clear()
        g.render_tile(0, 0, g.W, g.H, flags=crgpu.FLAG_ASYNC)
        g.request_stop()
        g.get_stats()
        done, busy = g.progress()
        assert not busy and 0 <= done <= spp
        g.clear_stop()
        st = g.render_tile(0, 0, g.W, g.H, pass_begin=done)
        assert st["stopped"] is False
        assert g.read().tobytes() == want.tobytes()
    finally:
        g.close()
        a.free()
        b.free()


@pytest.mark.gpu
def test_add_drains_a_render_in_flight():
    da, db = comp_docs()
    W, H, spp, bounces, mp = GOLDEN_FRAMES["hdr"]
    a, b = Loaded(da, W, H, spp, bounces), Loaded(db, W, H, spp, bounces)
    fresh = b.upload(max_paths=mp)
    want = full(fresh)
    fresh.close()
    g = a.upload(max_paths=mp)
    try:
        g.clear()
        g.render_tile(0, 0, g.W, g.H, flags=crgpu.FLAG_ASYNC)
        g.add_objects(b.flat)
        assert full(g).tobytes() == want.tobytes()
    finally:
        g.close()
        a.free()
        b.free()


# ---- GPU: refusals -------------------------------------------------------------------------------------------------------------

def poke(flat, name, values):
    """writes a record array over the flat scene's own (meshes, spheres, materials: write_back refuses those)"""
    arr = np.ascontiguousarray(values)
    C.memmove(getattr(flat, name), arr.ctypes.data, arr.nbytes)


@pytest.mark.gpu
@pytest.mark.parametrize("grown_first", [False, True])
def test_refusals_leave_the_scene_unchanged(grown_first):
    da, db = comp_docs()
    cfg = (*SMALL, BOUNCES["hdr"])
    a, b = Loaded(da, *cfg), Loaded(db, *cfg)
    g = a.upload()
    L = crgpu.lib()
    try:
        if grown_first:
            g.add_objects(b.flat)
        live = b if grown_first else a
        rays = ray_set(live.camera)
        before_img, before_tr = full(g), traced(g, rays)
        c = Loaded(with_mesh(db, "venusscaled.obj", (0.0, 0.05, 0.0)), *cfg)     # one mesh more than b: refusals also when grown
        B = crscene.arrays(c.flat)
        M = a.flat.mesh_count if not grown_first else b.flat.mesh_count
        S = a.flat.sphere_count if not grown_first else b.flat.sphere_count
        try:
            def refused(code, field, values, what):
                poke(c.flat, field, values)
                try:
                    assert add(g, c) == code, what
                finally:
                    poke(c.flat, field, B[field])

            for fld, cnt in (("mesh_count", M - 1), ("sphere_count", S - 1)):
                old = getattr(c.flat, fld)
                setattr(c.flat, fld, cnt)
                assert add(g, c) == BAD_ARGUMENT, fld
                setattr(c.flat, fld, old)
            m = B["meshes"].copy(); m["material_count"][0] += 1
            refused(BAD_ARGUMENT, "meshes", m, "a changed existing mesh")
            sp = B["spheres"].copy(); sp["radius"][0] += 1.0
            refused(BAD_ARGUMENT, "spheres", sp, "a changed sphere radius")
            new = c.flat.mesh_count - 1
            m = B["meshes"].copy(); m["poly_offset"][new] = m["poly_offset"][new - 1]
            refused(BAD_ARGUMENT, "meshes", m, "overlapping new meshes")
            m = B["meshes"].copy(); m["poly_offset"][new] = m["poly_offset"][M - 1]
            refused(BAD_ARGUMENT, "meshes", m, "a new mesh over the scene's polys")
            m = B["meshes"].copy(); m["poly_count"][new] += 1
            refused(BAD_ARGUMENT, "meshes", m, "a poly range out of bounds")
            for bvh in (c.flat.top_bvh, m["bvh"][0], c.flat.bvh_count):
                m = B["meshes"].copy(); m["bvh"][new] = bvh
                refused(BAD_ARGUMENT, "meshes", m, f"bvh index {bvh}")
            m = B["meshes"].copy(); m["material_offset"][new] = c.flat.material_count
            refused(BAD_ARGUMENT, "meshes", m, "a material range out of bounds")
            s0 = int(B["meshes"]["poly_offset"][new])
            for col, count in (("v", len(B["vertices"])), ("n", len(B["normals"]))):
                polys = B["polys"].copy()
                polys[col][s0, 1] = count
                polys["has_normals"][s0] = 1
                crscene.write_back(c.flat, "polys", polys)
                assert add(g, c) == BAD_ARGUMENT, col
            polys = B["polys"].copy()
            polys["material"][s0] = B["meshes"]["material_count"][new]
            crscene.write_back(c.flat, "polys", polys)
            assert add(g, c) == BAD_ARGUMENT, "a poly material out of range"
            crscene.write_back(c.flat, "polys", B["polys"])
            inst = B["instances"].copy(); inst["object"][-1] = 10 ** 6
            refused(BAD_ARGUMENT, "instances", inst, "an instance of no object")
            # the shading is refused with crgpu_prepare's code
            mats = B["materials"].copy(); mats["bsdf"][0] = c.flat.node_count + 5
            poke(c.flat, "materials", mats)
            L.crgpu_prepare.argtypes = [C.POINTER(crgpu.FlatScene), C.POINTER(C.c_void_p)]
            L.crgpu_prepare.restype = C.c_int
            p = C.c_void_p()
            want = L.crgpu_prepare(C.byref(c.flat), C.byref(p))
            assert want < 0 and add(g, c) == want
            poke(c.flat, "materials", B["materials"])
            # limits: a new mesh of more than 4,194,304 polys, more than 4,194,304 instances (neither is read)
            old = c.flat.poly_count
            m = B["meshes"].copy(); m["poly_count"][new] = 4194305
            c.flat.poly_count = int(m["poly_offset"][new]) + 4194305
            refused(UNSUPPORTED, "meshes", m, "a mesh of 4194305 polys")
            c.flat.poly_count = old
            old = c.flat.instance_count
            c.flat.instance_count = 4194305
            assert add(g, c) == UNSUPPORTED
            c.flat.instance_count = old
            assert L.crgpu_scene_add_objects(g.handle, None) == BAD_ARGUMENT
        finally:
            c.free()
        img, tr = full(g), traced(g, rays)
        assert img.tobytes() == before_img.tobytes(), "a refused add changed the frame"
        assert tr[0].tobytes() == before_tr[0].tobytes() and tr[1:] == before_tr[1:], "a refused add changed the traversal"
        g.add_objects(b.flat)                                   # and the scene still takes a valid add
        assert_same_as_fresh(g, b, ray_set(b.camera))
    finally:
        g.close()
        a.free()
        b.free()
