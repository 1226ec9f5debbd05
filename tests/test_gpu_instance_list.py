"""Adding and removing instances of a resident GPU scene between renders (crgpu_scene_set_instance_list, include/crgpu.h).

The target is exact: a scene A given the instance array of a scene B renders, traces and shades the same bits as B loaded fresh
from its JSON, including the P/T/S/I counts of the instrumented traversal, which pin the shape and BFS packing of the new top
level.  A and B have the same objects (spheres and meshes); a sphere or mesh entry with "instances": [] loads as an object without
an instance, which is how A holds objects that only B instances.

CPU: argument checks of the new entry point.  GPU: everything else.
"""
import copy
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import crgpu
import crscene
from conftest import GOLDEN, ROOT
from test_gpu_scene_edit import (BOUNCES, DIGESTS, GOLDEN_FRAMES, SMALL, STEP, Loaded, assert_same_as_fresh, digest, full, ray_set,
                                 scene_json, sphere_scene, spread, teapots, traced)

BAD_ARGUMENT, UNSUPPORTED = -3, -4
GEN = (160, 90, 2, 8)                                   # W, H, spp, bounces of the generated scenes
ALL = range(10)                                         # every teapot entry (teapot_white.obj is missing: 9 meshes load)
DUP = {"hdr": "venusscaled.obj", "venus": "torus.obj", "refraction": "torus.obj"}


# ---- CPU -----------------------------------------------------------------------------------------------------------------------

def test_entry_point_rejects_null_arguments():
    L = crgpu.lib()
    inst = np.zeros(1, dtype=crscene.INSTANCE)
    assert L.crgpu_scene_set_instance_list(None, None, 0) == BAD_ARGUMENT
    assert L.crgpu_scene_set_instance_list(None, inst.ctypes.data, 1) == BAD_ARGUMENT
    assert L.crgpu_scene_set_instance_list(None, None, 1) == BAD_ARGUMENT


def test_no_scene_to_edit_without_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    with pytest.raises(crgpu.CrgpuError):
        crgpu.GpuScene(os.path.join(GOLDEN, "g_single.crscene")).set_instance_list(np.zeros(0, dtype=crscene.INSTANCE))


# ---- helpers ---------------------------------------------------------------------------------------------------------------------

def translate(p):
    return {"transforms": [{"type": "translate", "x": float(p[0]), "y": float(p[1]), "z": float(p[2])}]}


def objects(sphere_pos, mesh_on=(), groups=40, radius=2.0, shift=0.0):
    """sphere_scene's 40 sphere objects and the refraction teapots, each with an explicit instance list: sphere object g takes the
    positions sphere_pos[g] (a dict; missing: none), teapot m keeps its instance when m is in mesh_on."""
    d = sphere_scene(np.zeros((groups, 3)), groups=groups, meshes=teapots(shift), radius=radius)
    for g, prim in enumerate(d["scene"]["primitives"]):
        prim["instances"] = [translate(p) for p in sphere_pos.get(g, ())]
    for m, mesh in enumerate(d["scene"]["meshes"]):
        if m not in mesh_on:
            mesh["instances"] = []
    return d


def scattered(n, seed, groups=40):
    """n sphere positions dealt over the groups"""
    pos = spread(n, seed)
    return {g: pos[g::groups] for g in range(groups) if len(pos[g::groups])}


def set_list(g, instances):
    inst = np.ascontiguousarray(instances)
    return crgpu.lib().crgpu_scene_set_instance_list(g.handle, inst.ctypes.data if len(inst) else None, len(inst))


def check_list(g, doc_b, cfg=GEN, rays=None):
    """g takes the instance list of doc_b and must equal doc_b loaded fresh."""
    b = Loaded(doc_b, *cfg)
    try:
        g.set_instance_list(b.instances)
        assert_same_as_fresh(g, b, ray_set(b.camera) if rays is None else rays)
        return len(b.instances)
    finally:
        b.free()


def duplicated(doc, name, file=None, step=None):
    """a second instance of DUP[name]'s mesh (or of the first instance of mesh file `file`), moved by STEP[name] * 5 (or `step`)"""
    d = copy.deepcopy(doc)
    mesh = next(m for m in d["scene"]["meshes"] if m["fileName"] == (file or DUP[name]) and m.get("instances"))
    extra = copy.deepcopy(mesh["instances"][0])
    extra.setdefault("transforms", [])
    s = STEP[name] * 5 if step is None else step
    extra["transforms"].append({"type": "translate", "x": s, "y": 0.0, "z": -s})
    mesh["instances"].append(extra)
    return d


def removed(doc, k=1):
    """sphere primitive k without its instances"""
    d = copy.deepcopy(doc)
    d["scene"]["primitives"][k]["instances"] = []
    return d


def bundled(name, doc_a, doc_b):
    W, H, spp = SMALL
    a, b = Loaded(doc_a, W, H, spp, BOUNCES[name]), Loaded(doc_b, W, H, spp, BOUNCES[name])
    g = a.upload()
    try:
        assert len(a.instances) != len(b.instances) or a.instances.tobytes() != b.instances.tobytes()
        g.set_instance_list(b.instances)
        assert_same_as_fresh(g, b, ray_set(b.camera))
    finally:
        g.close()
        a.free()
        b.free()


# ---- GPU: bundled scenes -------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(DUP))
def test_duplicated_mesh_instance(name):
    doc = scene_json(name)
    bundled(name, doc, duplicated(doc, name))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(DUP))
def test_removed_sphere_instance(name):
    doc = scene_json(name)
    bundled(name, doc, removed(doc))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(DUP))
def test_sphere_without_instances_gets_one(name):
    """A loads sphere primitive 2 with no instance; the list instances it, with its uploaded radius and material."""
    doc = scene_json(name)
    bundled(name, removed(doc, 2), doc)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GOLDEN_FRAMES))
def test_editing_back_gives_the_committed_frames(name):
    doc = scene_json(name)
    W, H, spp, bounces, mp = GOLDEN_FRAMES[name]
    a, b = Loaded(doc, W, H, spp, bounces), Loaded(removed(duplicated(doc, name)), W, H, spp, bounces)
    g = a.upload(max_paths=mp)
    try:
        g.set_instance_list(b.instances)
        moved = full(g)
        g.set_instance_list(a.instances)
        back = full(g)
        want = json.load(open(DIGESTS))[name]
        assert digest(back) == want
        assert digest(moved) != want
    finally:
        g.close()
        a.free()
        b.free()


# ---- GPU: generated scenes -----------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_growing_and_shrinking_generated_lists():
    """1 -> 20,009 -> 200,000 -> 3 instances, each against its fresh scene."""
    a = Loaded(objects({0: spread(1, 3)}), *GEN)
    g = a.upload()
    try:
        assert check_list(g, objects(scattered(20000, 1), mesh_on=ALL)) == 20009
        assert check_list(g, objects(scattered(199991, 2), mesh_on=ALL)) == 200000
        assert check_list(g, objects({5: spread(2, 4)}, mesh_on=(4,))) == 3
    finally:
        g.close()
        a.free()


@pytest.mark.gpu
def test_empty_list_and_back():
    """0 instances: every ray misses and the frame is the empty scene's; then the list grows again."""
    a = Loaded(objects(scattered(300, 5), mesh_on=(0, 1)), *GEN)
    g = a.upload()
    try:
        rays = ray_set(a.camera)
        assert check_list(g, objects({}), rays=rays) == 0
        rec, misses, _ = traced(g, rays)
        assert misses == len(rays) and (rec["inst"] == -1).all()
        assert check_list(g, objects(scattered(500, 6), mesh_on=(2, 4))) == 502
    finally:
        g.close()
        a.free()


@pytest.mark.gpu
def test_coincident_instances_take_the_median_fallback():
    pos = spread(1, 7)
    a = Loaded(objects({k: spread(10, 8 + k) for k in range(4)}), *GEN)
    g = a.upload()
    try:
        assert check_list(g, objects({k: np.repeat(pos, 15, axis=0) for k in range(4)})) == 60
    finally:
        g.close()
        a.free()


def _oversized_top():
    """(A, the instances of a list whose top level needs more than 2n - 1 nodes, A's list after a growth): test_bvh_degenerate's
    17 radius-0 spheres on one point among 23 spread radius-0 spheres"""
    import test_bvh_degenerate as D
    rng = np.random.default_rng(23)
    before = np.round(rng.uniform(-2, 2, (17, 3)) + [0, 0, 6], 3)
    spread23 = np.round(rng.uniform(-2, 2, (23, 3)) + [0, 0, 6], 3)
    cfg = (64, 48, 2, 4)
    a = Loaded(D.edit_doc(before, spread23[:5], 0.0), *cfg)
    grown = Loaded(D.edit_doc(before, spread23, 0.0), *cfg)
    bad = Loaded(D.edit_doc([[0.2, 0.1, 5.0]] * 17, spread23, 0.0), *cfg)
    rc, nodes, *_ = D._host_build(*D.top_boxes(bad.instances, 0.0))
    assert rc == -2 and nodes > 2 * len(bad.instances) - 1, (rc, nodes)
    return a, grown, bad


@pytest.mark.gpu
def test_top_level_of_more_than_2n_minus_1_nodes_is_refused():
    a, grown, bad = _oversized_top()
    g = a.upload()
    try:
        rays = ray_set(grown.camera)
        g.set_instance_list(grown.instances)
        assert_same_as_fresh(g, grown, rays)
        before_img, before_tr = full(g), traced(g, rays)
        assert set_list(g, bad.instances) == UNSUPPORTED
        img, tr = full(g), traced(g, rays)
        assert img.tobytes() == before_img.tobytes() and tr[0].tobytes() == before_tr[0].tobytes() and tr[1:] == before_tr[1:]
        g.set_instances(grown.instances)                       # the refused list left the scene's list as it was
    finally:
        g.close()
        for x in (a, grown, bad):
            x.free()


@pytest.mark.gpu
def test_top_region_grows_behind_an_edited_mesh():
    """2 instances uploaded; set_meshes gives teapot 0 its region behind the small top region; the list then grows to 50,000 and its
    top level takes a new region at the end of the pairs block.  Teapot 0 and the teapots set_meshes never rebuilt render from
    their regions as they were."""
    a = Loaded(objects({0: spread(1, 9)}, mesh_on=(0,)), *GEN)
    g = a.upload()
    try:
        g.set_meshes(a.flat, [0])
        assert check_list(g, objects(scattered(49991, 10), mesh_on=ALL)) == 50000
    finally:
        g.close()
        a.free()


# ---- GPU: composition, stops, staging, refusals ------------------------------------------------------------------------------

def _composed_docs():
    """(A, B, C, assets): A small; B a larger list of A's objects; C B's list moved, with a deformed teapot.obj, recoloured spheres
    and a moved camera"""
    from test_gpu_mesh_edit import Assets, deform_obj
    a = objects({0: spread(2, 11)}, mesh_on=(0,))
    b = objects(scattered(900, 12), mesh_on=(0, 1, 4))
    c = objects({k: v + 7.5 for k, v in scattered(900, 12).items()}, mesh_on=(0, 1, 4), shift=30.0)
    for prim in c["scene"]["primitives"]:
        prim["color"] = {"r": 0.9, "g": 0.2, "b": 0.1}
    for tr in c["camera"]["transforms"]:
        if tr["type"] == "translate":
            for k in ("x", "y", "z"):
                if k in tr:
                    tr[k] += 15.0
    assets = Assets()
    assets.write("teapot.obj", deform_obj(assets.original("teapot.obj"), "v", 3))
    return a, b, c, assets


@pytest.mark.gpu
@pytest.mark.parametrize("meshes_first", [False, True])
def test_list_composes_with_the_other_edits(meshes_first):
    """list, set_instances at the new count, set_meshes, set_shading, set_camera; or set_meshes before the list edit"""
    from test_gpu_mesh_edit import LoadedFrom, changed_meshes
    da, db, dc, assets = _composed_docs()
    a, b, c = Loaded(da, *GEN), Loaded(db, *GEN), LoadedFrom(dc, assets.dir, *GEN)
    g = a.upload()
    try:
        ch = changed_meshes(a, c)
        assert ch
        if meshes_first:
            g.set_meshes(c.flat, ch)
            g.set_instance_list(c.instances)
        else:
            g.set_instance_list(b.instances)
            g.set_instances(c.instances)
            g.set_meshes(c.flat, ch)
        g.set_shading(c.flat)
        g.set_camera(c.camera)
        assert_same_as_fresh(g, c, ray_set(c.camera))
    finally:
        g.close()
        for x in (a, b, c):
            x.free()
        assets.close()


@pytest.mark.gpu
def test_list_edit_after_a_stopped_render():
    doc = scene_json("hdr")
    W, H, spp, bounces, mp = GOLDEN_FRAMES["hdr"]
    a, b = Loaded(doc, W, H, spp, bounces), Loaded(removed(duplicated(doc, "hdr")), W, H, spp, bounces)
    fresh = b.upload(max_paths=mp)
    want = full(fresh)
    fresh.close()
    g = a.upload(max_paths=mp)
    try:
        g.enable_stop()
        g.clear()
        g.render_tile(0, 0, g.W, g.H, flags=crgpu.FLAG_ASYNC)
        g.request_stop()
        g.set_instance_list(b.instances)
        g.clear_stop()
        g.clear()
        st = g.render_tile(0, 0, g.W, g.H)
        assert st["stopped"] is False
        assert g.read().tobytes() == want.tobytes()
    finally:
        g.close()
        a.free()
        b.free()


def crowded(doc):
    """hdr with a second Venus and 60 instances of sphere primitive 3, each moved a little further"""
    d = duplicated(doc, "hdr")
    prim = d["scene"]["primitives"][3]
    tf = prim["instances"][0]["transforms"]
    prim["instances"] = [{"transforms": tf + [{"type": "translate", "x": 0.01 * k, "y": 0.0, "z": 0.0}]} for k in range(60)]
    return d


STAGED = r"""
import sys
sys.path[:0] = [{pkg!r}, {tests!r}]
import test_gpu_scene_edit as T
import test_gpu_instance_list as I
doc = T.scene_json("hdr")
a = T.Loaded(doc, 320, 240, 2, 32)
g = a.upload()
for d in (I.crowded(doc), I.removed(doc), doc):
    b = T.Loaded(d, 320, 240, 2, 32)
    g.set_instance_list(b.instances)
    T.assert_same_as_fresh(g, b, T.ray_set(b.camera, n=70000))
    b.free()
g.close()
print("staged ok")
"""


@pytest.mark.gpu
def test_list_edits_with_staged_top_nodes():
    """CRGPU_TRACE_STAGE=128 (read at prepare time) stages up to 32 top-level pairs; lists of 73, 12 and 13 instances rewrite that
    prefix."""
    scene_json("hdr")
    env = dict(os.environ, CRGPU_TRACE_STAGE="128")
    code = STAGED.format(pkg=os.path.join(ROOT, "c-ray_b200"), tests=os.path.join(ROOT, "tests"))
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0 and "staged ok" in r.stdout, r.stdout[-3000:]


@pytest.mark.gpu
@pytest.mark.parametrize("grown_first", [False, True])
def test_refused_lists_leave_the_scene_unchanged(grown_first):
    doc = scene_json("hdr")
    W, H, spp = SMALL
    a, b = Loaded(doc, W, H, spp, BOUNCES["hdr"]), Loaded(duplicated(doc, "hdr"), W, H, spp, BOUNCES["hdr"])
    g = a.upload()
    L = crgpu.lib()
    try:
        if grown_first:
            g.set_instance_list(b.instances)
        live = b if grown_first else a
        rays = ray_set(live.camera)
        before_img, before_tr = full(g), traced(g, rays)
        inst = b.instances.copy()
        bad = inst.copy()
        bad["kind"][0] = 2
        assert set_list(g, bad) == BAD_ARGUMENT
        for kind, count in ((0, a.flat.sphere_count), (1, a.flat.mesh_count)):
            bad = inst.copy()
            k = int(np.flatnonzero(bad["kind"] == kind)[-1])
            bad["object"][k] = count
            assert set_list(g, bad) == BAD_ARGUMENT
        assert L.crgpu_scene_set_instance_list(g.handle, None, 5) == BAD_ARGUMENT
        assert L.crgpu_scene_set_instance_list(g.handle, inst.ctypes.data, 4194305) == UNSUPPORTED
        img, tr = full(g), traced(g, rays)
        assert img.tobytes() == before_img.tobytes(), "a refused list changed the frame"
        assert tr[0].tobytes() == before_tr[0].tobytes() and tr[1:] == before_tr[1:], "a refused list changed the traversal"
        # set_instances checks against the live list: the other count is refused
        other = a if grown_first else b
        assert L.crgpu_scene_set_instances(g.handle, np.ascontiguousarray(other.instances).ctypes.data, len(other.instances)) == BAD_ARGUMENT
        g.set_instances(live.instances)
    finally:
        g.close()
        a.free()
        b.free()


# ---- GPU: isolation and memory ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_list_edit_applies_to_one_scene_only():
    a, b = Loaded(objects(scattered(40, 13), mesh_on=(0,)), *GEN), Loaded(objects(scattered(4000, 14), mesh_on=(1, 2)), *GEN)
    L = crgpu.lib()
    L.crgpu_prepare.argtypes = [C.POINTER(crgpu.FlatScene), C.POINTER(C.c_void_p)]
    L.crgpu_prepare.restype = C.c_int
    L.crgpu_prepared_free.argtypes = [C.c_void_p]
    L.crgpu_prepared_free.restype = None
    p = C.c_void_p()
    assert L.crgpu_prepare(C.byref(a.flat), C.byref(p)) == 0
    scenes = []
    try:
        for _ in range(2):
            g = crgpu.GpuScene(None, *GEN, prepared=p.value)
            g.W, g.H = GEN[:2]
            scenes.append(g)
        rays = ray_set(a.camera)
        want_img, want_tr = full(scenes[1]), traced(scenes[1], rays)
        scenes[0].set_instance_list(b.instances)
        assert_same_as_fresh(scenes[0], b, ray_set(b.camera))
        img, tr = full(scenes[1]), traced(scenes[1], rays)
        assert img.tobytes() == want_img.tobytes() and tr[0].tobytes() == want_tr[0].tobytes() and tr[1:] == want_tr[1:]
    finally:
        for g in scenes:
            g.close()
        L.crgpu_prepared_free(p)
        a.free()
        b.free()


@pytest.mark.gpu
def test_alternating_lists_stay_exact_and_do_not_leak():
    """20 lists alternating 10 and 20,000 instances: exact, and the device's free memory does not fall after the first growth."""
    import torch
    docs = [objects(scattered(10, 15)), objects(scattered(19991, 16), mesh_on=ALL)]
    loaded = [Loaded(d, *GEN) for d in docs]
    a = Loaded(objects({0: spread(3, 17)}), *GEN)
    g = a.upload()
    try:
        want = []
        for x in loaded:
            f = x.upload()
            want.append(full(f).tobytes())
            f.close()
        torch.cuda.init()
        free = []
        for k in range(20):
            g.set_instance_list(loaded[k % 2].instances)
            assert full(g).tobytes() == want[k % 2], f"list {k}"
            free.append(torch.cuda.mem_get_info()[0])
        assert min(free[2:]) >= free[1], free
    finally:
        g.close()
        a.free()
        for x in loaded:
            x.free()
