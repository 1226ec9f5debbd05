"""The device blocks of the resident-scene edits, on the CPU against the stub CUDA runtime (tests/stub/, test tooling only).

Every edit call stages the blocks it replaces, publishes the scene's descriptor once and only then releases the replaced blocks
(DESIGN §4 "Editing a resident scene").  tests/stub/edit_blocks_harness.c, linked with AddressSanitizer, runs each edit that needs no
kernel result on a golden scene: set_camera, set_views (grow, shrink, grow), set_render (with a resize and without), set_shading,
set_instance_list with no instances, and add_objects of a sphere with a new material and of a mesh with no polys, both with an empty
instance list.  It checks that no device allocation outlives the scenes, that no block is read after it went back to the cache, and
that a call whose k-th allocation fails, for every k it makes, returns CRGPU_ERR_NOMEM and leaves the scene as it was."""
import copy
import ctypes as C
import json
import os
import shutil
import subprocess

import pytest

import crgpu
import crscene
from conftest import ROOT, GOLDEN
from test_gpu_add_objects import with_mesh, with_sphere
from test_gpu_shading_edit import Shading, variants

PKG = os.path.join(ROOT, "c-ray_b200")
OPS = ["set_camera", "set_views_3", "set_views_2", "set_views_4", "set_render_resize", "set_render", "set_shading",
       "set_instance_list_empty", "add_objects_sphere", "add_objects_empty_mesh"]


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    objs = [os.path.join(PKG, "build", n) for n in ("crgpu_api.o", "crgpu_trace.o", "crgpu_shade.o", "crgpu_bvh_build.o")]
    if not all(os.path.exists(o) for o in objs):
        pytest.skip("c-ray_b200/build/*.o not present (built by nvcc in build())")
    d = tmp_path_factory.mktemp("edit_blocks")
    exe = str(d / "edit_blocks_harness")
    stub = os.path.join(ROOT, "tests", "stub")
    cc = ["gcc", "-O1", "-g", "-fsanitize=address", "-c"]
    subprocess.run(cc + ["-o", str(d / "stub.o"), os.path.join(stub, "cudart_stub.c")], check=True)
    subprocess.run(cc + ["-I" + os.path.join(ROOT, "include"), "-o", str(d / "h.o"), os.path.join(stub, "edit_blocks_harness.c")], check=True)
    subprocess.run(cc + ["-o", str(d / "io.o"), os.path.join(PKG, "host", "crscene_io.c")], check=True)
    subprocess.run(["g++", "-fsanitize=address", "-o", exe, str(d / "h.o")] + objs + [str(d / "io.o"), str(d / "stub.o"), "-lpthread"],
                   check=True)
    return exe, d


def bare(doc):
    """doc without instances"""
    d = copy.deepcopy(doc)
    for o in d["scene"]["meshes"] + d["scene"]["primitives"]:
        o["instances"] = []
    return d


def save(flat, path):
    L = crgpu.lib()
    L.crscene_save.argtypes = [C.POINTER(crgpu.FlatScene), C.c_char_p]
    assert L.crscene_save(C.byref(flat), str(path).encode()) == 0
    return str(path)


def scenes(d):
    """A (g_legacy: meshes, spheres, instances), A's shading with an image material and background, B1 (A's objects and one more
    sphere with a material of its own, no instances) and B2 (B1 and a mesh with no polys)"""
    root = d / "scene"
    shutil.copytree(os.path.join(GOLDEN, "assets"), root / "assets", dirs_exist_ok=True)
    (root / "assets" / "empty.obj").write_text("o empty\nv 0 0 0\n")
    doc = json.load(open(os.path.join(GOLDEN, "g_legacy.json")))
    b1 = with_sphere(bare(doc), 0, instanced=False)
    b2 = with_mesh(b1, {"fileName": "assets/empty.obj", "bsdf": "lambertian", "instances": []}, instanced=False)
    here = os.getcwd()
    os.chdir(root)
    try:
        flats = [crscene.load_json_buf(json.dumps(x)) for x in (doc, b1, b2)]
    finally:
        os.chdir(here)
    try:
        a, B1, B2 = (crscene.arrays(f) for f in flats)
        assert len(B1["spheres"]) == len(a["spheres"]) + 1 and len(B1["materials"]) == len(a["materials"]) + 1
        assert len(B2["meshes"]) == len(a["meshes"]) + 1 and B2["meshes"]["poly_count"][-1] == 0
        assert a["instances"].size and not B1["instances"].size and not B2["instances"].size
        shade = next(v for what, v, _ in variants(Shading(flats[0])) if what == "image")
        return [save(flats[0], d / "a.crscene"), save(shade.flat(), d / "shade.crscene"), save(flats[1], d / "b1.crscene"),
                save(flats[2], d / "b2.crscene")]
    finally:
        for f in flats:
            crscene.free(f)


def test_edits_release_nothing_live_and_fail_without_a_trace(harness):
    exe, d = harness
    r = subprocess.run([exe] + scenes(d), stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=600)
    assert r.returncode == 0 and "AddressSanitizer" not in r.stderr, r.stdout[-2000:] + r.stderr[-4000:]
    lines = r.stdout.splitlines()
    allocs = {l.split()[1]: int(l.split()[3]) for l in lines if l.startswith("op ")}
    assert list(allocs) == OPS, r.stdout
    # the calls that replace blocks make allocations, so each of them was failed at every one of those
    for op in ("set_views_3", "set_views_4", "set_render_resize", "set_shading", "add_objects_sphere", "add_objects_empty_mesh"):
        assert allocs[op] > 0, (op, r.stdout)
    assert lines[-1] == "live 0", r.stdout
