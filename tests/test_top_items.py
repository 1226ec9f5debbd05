"""The top-level item records the traversal's instance step reads (DevTopItem, crgpu_prepared_top_level), on the CPU.

Each top-level primIndices entry gets one 64-byte record: the instance's Ainv rows, its index with a mesh bit and a "read the mesh's
BVH record" bit, its ray offset, a sphere's radius or the mesh BVH's pair offset, and the mesh BVH's slot offset.  The step trusts
the record instead of following primIndices -> instance -> BVH, so every record must say exactly what those three say, for every
golden and bundled scene, for a scene of about 20,000 instances, and with staged top-of-tree nodes (which send every mesh whose BVH
has staged nodes to its BVH record)."""
import ctypes as C
import os

import numpy as np
import pytest

import crgpu
import crscene
import oracle_lib as O
from conftest import GOLDEN, GOLDEN_FLAT

ITEM = np.dtype([("Ainv", "<f4", 12), ("inst", "<u4"), ("ray_offset", "<f4"), ("shape", "<u4"), ("slot_offset", "<u4")])
DEV_INSTANCE = np.dtype([("Ainv", "<f4", 12), ("A", "<f4", 12), ("kind", "<u4"), ("bvh", "<u4"), ("ray_offset", "<f4"),
                         ("radius", "<f4"), ("material", "<u4"), ("pad", "<u4", 3)])
DEV_BVH = np.dtype([("pair_offset", "<u4"), ("pair_end", "<u4"), ("node_count", "<u4"), ("slot_offset", "<u4"), ("root_first", "<u4"),
                    ("root_count", "<u4"), ("root_bounds", "<f4", 6), ("stage_base", "<u4"), ("stage_count", "<u4"), ("pad", "<u4")])
assert (ITEM.itemsize, DEV_INSTANCE.itemsize, DEV_BVH.itemsize) == (64, 128, 60)
MESH, READ_BVH, INDEX = 1 << 31, 1 << 30, (1 << 30) - 1
CRS_INST_MESH = 1
BUNDLED = ["hdr", "scene", "refraction", "venus", "alphanode", "fence", "glowmetal", "statues", "uvsphere"]


def prepared_top_level(flat):
    """(items, instances, bvhs) of crgpu_prepare(flat), as numpy copies"""
    L = crgpu.lib()
    L.crgpu_prepare.argtypes = [C.POINTER(crgpu.FlatScene), C.POINTER(C.c_void_p)]
    L.crgpu_prepared_free.argtypes = [C.c_void_p]
    L.crgpu_prepared_top_level.argtypes = [C.c_void_p] + [C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)] * 3
    p = C.c_void_p()
    assert L.crgpu_prepare(C.byref(flat), C.byref(p)) == 0
    try:
        ptrs = [C.c_void_p() for _ in range(3)]
        lens = [C.c_size_t() for _ in range(3)]
        assert L.crgpu_prepared_top_level(p, C.byref(ptrs[0]), C.byref(lens[0]), C.byref(ptrs[1]), C.byref(lens[1]),
                                          C.byref(ptrs[2]), C.byref(lens[2])) == 0
        return tuple(np.frombuffer(C.string_at(q, n.value), dtype=dt).copy() if n.value else np.zeros(0, dt)
                     for q, n, dt in zip(ptrs, lens, (ITEM, DEV_INSTANCE, DEV_BVH)))
    finally:
        L.crgpu_prepared_free(p)


def check_items(flat):
    """every record against primIndices, the prepared instance and its mesh's prepared BVH record; returns (items, flagged meshes)"""
    items, insts, bvhs = prepared_top_level(flat)
    a = crscene.arrays(flat)
    top = a["bvhs"][flat.top_bvh]
    prims = a["prim_indices"][top["prim_offset"]:top["prim_offset"] + top["prim_count"]]
    assert len(items) == len(prims) and len(insts) == flat.instance_count
    idx = prims.astype(np.int64)
    inst = insts[idx]
    assert np.array_equal(items["inst"] & INDEX, prims.astype(np.uint32))
    assert np.array_equal(items["Ainv"].view(np.uint32), inst["Ainv"].view(np.uint32))
    assert np.array_equal(items["Ainv"].view(np.uint32), a["instances"]["Ainv"][idx][:, :12].view(np.uint32))
    assert np.array_equal(items["ray_offset"].view(np.uint32), inst["ray_offset"].view(np.uint32))
    mesh = inst["kind"] == CRS_INST_MESH
    assert np.array_equal((items["inst"] & MESH) != 0, mesh)
    sph = ~mesh
    assert np.array_equal(items["shape"][sph], inst["radius"][sph].view(np.uint32))
    assert not items["slot_offset"][sph].any() and not (items["inst"][sph] & READ_BVH).any()
    b = bvhs[inst["bvh"][mesh].astype(np.int64)]
    assert np.array_equal(items["shape"][mesh], b["pair_offset"])
    assert np.array_equal(items["slot_offset"][mesh], b["slot_offset"])
    want_bvh = (b["node_count"] <= 1) | (b["stage_count"] > 0)
    assert np.array_equal((items["inst"][mesh] & READ_BVH) != 0, want_bvh)
    return items, int(want_bvh.sum())


def load_crscene(path):
    f = crgpu.FlatScene()
    assert crgpu.lib().crscene_load(C.byref(f), path.encode()) == 0, path
    return f


def free(f):
    crgpu.lib().crscene_free(C.byref(f))


@pytest.mark.parametrize("name", GOLDEN_FLAT)
def test_golden_scene_items(name):
    f = load_crscene(os.path.join(GOLDEN, name + ".crscene"))
    try:
        items, _ = check_items(f)
        assert len(items) == f.instance_count
    finally:
        free(f)


@pytest.mark.parametrize("name", BUNDLED)
def test_bundled_scene_items(name, tmp_path):
    path = O.bundled_scene(name, str(tmp_path))
    if path is None:
        pytest.skip(f"{name}.json not available")
    f = load_crscene(path)
    try:
        items, flagged = check_items(f)
        assert len(items) == f.instance_count
        if name == "hdr":       # staging is off by default: all but one mesh of hdr.json (a one-node BVH) take their record alone
            meshes = int(((items["inst"] & MESH) != 0).sum())
            assert meshes > 1 and flagged == 1
    finally:
        free(f)


def test_staged_meshes_read_their_bvh(tmp_path, monkeypatch):
    """CRGPU_TRACE_STAGE is read at every prepare: with staged nodes, the meshes whose BVHs have some are sent to their BVH record"""
    path = O.bundled_scene("hdr", str(tmp_path))
    if path is None:
        pytest.skip("hdr.json not available")
    monkeypatch.setenv("CRGPU_TRACE_STAGE", "1024")
    f = load_crscene(path)
    try:
        _, flagged = check_items(f)
        assert flagged > 0
    finally:
        free(f)


def test_many_instance_scene_items():
    """the scene of tests/test_gpu_scene_edit.py::test_many_instances_all_moved: 20,000 spheres of 40 objects and the teapots"""
    from test_gpu_scene_edit import load, sphere_scene, spread, teapots
    f = load(sphere_scene(spread(20000, 1), groups=40, meshes=teapots(), radius=2.0))
    try:
        items, _ = check_items(f)
        assert len(items) == f.instance_count > 20000
        assert (items["inst"] & MESH).any() and not (items["inst"] & MESH).all()
    finally:
        crscene.free(f)
