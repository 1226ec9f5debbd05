"""The traversal kernel (K2) keeps the top CRG_SSTACK entries of every lane's BVH stack in shared memory and the deeper ones in a
thread-local array.  These scenes make the traversal push past that boundary, at the top level alone, in a mesh alone, and in
a mesh behind a top level of spheres.  The depth is counted from the flat scene's BVH, and the records
and P/T/S/I counters of every launch variant must equal the oracle's (device semantics)."""
import json
import os

import numpy as np
import pytest

import crgpu
import oracle_lib as O
from test_gpu_trace import VARIANTS, _flat_arrays, _flatten, _name, check_counters, check_records

SSTACK = 8                      # CRG_SSTACK (crgpu_trace.cuh)
LEAF_BIT, COUNT_MASK = 1 << 30, (1 << 30) - 1
N_QUADS = 32768                 # parallel quads along z: a mesh BVH whose nearest leaf lies well below SSTACK pushes
N_SPHERES = 16384               # spheres along z: the same for the top level


def _quads_obj(path, n, z0=0.0, dz=0.001):
    """n unit quads (two triangles each) perpendicular to z at z0, z0 + dz, ...: a ray along +z through them enters both children
    of every internal node before the first leaf test"""
    lines = ["vn 0 0 -1"]
    for i in range(n):
        z = z0 + dz * i
        lines += ["v -1 -1 %.6f" % z, "v 1 -1 %.6f" % z, "v 1 1 %.6f" % z, "v -1 1 %.6f" % z]
        b = 4 * i + 1
        lines += ["f %d//1 %d//1 %d//1" % (b, b + 1, b + 2), "f %d//1 %d//1 %d//1" % (b, b + 2, b + 3)]
    open(path, "w").write("\n".join(lines) + "\n")


def _spheres(n, z0, dz):
    return [{"type": "sphere", "radius": 0.3, "color": [0.5, 0.5, 0.5],
             "instances": [{"transforms": [{"type": "translate", "Z": z0 + dz * i}]}]} for i in range(n)]


def _scene(d, name, prims, meshes):
    sc = {"renderer": {"width": 32, "height": 32, "samples": 1, "bounces": 2}, "camera": {"FOV": 30},
          "scene": {"ambientColor": {"down": [1, 1, 1], "up": [1, 1, 1]}, "primitives": prims, "meshes": meshes}}
    p = os.path.join(d, name + ".json")
    open(p, "w").write(json.dumps(sc))
    return _flatten(p, os.path.join(d, name + ".crscene"))


@pytest.fixture(scope="module")
def deep_scenes(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("deep"))
    _quads_obj(os.path.join(d, "quads.obj"), N_QUADS)
    return {
        # one mesh instance: the top level is a single leaf, every push is in the mesh BVH
        "mesh": _scene(d, "mesh", [], [{"fileName": "quads.obj", "instances": [{"transforms": [{"type": "translate", "Z": 5}]}]}]),
        # spheres only: every push is in the top-level BVH
        "top": _scene(d, "top", _spheres(N_SPHERES, 5.0, 0.01), []),
        # the mesh in front of a column of spheres: a two-level traversal whose mesh stack crosses the boundary
        "both": _scene(d, "both", _spheres(96, 30.0, 0.5),
                       [{"fileName": "quads.obj", "instances": [{"transforms": [{"type": "translate", "Z": 5}]}]}]),
    }


def _pushes_to_nearest_leaf(f, b, axis_min):
    """pushes of the traversal (one per internal node whose two children are both internal and both entered) on the way from the
    root of BVH b to the leaf it reaches first, for a ray that enters every box and visits the child with the smaller
    axis_min(bounds) first"""
    bvh = f["bvh"][b]
    nodes = f["node"][bvh["node_offset"]:bvh["node_offset"] + bvh["node_count"]]
    i, pushes = 0, 0
    while not (nodes[i]["count"] & LEAF_BIT):
        l, r = int(nodes[i]["first"]), int(nodes[i]["first"]) + 1
        if not (nodes[l]["count"] & LEAF_BIT) and not (nodes[r]["count"] & LEAF_BIT):
            pushes += 1
        i = l if axis_min(nodes[l]["bounds"]) <= axis_min(nodes[r]["bounds"]) else r
    return pushes


def _depths(o):
    """(top-level pushes, largest mesh pushes) on the way to the nearest leaf of a ray along +z, from the oracle's flat scene"""
    f = _flat_arrays(o.s)
    zmin = lambda bnd: bnd[4]                                # noqa: E731  bounds: minx,maxx,miny,maxy,minz,maxz
    top = _pushes_to_nearest_leaf(f, f["top"], zmin)
    mesh = max((_pushes_to_nearest_leaf(f, int(m["bvh"]), zmin) for m in f["mesh"]), default=0)
    return top, mesh


def _rays(n=512, seed=3):
    """rays along +z (slightly tilted) from z = -5 through the column at x, y in (-0.25, 0.25)"""
    rng = np.random.default_rng(seed)
    o = np.column_stack([rng.uniform(-0.25, 0.25, n), rng.uniform(-0.25, 0.25, n), np.full(n, -5.0)])
    d = np.column_stack([rng.uniform(-1e-3, 1e-3, n), rng.uniform(-1e-3, 1e-3, n), np.ones(n)])
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return np.column_stack([o, d]).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["mesh", "top", "both"])
def test_deep_stacks_every_variant(name, deep_scenes):
    path = deep_scenes[name]
    o = O.OracleScene(path)
    top, mesh = _depths(o)
    rays = _rays()
    r1, c1 = o.closest_hit(rays, O.SEM_DEVICE)
    o.close()
    # the BVH walk gives the pushes before the first leaf; the oracle counts the deepest stack any ray reached
    need = {"mesh": top == 0 and mesh > SSTACK, "top": mesh == 0 and top > SSTACK, "both": SSTACK < top + mesh}[name]
    assert need and c1["max_stack"] > SSTACK, f"{name}: no push across the shared/local boundary (top {top}, mesh {mesh}, oracle {c1['max_stack']})"
    assert (r1["inst"] >= 0).mean() > 0.9, f"{name}: most rays must hit"
    g = crgpu.GpuScene(path)
    for kn in VARIANTS:
        rec, perm, misses, st = g.trace_rays(rays, **kn)
        check_records(g, rec, perm, misses, r1, f"deep {name} {_name(kn)}")
        if kn.get("count"):
            check_counters(st, c1, len(rays), f"deep {name} {_name(kn)}")
    g.close()
