"""GPU tests of the traversal kernel that renders every frame (K2, k_trace) and of the bucket sort behind it (K4, k_bucket),
ray by ray, in every launch variant the library can select.

crgpu_trace_rays runs K2 through the same launch path and launch shape as a frame and returns one record per ray.  Each record
must be bit-identical to the oracle's cro_closest_hit in device semantics (semantics 1: the fused slab test and the exact culling
of axes whose 1/d is +-inf, DESIGN.md §2): t, instance and polygon for every ray, u and v for mesh hits, and the shading key.
Under the instrumented variant the P/T/S/I totals must equal the oracle's exactly: both visit the same nodes in the same order.

The rays are the rays of real paths (every bounce, from the oracle's event trace), adversarial rays built from each scene's
geometry (exact ties at shared vertices and edge midpoints, origins on triangles and on BVH box faces, +0 / -0 / denormal
direction components, origins far outside the world, rays that miss), and synthetic scenes that reach edges no bundled scene
does (tied instances and spheres, 300 materials, an oversized leaf, single-leaf BVHs).

The last part renders whole frames once per environment setting (one process each: the frame path reads its knobs once) and
requires the bits of the default run.
"""
import ctypes as C
import json
import os
import subprocess
import sys

import random

import numpy as np
import pytest

import crgpu
import oracle_lib as O
from conftest import GOLDEN, GOLDEN_FLAT, ROOT, SUMMARY_LINES
from test_loader import _write_obj

pytestmark = pytest.mark.gpu
FLT_MAX = np.float32(np.finfo(np.float32).max)
FLT_MIN = np.float32(np.finfo(np.float32).tiny)
STAGE_MIN_RAYS = 65536          # CRG_STAGE_MIN_RAYS: K2 stages the top BVH nodes only for launches of at least this many rays
BUNDLED = ["hdr", "venus", "refraction", "fence", "statues"]

# launch variants of K2 (crgpu_trace_opts); together they take every value of every knob
VARIANTS = [
    dict(),
    dict(defer=1, burst=4), dict(defer=2, burst=4),
    dict(minb=2), dict(minb=4), dict(minb=2, defer=2, burst=4), dict(minb=4, defer=1, burst=4),
    dict(count=1), dict(count=1, defer=1, burst=4), dict(count=1, defer=2, burst=4),
    dict(refill=1), dict(refill=32), dict(refill=1, defer=2, burst=4), dict(refill=32, defer=2, burst=1),
    dict(burst=1), dict(burst=8), dict(burst=8, defer=2),
    dict(inst_min=1), dict(inst_min=32), dict(inst_min=32, defer=2, burst=4), dict(inst_min=1, defer=1, burst=1),
]


def _name(kn):
    return ",".join(f"{k}={v}" for k, v in sorted(kn.items())) or "default"


# ------------------------------------------------------------------------------------------------ scenes
def _flat_arrays(s):
    """numpy views of the flat scene's geometry (struct crs_scene, include/crscene.h)"""
    def arr(ptr, count, dtype):
        dtype = np.dtype(dtype)
        if count == 0 or not ptr:
            return np.zeros(0, dtype)
        return np.frombuffer((C.c_uint8 * (count * dtype.itemsize)).from_address(ptr), dtype=dtype).copy()
    inst_t = np.dtype([("A", "<f4", 16), ("Ainv", "<f4", 16), ("kind", "<u4"), ("object", "<u4"), ("pad", "<u4", 2)])
    mesh_t = np.dtype([("poly_offset", "<u4"), ("poly_count", "<u4"), ("material_offset", "<u4"), ("material_count", "<u4"),
                       ("texcoord_count", "<u4"), ("bvh", "<u4"), ("ray_offset", "<f4"), ("pad", "<u4")])
    poly_t = np.dtype([("v", "<i4", 3), ("n", "<i4", 3), ("t", "<i4", 3), ("material", "<u4"), ("has_normals", "<u4")])
    node_t = np.dtype([("bounds", "<f4", 6), ("first", "<u4"), ("count", "<u4")])
    bvh_t = np.dtype([("node_offset", "<u4"), ("node_count", "<u4"), ("prim_offset", "<u4"), ("prim_count", "<u4")])
    return dict(inst=arr(s.instances, s.instance_count, inst_t), mesh=arr(s.meshes, s.mesh_count, mesh_t),
                poly=arr(s.polys, s.poly_count, poly_t), vert=arr(s.vertices, s.vertex_count * 3, "<f4").reshape(-1, 3),
                node=arr(s.bvh_nodes, s.bvh_node_count, node_t), bvh=arr(s.bvhs, s.bvh_count, bvh_t), top=s.top_bvh,
                prims=arr(s.prim_indices, s.prim_index_count, "<i4"))


LEAF_BIT, COUNT_MASK = 1 << 30, (1 << 30) - 1


def _leaf_boxes(f, m):
    """per local poly of mesh m: the bounds of its leaf box in the mesh BVH (minx, maxx, miny, maxy, minz, maxz)"""
    out = np.zeros((m["poly_count"], 6), np.float32)
    b = f["bvh"][m["bvh"]]
    nodes = f["node"][b["node_offset"]:b["node_offset"] + b["node_count"]]
    prims = f["prims"][b["prim_offset"]:b["prim_offset"] + b["prim_count"]]
    leaves = nodes if len(nodes) == 1 else nodes[(nodes["count"] & LEAF_BIT) != 0]   # a one-node BVH is a leaf (bvh.c:382-387)
    cnt = (leaves["count"] & COUNT_MASK).astype(np.int64)
    leaf = np.repeat(np.arange(len(leaves)), cnt)
    slot = leaves["first"].astype(np.int64)[leaf] + np.arange(len(leaf)) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    out[prims[slot]] = leaves["bounds"][leaf]
    return out


def _world_triangles(f):
    """(n, 3, 3) world-space vertices of every mesh instance's triangles (targets only: exact rounding does not matter), and per
    triangle and vertex the axes on which that vertex lies on a face of the triangle's leaf box (object space, exact): bit a for
    the low face, bit 3 + a for the high face"""
    out, face = [], []
    for inst in f["inst"]:
        if inst["kind"] != 1:
            continue
        m = f["mesh"][inst["object"]]
        p = f["poly"][m["poly_offset"]:m["poly_offset"] + m["poly_count"]]
        if len(p) == 0:
            continue
        v = f["vert"][p["v"].ravel()].astype(np.float64)
        A = inst["A"].reshape(4, 4).astype(np.float64)
        w = v @ A[:3, :3].T + A[:3, 3]
        out.append(w.reshape(-1, 3, 3))
        ov = f["vert"][p["v"]]                                             # (polys, 3 vertices, 3 axes), object space
        box = _leaf_boxes(f, m)[:, None, :]
        bits = np.zeros(ov.shape[:2], np.int64)
        for a in range(3):
            bits |= (ov[:, :, a] == box[:, :, 2 * a]).astype(np.int64) << a
            bits |= (ov[:, :, a] == box[:, :, 2 * a + 1]).astype(np.int64) << (3 + a)
        face.append(bits)
    return (np.concatenate(out), np.concatenate(face)) if out else (np.zeros((0, 3, 3)), np.zeros((0, 3), np.int64))


def _unit(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def adversarial_rays(o, rng, n=512):
    """Rays built from the scene's geometry, by class: tie / on_tri / on_box / degenerate / tiny / far / miss.  Also returns, per
    ray, whether it is aimed at a vertex or an edge that lies on a face of its triangle's leaf box."""
    f = _flat_arrays(o.s)
    top = f["bvh"][f["top"]]
    nodes = f["node"][top["node_offset"]:top["node_offset"] + top["node_count"]]
    if len(nodes) == 0:
        return np.zeros((0, 6), np.float32), np.zeros(0, "U10"), np.zeros(0, bool)
    root = nodes["bounds"][0].astype(np.float64)
    lo, hi = root[0::2], root[1::2]
    centre, ext = (lo + hi) / 2, np.maximum(hi - lo, 1e-3)
    tris, tri_face = _world_triangles(f)
    rays, cls, flat = [], [], []

    def add(org, d, c, fl=None):
        r = np.concatenate([org, d], axis=1).astype(np.float32)
        rays.append(r)
        cls.extend([c] * len(r))
        flat.append(np.zeros(len(r), bool) if fl is None else fl)

    def around(k):                      # origins outside the world box, on a sphere around it
        return centre + _unit(rng.normal(size=(k, 3))) * (np.linalg.norm(ext) * rng.uniform(0.6, 2.0, (k, 1)))

    if len(tris):
        ti = rng.integers(0, len(tris), n)
        pick = tris[ti]
        w = rng.integers(0, 3, n)
        vert = pick[np.arange(n), w]                                     # shared vertices
        mid = (pick[np.arange(n), w] + pick[np.arange(n), (w + 1) % 3]) / 2   # edge midpoints
        cen = pick.mean(axis=1)
        tgt = np.concatenate([vert[: n // 2], mid[: n // 2]])
        org = around(len(tgt))
        h = n // 2
        on_vert = tri_face[ti[:h], w[:h]] != 0
        on_edge = (tri_face[ti[:h], w[:h]] & tri_face[ti[:h], (w[:h] + 1) % 3]) != 0     # both ends on the same face
        add(org, _unit(tgt - org), "tie", np.concatenate([on_vert, on_edge]))
        k = n // 3
        org = np.concatenate([vert[:k], mid[:k], cen[:k]])                # t = 0 on a triangle
        add(org, _unit(rng.normal(size=(len(org), 3))), "on_tri")
    # origins on faces of the top-level boxes, directions random and along the face (one component +0 / -0)
    bx = nodes["bounds"][rng.integers(0, len(nodes), n)].astype(np.float64)
    axis = rng.integers(0, 3, n)
    side = rng.integers(0, 2, n)
    org = bx[:, 0::2] + rng.uniform(0, 1, (n, 3)) * (bx[:, 1::2] - bx[:, 0::2])
    org[np.arange(n), axis] = bx[np.arange(n), 2 * axis + side]
    org = org.astype(np.float32)
    d = _unit(rng.normal(size=(n, 3)))
    add(org, d, "on_box")
    d2 = d.copy().astype(np.float32)
    d2[np.arange(n), axis] = np.where(rng.integers(0, 2, n) == 1, np.float32(-0.0), np.float32(0.0))
    add(org, d2, "on_box")
    # +0 / -0 / denormal direction components from inside and outside the world
    org = np.concatenate([around(n // 2), centre + (rng.uniform(-0.5, 0.5, (n - n // 2, 3)) * ext)])
    d = _unit(centre - org + rng.normal(size=(n, 3)) * ext * 0.2).astype(np.float32)
    special = np.array([0.0, -0.0, 1e-45, -1e-45, 1e-40, -3e-39, 1.1754942e-38], np.float32)
    for j in range(n):
        for a in rng.choice(3, size=rng.integers(1, 3), replace=False):
            d[j, a] = special[rng.integers(0, len(special))]
    add(org, d, "degenerate")
    # tiny NORMAL direction components: 1/d is finite but o*(1/d) can overflow (the fused slab test alone would give -inf there)
    org = np.concatenate([around(n // 2), centre + (rng.uniform(-0.5, 0.5, (n - n // 2, 3)) * ext)])
    d = _unit(centre - org + rng.normal(size=(n, 3)) * ext * 0.2).astype(np.float32)
    tiny = np.array([1.1754944e-38, -1.1754944e-38, 3e-38, -2e-37, 2e-37, 1e-36, -5e-36], np.float32)
    for j in range(n):
        d[j, rng.integers(0, 3)] = tiny[rng.integers(0, len(tiny))]
    add(org, d, "tiny")
    # origins far outside the world box, aimed at it, and rays that miss everything
    org = centre + _unit(rng.normal(size=(n, 3))) * np.linalg.norm(ext) * 1e4
    add(org, _unit(centre + rng.uniform(-0.5, 0.5, (n, 3)) * ext - org), "far")
    org = around(n)
    add(org, _unit(org - centre), "miss")
    return np.concatenate(rays), np.array(cls), np.concatenate(flat)


def _write_synthetic(d):
    """JSON + OBJ scenes for edges no bundled scene reaches; returns {name: json path}"""
    os.makedirs(d, exist_ok=True)
    cam = {"FOV": 70}
    out = {}

    def scene(name, prims, meshes, w=64, h=48, spp=4, bounces=6):
        sc = {"renderer": {"width": w, "height": h, "samples": spp, "bounces": bounces}, "camera": cam,
              "scene": {"ambientColor": {"down": [1, 1, 1], "up": [0.5, 0.7, 1.0]}, "primitives": prims, "meshes": meshes}}
        p = os.path.join(d, name + ".json")
        open(p, "w").write(json.dumps(sc))
        out[name] = p

    # a quad of two triangles, instanced twice at the same transform (tie on instance order), coplanar duplicate faces of
    # different materials (tie on polygon order), two coincident spheres (t <= distance: the later one wins) and 48 copies of
    # one face (one leaf of more than 32 triangles: the oversized-leaf fallback of the cooperative leaf phase)
    open(os.path.join(d, "quad.mtl"), "w").write("newmtl a\nKd 0.8 0.2 0.2\nnewmtl b\nKd 0.2 0.8 0.2\n")
    open(os.path.join(d, "quad.obj"), "w").write("mtllib quad.mtl\nv -1 -1 0\nv 1 -1 0\nv 1 1 0\nv -1 1 0\nvn 0 0 -1\nusemtl a\n"
                                                 "f 1//1 2//1 3//1\nf 1//1 3//1 4//1\nusemtl b\nf 1//1 2//1 3//1\nf 1//1 3//1 4//1\n")
    big = ["v %.4f %.4f %.4f" % (np.cos(a), np.sin(a), 0.1 * np.sin(3 * a)) for a in np.linspace(0, 6, 12)]
    big += ["vn 0 0 -1"] + ["f 1//1 5//1 9//1"] * 48 + ["f %d//1 %d//1 %d//1" % (i, i + 1, i + 2) for i in range(1, 10)]
    open(os.path.join(d, "bigleaf.obj"), "w").write("\n".join(big) + "\n")
    # a random mesh of the loader tests (vertex normals, repeated faces) instanced twice at the same transform; without texture
    # coordinates, because that generator mixes faces with and without them, which the device upload rejects
    _write_obj(random.Random(11), os.path.join(d, "fuzz.obj"), None, False, True, [])
    tr = [{"type": "translate", "Z": 4}]
    fz = [{"type": "translate", "Y": -1.2, "Z": 6}]
    scene("syn_ties", [{"type": "sphere", "radius": 0.5, "color": [0.9, 0.1, 0.1], "instances": [{"transforms": [{"type": "translate", "X": 1.5, "Z": 5}]}]},
                       {"type": "sphere", "radius": 0.5, "color": [0.1, 0.1, 0.9], "instances": [{"transforms": [{"type": "translate", "X": 1.5, "Z": 5}]}]}],
          [{"fileName": "quad.obj", "instances": [{"transforms": tr}, {"transforms": tr}]},
           {"fileName": "bigleaf.obj", "instances": [{"transforms": [{"type": "translate", "X": -1.5, "Z": 5}]}]},
           {"fileName": "fuzz.obj", "instances": [{"transforms": fz}, {"transforms": fz}]}])
    # 300 spheres, each with its own material: keys saturate at 255 (materials >= 254 share one K3 bucket)
    prims = []
    for i in range(300):
        x, y = i % 20, i // 20
        prims.append({"type": "sphere", "radius": 0.09, "color": [(i % 7) / 7, (i % 11) / 11, (i % 13) / 13],
                      "instances": [{"transforms": [{"type": "translate", "X": (x - 9.5) * 0.2, "Y": (y - 7) * 0.2, "Z": 4}]}]})
    scene("syn_materials", prims, [], w=96, h=72)
    # one sphere: the top-level BVH is a single leaf; one triangle: so is its mesh BVH
    open(os.path.join(d, "one.obj"), "w").write("v -1 -1 0\nv 1 -1 0\nv 0 1 0\nvn 0 0 -1\nf 1//1 2//1 3//1\n")
    scene("syn_single", [{"type": "sphere", "radius": 1.0, "color": [0.5, 0.5, 0.5], "instances": [{"transforms": [{"type": "translate", "Z": 6}]}]}], [])
    scene("syn_onetri", [], [{"fileName": "one.obj", "instances": [{"transforms": [{"type": "translate", "Z": 3}]}]}])
    return out


def _flatten(json_path, out):
    import crscene
    flat = crscene.load_json(json_path)
    L = crgpu.lib()
    L.crscene_save.argtypes = [C.POINTER(crgpu.FlatScene), C.c_char_p]
    rc = L.crscene_save(C.byref(flat), out.encode())
    crscene.free(flat)
    assert rc == 0, f"crscene_save({out}) failed ({rc})"
    return out


@pytest.fixture(scope="module")
def scenes(tmp_path_factory):
    """name -> flat .crscene path: the golden scenes, the bundled ones where oracle/_ref/input exists, the synthetic ones"""
    d = str(tmp_path_factory.mktemp("scenes"))
    out = {n: os.path.join(GOLDEN, n + ".crscene") for n in GOLDEN_FLAT}
    for n in BUNDLED:
        p = O.bundled_scene(n, d)
        if p:
            out[n] = p
    for n, p in _write_synthetic(os.path.join(d, "syn")).items():
        out[n] = _flatten(p, os.path.join(d, n + ".crscene"))
    return out


_RAYSETS = {}


def raysets(name, path):
    """(rays, class, oracle mode-1 records, mode-1 counters, mode-0 records, aimed-at-a-leaf-face flags) of a scene, built once per
    session (seeded)"""
    if name in _RAYSETS:
        return _RAYSETS[name]
    o = O.OracleScene(path)
    rng = np.random.default_rng(sum(map(ord, name)))
    W, H = o.W, o.H
    # every ray of every bounce of the paths of a block of pixels (the whole image for the small scenes)
    bw, bh = min(W, 48), min(H, 32)
    x0, y0 = (W - bw) // 2, (H - bh) // 2
    p = o.path_rays(x0, y0, x0 + bw, y0 + bh, passes=(0, min(2, o.s.prefs.sample_count)))
    a, ac, af = adversarial_rays(o, rng)
    rays = np.concatenate([p, a]).astype(np.float32)
    cls = np.concatenate([np.array(["path"] * len(p)), ac])
    flat = np.concatenate([np.zeros(len(p), bool), af])
    r1, c1 = o.closest_hit(rays, O.SEM_DEVICE)
    r0, _ = o.closest_hit(rays, O.SEM_REFERENCE)
    o.close()
    _RAYSETS[name] = (rays, cls, r1, c1, r0, flat)
    return _RAYSETS[name]


def expected_key(rec):
    return np.where(rec["inst"] >= 0, np.minimum(rec["material"] + 1, 255), 0).astype(np.uint32)


def check_records(g, rec, perm, misses, exp, what):
    """GPU records vs oracle mode-1 records, bit for bit, plus the K4 invariants"""
    n = len(exp)
    assert len(rec) == n
    assert not (rec["inst"] < -1).any(), f"{what}: poisoned records left: {np.count_nonzero(rec['inst'] < -1)}"
    bad = np.nonzero(rec["inst"] != exp["inst"])[0]
    assert len(bad) == 0, f"{what}: instance differs on {len(bad)} rays, first {bad[:5]}: gpu {rec['inst'][bad[:5]]} oracle {exp['inst'][bad[:5]]}"
    bad = np.nonzero(rec["t"].view(np.uint32) != exp["t"].view(np.uint32))[0]
    assert len(bad) == 0, f"{what}: t differs on {len(bad)} rays, first {bad[:5]}: gpu {rec['t'][bad[:5]]} oracle {exp['t'][bad[:5]]}"
    bad = np.nonzero(rec["poly"] != exp["poly"])[0]
    assert len(bad) == 0, f"{what}: poly differs on {len(bad)} rays, first {bad[:5]}: gpu {rec['poly'][bad[:5]]} oracle {exp['poly'][bad[:5]]}"
    mesh = exp["poly"] >= 0
    for f in ("u", "v"):
        bad = np.nonzero(rec[f][mesh].view(np.uint32) != exp[f][mesh].view(np.uint32))[0]
        assert len(bad) == 0, f"{what}: {f} differs on {len(bad)} mesh hits"
    key = expected_key(exp)
    bad = np.nonzero(rec["key"] != key)[0]
    assert len(bad) == 0, f"{what}: key differs on {len(bad)} rays, first {bad[:5]}: gpu {rec['key'][bad[:5]]} expected {key[bad[:5]]}"
    # K4: perm is a permutation of [0, n), keys never decrease along it, and its first `misses` entries are exactly the misses
    assert np.array_equal(np.sort(perm), np.arange(n, dtype=np.uint32)), f"{what}: perm is not a permutation"
    assert (np.diff(key[perm].astype(np.int64)) >= 0).all(), f"{what}: keys decrease along perm"
    assert misses == int((exp["inst"] < 0).sum()), what
    assert (exp["inst"][perm[:misses]] < 0).all(), what


def check_counters(st, c1, n, what):
    assert st["rays"] == n, (what, st["rays"], n)
    for k in ("node_pairs", "tri_tests", "sphere_tests", "inst_visits"):
        assert st[k] == c1[k], f"{what}: {k} gpu {st[k]} oracle (device semantics) {c1[k]}"


# ------------------------------------------------------------------------------------------------ records, every variant
SCENE_NAMES = GOLDEN_FLAT + BUNDLED + ["syn_ties", "syn_materials", "syn_single", "syn_onetri"]


@pytest.mark.parametrize("name", SCENE_NAMES)
def test_trace_records_every_variant(name, scenes):
    if name not in scenes:
        pytest.skip(f"{name}: bundled scenes need oracle/_ref/input")
    rays, cls, r1, c1, r0, flat = raysets(name, scenes[name])
    g = crgpu.GpuScene(scenes[name])
    rng = np.random.default_rng(7)
    orders = {"shuffled": rng.permutation(len(rays)).astype(np.uint32),
              "octant": np.argsort((rays[:, 3] < 0) * 1 + (rays[:, 4] < 0) * 2 + (rays[:, 5] < 0) * 4, kind="stable").astype(np.uint32)}
    for kn in VARIANTS:
        rec, perm, misses, st = g.trace_rays(rays, **kn)
        check_records(g, rec, perm, misses, r1, f"{name} {_name(kn)}")
        if kn.get("count"):
            check_counters(st, c1, len(rays), f"{name} {_name(kn)}")
    for oname, order in orders.items():
        for kn in (dict(), dict(defer=2, burst=4), dict(count=1, defer=1, burst=4)):
            rec, perm, misses, st = g.trace_rays(rays, order=order, **kn)
            check_records(g, rec, perm, misses, r1, f"{name} order={oname} {_name(kn)}")
            if kn.get("count"):
                check_counters(st, c1, len(rays), f"{name} order={oname} {_name(kn)}")
    g.close()
    # semantics 0 (the reference) vs 1 (the device): per ray class, records that differ
    diff = (r0.view(np.uint8).reshape(len(r0), -1) != r1.view(np.uint8).reshape(len(r1), -1)).any(axis=1)
    counts = {c: f"{int(diff[cls == c].sum())}/{int((cls == c).sum())}" for c in np.unique(cls)}
    line = f"trace records, reference vs device semantics, {name}: " + " ".join(f"{c} {v}" for c, v in sorted(counts.items()))
    print(line)
    SUMMARY_LINES.append(line)
    assert not diff[cls == "path"].any(), line
    # a difference is allowed only (1) where an axis is culled exactly: -o/d not finite (a +-0 or denormal component, or o*(1/d)
    # overflows), (2) for an origin on a box face, (3) for a ray aimed exactly at a vertex or edge of a triangle that
    # lies on a face of that triangle's leaf box (every point of a leaf of zero thickness does): the ray meets the face exactly
    # at the tie point, and the fused and the two-rounding slab test can disagree by an ulp on entering the box (DESIGN.md §2)
    with np.errstate(all="ignore"):
        culled = ~np.isfinite(-(rays[:, :3] * (np.float32(1) / rays[:, 3:]))).all(axis=1)
    allowed = culled | (cls == "on_box") | ((cls == "tie") & flat)
    assert not (diff & ~allowed).any(), (line, np.nonzero(diff & ~allowed)[0][:8])


# ------------------------------------------------------------------------------------------------ staging and batch sizes
def _pool(name, scenes, n):
    rays, cls, r1, c1, r0, _ = raysets(name, scenes[name])
    idx = np.resize(np.arange(len(rays)), n)
    return rays[idx], idx, r1


def _stage_scene(scenes):
    return "hdr" if "hdr" in scenes else "g_nodes"


@pytest.mark.parametrize("stage", [0, 128, 1024])
def test_staged_top_nodes(stage, scenes, monkeypatch):
    """CRGPU_TRACE_STAGE=<pairs> copies the top BVH nodes into shared memory (cp.async.bulk + mbarrier) for launches of at least
    65,536 rays: the records of every leaf variant and the counters must not change."""
    monkeypatch.setenv("CRGPU_TRACE_STAGE", str(stage))
    name = _stage_scene(scenes)
    rays, idx, r1 = _pool(name, scenes, 1 << 18)
    exp = r1[idx]
    o = O.OracleScene(scenes[name])
    _, c1 = o.closest_hit(rays, O.SEM_DEVICE)
    o.close()
    g = crgpu.GpuScene(scenes[name])
    for kn in (dict(), dict(defer=1, burst=4), dict(defer=2, burst=4), dict(minb=2), dict(minb=4, refill=32),
               dict(count=1), dict(count=1, defer=2, burst=4)):
        rec, perm, misses, st = g.trace_rays(rays, **kn)
        check_records(g, rec, perm, misses, exp, f"{name} stage={stage} {_name(kn)}")
        if kn.get("count"):
            check_counters(st, c1, len(rays), f"{name} stage={stage} {_name(kn)}")
    g.close()


@pytest.mark.parametrize("n", [0, 1, 31, 33, STAGE_MIN_RAYS - 1, STAGE_MIN_RAYS, STAGE_MIN_RAYS + 1, 1 << 18])
def test_batch_sizes(n, scenes, monkeypatch):
    """Warp-partial, single-ray, empty and staging-threshold batches (staging on: 128 pairs)."""
    monkeypatch.setenv("CRGPU_TRACE_STAGE", "128")
    name = _stage_scene(scenes)
    rays, idx, r1 = _pool(name, scenes, n)
    g = crgpu.GpuScene(scenes[name])
    for kn in (dict(), dict(defer=2, burst=4)):
        rec, perm, misses, st = g.trace_rays(rays, **kn)
        check_records(g, rec, perm, misses, r1[idx], f"{name} n={n} {_name(kn)}")
        assert st["rays"] == n
    g.close()


def test_trace_rays_rejects_bad_options(scenes):
    g = crgpu.GpuScene(scenes["g_single"])
    rays = np.zeros((4, 6), np.float32)
    rays[:, 5] = 1.0
    for kn in (dict(minb=1), dict(defer=3), dict(refill=0), dict(refill=33), dict(burst=0), dict(inst_min=0)):
        with pytest.raises(crgpu.CrgpuError):
            g.trace_rays(rays, **kn)
    with pytest.raises(crgpu.CrgpuError):
        g.trace_rays(rays, order=np.array([0, 1, 1, 3], np.uint32))      # not a permutation: rejected before any launch
    g.close()


# ------------------------------------------------------------------------------------------------ whole frames
FRAME_ENVS = [{"CRGPU_TRACE_DEFER": "1"}, {"CRGPU_TRACE_DEFER": "2"}, {"CRGPU_TRACE_STAGE": "128"}, {"CRGPU_TRACE_STAGE": "1024"},
              {"CRGPU_TRACE_SORT": "1"}, {"CRGPU_TRACE_SORT": "2"}, {"CRGPU_TRACE_SORT": "3"},
              {"CRGPU_TRACE_MINB": "2"}, {"CRGPU_TRACE_MINB": "4"}, {"CRGPU_TRACE_REFILL": "1"}, {"CRGPU_TRACE_REFILL": "32"},
              {"CRGPU_TRACE_BURST": "1"}, {"CRGPU_TRACE_BURST": "8"}, {"CRGPU_TRACE_INSTMIN": "1"}, {"CRGPU_TRACE_INSTMIN": "32"},
              {"CRGPU_SHADE_SPLIT": "0"}, {"CRGPU_SHADE_MINB": "2"}, {"CRGPU_SHADE_MINB": "4"}, {"CRGPU_SHADE_PREFETCH": "1"},
              {"CRGPU_OVERLAP": "0"}]
_FRAME_CODE = r"""
import hashlib, json, sys
sys.path[:0] = sys.argv[1:3]
import numpy as np, crgpu
out = {}
for name, path, W, H, spp, b, mp in json.loads(sys.argv[3]):
    g = crgpu.GpuScene(path, W, H, spp, b)
    if mp:
        g.set_max_paths(mp)            # several batches per frame: the two-stream overlap engages
    g.render_frame()
    out[name] = hashlib.sha256(g.read().tobytes()).hexdigest()
    g.close()
print("FRAMES " + json.dumps(out))
"""


def _frames(env, jobs):
    e = {k: v for k, v in os.environ.items() if not k.startswith("CRGPU_")}
    e.update(env)
    r = subprocess.run([sys.executable, "-c", _FRAME_CODE, os.path.join(ROOT, "c-ray_b200"), os.path.join(ROOT, "tests"), json.dumps(jobs)],
                       env=e, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("FRAMES ")]
    assert r.returncode == 0 and lines, r.stdout[-2000:]
    return json.loads(lines[-1][7:])


def test_frame_variants_are_bit_identical(scenes):
    """Every K2 / K3 / driver setting renders the frame of the default setting, bit for bit: g_nodes, g_f4 (the complete node
    interpreter in K3 and the tail kernel), hdr at 240x135x16 with 32 bounces (>= 65,536 rays per K2, so staging engages) and
    refraction at 240x135x8 with 512 bounces (the tail kernel)."""
    jobs = [["g_nodes", scenes["g_nodes"], 0, 0, 0, 0, 0], ["g_f4", scenes["g_f4"], 0, 0, 0, 0, 0]]
    if "hdr" in scenes:
        jobs.append(["hdr", scenes["hdr"], 240, 135, 16, 32, 240 * 135 * 4])
    if "refraction" in scenes:
        jobs.append(["refraction", scenes["refraction"], 240, 135, 8, 512, 0])
    base = _frames({}, jobs)
    bad = []
    for env in FRAME_ENVS:
        got = _frames(env, jobs)
        bad += [(env, k) for k in base if got[k] != base[k]]
    assert not bad, bad


def test_key_saturation_frame_vs_oracle(scenes):
    """300 sphere materials: materials 254.. share K3 bucket 255, whose warps shade many materials; the frame is held to the
    RMSE bound against the oracle."""
    if "syn_materials" not in scenes:
        pytest.skip("synthetic scene not loadable")
    path = scenes["syn_materials"]
    g = crgpu.GpuScene(path)
    g.render_frame()
    img = g.read()
    g.close()
    o = O.OracleScene(path)
    ref = o.render(threads=os.cpu_count())
    o.close()
    rays, cls, r1, c1, r0, _ = raysets("syn_materials", path)
    assert (r1["material"] >= 254).sum() > 100              # many hits land in the saturated bucket
    rmse = float(np.sqrt(((img.astype(np.float64) - ref) ** 2).mean()))
    assert np.isfinite(img).all() and rmse <= 1e-4, rmse
