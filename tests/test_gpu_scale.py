"""Tests at the sizes only full-size frames reach: branches of the BVH builder, the traversal kernel, the tile list and the tile
gather that small inputs never take.

  A  the device BVH build's third prefix-sum level.  scan64 (crgpu_bvh_build.cu) scans 1,024 elements per block, then the block
     sums, then, above 1,048,576 primitives, the sums of those (up to 4,194,304 primitives, the builder's limit).  Every partition
     is decided by these sums, so a wrong carry gives a different tree, not a crash.  Mixed box sets at 2^20, 2^20 + 1, 2.5 M and
     2^22 must give the host builder's tree; 2^22 + 1 is refused, and the loader then builds on the host.
  B  a 1.2 M-triangle mesh (its device-built BVH also goes through the third level) through K2 in every launch variant, ray by ray
     against the oracle, and through a whole frame.
  C  leaves of 65,535, 65,536 and 70,000 triangles.  K2's deferred and cooperative leaf phases pack two leaf counts into 16 bits
     each and fall back to the direct leaf loop for larger leaves (crgpu_trace.cuh, node_step).
  D  tile sets of 40,000 to 70,000 rectangles: k_pixel_list runs in launches of 32,768 rectangles (gridDim.y <= 65,535).
  E  the NCCL tile gather with more than 65,535 tiles per peer: k_tiles_copy runs in launches of 32,768 tiles (two GPUs).

Host trees are built once per module and their build times are printed.
"""
import ctypes as C
import json
import os
import subprocess
import time

import numpy as np
import pytest

import crgpu
import crscene
import oracle_lib as O
from conftest import GOLDEN, ROOT, SUMMARY_LINES
from test_bvh_build import check_tree, mesh_inputs, same_tree
from test_gpu_shade import Tally
from test_gpu_trace import VARIANTS, _flatten, _name, adversarial_rays, check_counters, check_records
from test_oracle import same_bits

CRGPU_ERR_UNSUPPORTED, CRGPU_ERR_NOMEM = -4, -5         # include/crgpu.h
BUILD_LIMIT = 1 << 22                                    # crgpu_bvh_build: primitives per call
SCAN_SIZES = [1 << 20, (1 << 20) + 1, 2_500_000, BUILD_LIMIT]
BINS_BYTES, REC_BYTES = 4992, 116                        # sizeof(Bins), sizeof(Rec) in crgpu_bvh_build.cu
STAGE_MIN_RAYS = 65536                                   # K2 stages the top BVH nodes only for launches of at least this many rays
BIG_LEAVES = [65535, 65536, 70000]


def _note(line):
    print(line)
    SUMMARY_LINES.append(line)


def _device_build(bb, ct):
    """crgpu_bvh_build -> (return code, nodes, prims), without raising"""
    G = crgpu.lib()
    G.crgpu_bvh_build.restype = C.c_int
    return crscene._build(G.crgpu_bvh_build, bb, ct, C.c_int(0))


def _scratch_bytes(n):
    """the device builder's scratch for n primitives, as crgpu_bvh_build computes it (it asks for twice this much free)"""
    return (n // 2 + 1) * BINS_BYTES + 2 * n * REC_BYTES + n * 96


def _write_obj(path, verts, faces):
    """OBJ of float vertices and 0-based triangles with one shared normal (the loader takes v, v/vt/vn or v//vn), in bulk"""
    with open(path, "w") as f:
        f.write("".join(map("v %.6f %.6f %.6f\n".__mod__, map(tuple, np.asarray(verts, np.float64).tolist()))))
        f.write("vn 0 0 -1\n")
        f.write("".join(map("f %d//1 %d//1 %d//1\n".__mod__, map(tuple, (np.asarray(faces, np.int64) + 1).tolist()))))


def _write_scene(d, name, meshes, prims=(), w=64, h=48, spp=2, bounces=4):
    """JSON scene of OBJ meshes [(file, translate xyz)] and spheres; camera at the origin looking down +z"""
    sc = {"renderer": {"width": w, "height": h, "samples": spp, "bounces": bounces}, "camera": {"FOV": 70},
          "scene": {"ambientColor": {"down": [1, 1, 1], "up": [0.5, 0.7, 1.0]}, "primitives": list(prims),
                    "meshes": [{"fileName": f, "instances": [{"transforms": [{"type": "translate", "X": t[0], "Y": t[1], "Z": t[2]}]}]}
                               for f, t in meshes]}}
    p = os.path.join(d, name + ".json")
    with open(p, "w") as f:
        f.write(json.dumps(sc))
    return p


def _grid(nx, ny, size, z, amp, rng):
    """displaced height field of nx x ny cells, two triangles per cell"""
    x, y = np.meshgrid(np.linspace(-size[0], size[0], nx + 1), np.linspace(-size[1], size[1], ny + 1))
    zz = z + amp * np.sin(3 * x) * np.cos(2 * y) + rng.uniform(-0.02, 0.02, x.shape)
    verts = np.stack([x, y, zz], -1).reshape(-1, 3)
    i, j = np.meshgrid(np.arange(nx), np.arange(ny))
    v00 = (j * (nx + 1) + i).ravel()
    v10, v01 = v00 + 1, v00 + nx + 1
    faces = np.concatenate([np.stack([v00, v10, v01 + 1], 1), np.stack([v00, v01 + 1, v01], 1)])
    return verts, faces


# ================================================================================================ A: BVH build past two scan levels
def mixed_boxes(n):
    """n boxes, shuffled so that every class sits in every scan block: a uniform half, a tight cluster, blocks of 64 duplicates
    and a plane of flat boxes at z = +0 / -0"""
    rng = np.random.default_rng(n)
    nu, nc, nd = n // 2, n // 4, n // 8
    nz = n - nu - nc - nd
    c_u, e_u = rng.uniform(-100, 100, (nu, 3)), rng.uniform(0, 0.5, (nu, 3))
    c_c, e_c = rng.normal(20, 1e-3, (nc, 3)), rng.uniform(0, 1e-3, (nc, 3))
    blocks = (nd + 63) // 64
    c_d = np.repeat(rng.uniform(-60, 60, (blocks, 3)), 64, axis=0)[:nd]
    e_d = np.repeat(rng.uniform(0.01, 0.2, (blocks, 3)), 64, axis=0)[:nd]
    c_z = np.concatenate([rng.integers(-512, 512, (nz, 2)) / 8.0, np.where(rng.integers(0, 2, (nz, 1)) == 1, -0.0, 0.0)], 1)
    e_z = np.concatenate([rng.uniform(0, 0.1, (nz, 2)), np.zeros((nz, 1))], 1)
    c = np.concatenate([c_u, c_c, c_d, c_z]).astype(np.float32)
    e = np.concatenate([e_u, e_c, e_d, e_z]).astype(np.float32)
    p = rng.permutation(n)
    c, e = c[p], e[p]
    return np.ascontiguousarray(np.concatenate([c - e, c + e], 1)), np.ascontiguousarray(c)


@pytest.fixture(scope="module")
def host_trees():
    """n -> (boxes, centres, host nodes, host prims), each built once"""
    cache = {}

    def get(n):
        if n not in cache:
            bb, ct = mixed_boxes(n)
            t = time.perf_counter()
            nodes, prims = crscene.build_bvh(bb, ct)
            _note(f"host BVH build, {n} mixed boxes: {time.perf_counter() - t:.2f} s, {len(nodes)} nodes")
            cache[n] = (bb, ct, nodes, prims)
        return cache[n]
    return get


@pytest.mark.parametrize("n", SCAN_SIZES)
def test_host_builder_past_two_scan_levels(n, host_trees):
    bb, ct, nodes, prims = host_trees(n)
    check_tree(nodes, prims, n)
    leaf = (nodes["count_leaf"] & crscene.LEAF_BIT) != 0
    assert (nodes["count_leaf"][leaf] & crscene.COUNT_MASK).max() >= 64          # the duplicate blocks stay whole


def test_device_builder_refuses_past_its_limit():
    """n = 2^22 + 1 is refused before any device work (so also without a GPU), and nothing is written"""
    n = BUILD_LIMIT + 1
    bb = np.zeros((n, 6), np.float32)
    rc, nodes, prims = _device_build(bb, np.zeros((n, 3), np.float32))
    assert rc == CRGPU_ERR_UNSUPPORTED and len(nodes) == 0
    assert b"4194304" in crgpu.lib().crgpu_last_error()


@pytest.mark.gpu
@pytest.mark.parametrize("n", SCAN_SIZES)
def test_device_builder_past_two_scan_levels(n, host_trees):
    bb, ct, h_nodes, h_prims = host_trees(n)
    t = time.perf_counter()
    rc, d_nodes, d_prims = _device_build(bb, ct)
    if rc == CRGPU_ERR_NOMEM:
        pytest.skip(f"device BVH build of {n} boxes: {_scratch_bytes(n)} B of scratch needed, twice that free: "
                    + crgpu.lib().crgpu_last_error().decode(errors="replace"))
    assert rc == 0, crgpu.lib().crgpu_last_error().decode(errors="replace")
    _note(f"device BVH build, {n} mixed boxes: {time.perf_counter() - t:.2f} s")
    same_tree(d_nodes, d_prims, h_nodes, h_prims)


@pytest.mark.gpu
def test_cli_builds_past_the_device_limit_on_the_host(tmp_path):
    """cray_b200 --gpu-bvh with a 4,194,305-triangle mesh: the device build is refused, the loader builds that BVH on the host and
    the frame is the one rendered without the flag, bit for bit."""
    d = str(tmp_path)
    verts, faces = _grid(2048, 1024, (4.0, 2.0), 6.0, 0.3, np.random.default_rng(3))
    extra = len(verts)
    verts = np.concatenate([verts, [[-0.5, -0.5, 3.0], [0.5, -0.5, 3.0], [0.0, 0.5, 3.0]]])
    faces = np.concatenate([faces, [[extra, extra + 1, extra + 2]]])
    assert len(faces) == BUILD_LIMIT + 1
    _write_obj(os.path.join(d, "big.obj"), verts, faces)
    scene = _write_scene(d, "big", [("big.obj", (0, 0, 0))], w=32, h=18, spp=2, bounces=2)
    exe = os.path.join(ROOT, "c-ray_b200", "cray_b200")
    outs = []
    for extra_args in ([], ["--gpu-bvh"]):
        f32 = os.path.join(d, f"o{len(outs)}.f32")
        r = subprocess.run([exe, scene, "--dump-f32", f32, "-o", os.path.join(d, "o.png"), "-q"] + extra_args, cwd=d,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-2000:]
        outs.append((np.fromfile(f32, dtype=np.float32), r.stdout))
    assert "building on the host" not in outs[0][1]
    assert "building on the host" in outs[1][1] and "limit 4194304" in outs[1][1], outs[1][1][-2000:]
    assert np.array_equal(outs[0][0].view(np.uint32), outs[1][0].view(np.uint32))


# ================================================================================================ B: a 1.2 M-triangle mesh
GRID_CELLS = 776                                         # 2 x 776^2 = 1,204,352 triangles: above 2^20


@pytest.fixture(scope="module")
def grid_scene(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("grid"))
    verts, faces = _grid(GRID_CELLS, GRID_CELLS, (2.5, 2.5), 4.0, 0.25, np.random.default_rng(5))
    _write_obj(os.path.join(d, "grid.obj"), verts, faces)
    ball = {"type": "sphere", "radius": 0.4, "color": [0.8, 0.3, 0.2], "instances": [{"transforms": [{"type": "translate", "X": 0.8, "Y": 0.5, "Z": 3.2}]}]}
    p = _write_scene(d, "scale_grid", [("grid.obj", (0, 0, 0))], [ball], w=64, h=48, spp=2, bounces=4)
    t = time.perf_counter()
    out = _flatten(p, os.path.join(d, "scale_grid.crscene"))
    _note(f"load + host BVH build, {len(faces)}-triangle grid: {time.perf_counter() - t:.2f} s")
    return out


@pytest.mark.gpu
def test_large_mesh_device_bvh_equals_the_scene_bvh(grid_scene):
    (label, bb, ct, nodes, prims), = mesh_inputs(grid_scene)
    assert len(bb) > 1 << 20
    d_nodes, d_prims = crscene.build_bvh_gpu(bb, ct)
    same_tree(d_nodes, d_prims, nodes, prims)


_GRID_RAYS = {}


def grid_rays(path):
    """raysets() of test_gpu_trace without its reference-semantics pass (there, the degenerate rays of the adversarial set open
    every node of a 1.2 M-triangle tree): every ray of every bounce of the paths of the central 48 x 32 pixels, two passes, and the
    adversarial classes; the oracle's device-semantics records and counters"""
    if not _GRID_RAYS:
        o = O.OracleScene(path)
        x0, y0 = (o.W - 48) // 2, (o.H - 32) // 2
        p = o.path_rays(x0, y0, x0 + 48, y0 + 32, passes=(0, 2))
        a, ac, _ = adversarial_rays(o, np.random.default_rng(1204352))
        rays = np.concatenate([p, a]).astype(np.float32)
        r1, c1 = o.closest_hit(rays, O.SEM_DEVICE)
        o.close()
        _GRID_RAYS.update(rays=rays, r1=r1, c1=c1)
    return _GRID_RAYS["rays"], _GRID_RAYS["r1"], _GRID_RAYS["c1"]


@pytest.mark.gpu
def test_large_mesh_trace_records_every_variant(grid_scene):
    rays, r1, c1 = grid_rays(grid_scene)
    assert (r1["poly"] >= 0).sum() > len(rays) // 2                 # most rays hit the mesh
    g = crgpu.GpuScene(grid_scene)
    for kn in VARIANTS:
        rec, perm, misses, st = g.trace_rays(rays, **kn)
        check_records(g, rec, perm, misses, r1, f"scale_grid {_name(kn)}")
        if kn.get("count"):
            check_counters(st, c1, len(rays), f"scale_grid {_name(kn)}")
    g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("stage", [0, 128, 1024])
def test_large_mesh_staged_top_nodes(stage, grid_scene, monkeypatch):
    """CRGPU_TRACE_STAGE=<pairs>: the top pairs of the 1.2 M-triangle tree staged in shared memory (launches of >= 65,536 rays)"""
    monkeypatch.setenv("CRGPU_TRACE_STAGE", str(stage))
    rays, r1, c1 = grid_rays(grid_scene)
    k = -(-STAGE_MIN_RAYS // len(rays))                              # whole copies of the set: the counters scale by k
    rays, exp = np.tile(rays, (k, 1)), np.tile(r1, k)
    c = {f: v * k for f, v in c1.items()}
    g = crgpu.GpuScene(grid_scene)
    for kn in (dict(), dict(defer=1, burst=4), dict(defer=2, burst=4), dict(count=1), dict(count=1, defer=2, burst=4)):
        rec, perm, misses, st = g.trace_rays(rays, **kn)
        check_records(g, rec, perm, misses, exp, f"scale_grid stage={stage} {_name(kn)}")
        if kn.get("count"):
            check_counters(st, c, len(rays), f"scale_grid stage={stage} {_name(kn)}")
    g.close()


def _frame_vs_device_semantics(path, W, H, spp, b, what):
    g = crgpu.GpuScene(path, W, H, spp, b)
    g.render_frame()
    img = g.read()
    g.close()
    o = O.OracleScene(path, W, H, spp, b)
    ref, flagged = o.render_sem(O.SEM_DEVICE)
    o.close()
    tally = Tally(f"frame {what}")
    tally.add(W * H * spp, flagged.sum())
    tally.check()
    bad = np.nonzero((~same_bits(img, ref)).any(axis=2) & (flagged == 0))
    assert len(bad[0]) == 0, f"{what}: {len(bad[0])} unflagged pixels differ, first rows {bad[0][:5]} cols {bad[1][:5]}"


@pytest.mark.gpu
def test_large_mesh_frame_equals_device_semantics(grid_scene):
    _frame_vs_device_semantics(grid_scene, 64, 48, 2, 4, "scale_grid")


# ================================================================================================ C: leaves of 64 K triangles
# 16 triangles through the point (0, 0, 4), vertex offsets in 1/16ths: the centroid sums are exact, so every copy has the same
# centroid and the binned SAH cannot split them
_CLUMP_RNG = np.random.default_rng(65536)
_D0 = np.concatenate([_CLUMP_RNG.integers(-16, 17, (16, 2)), _CLUMP_RNG.integers(-2, 3, (16, 1))], 1) / 16.0
_D1 = np.concatenate([_CLUMP_RNG.integers(-16, 17, (16, 2)), _CLUMP_RNG.integers(-2, 3, (16, 1))], 1) / 16.0
CLUMP = np.stack([_D0, _D1, -_D0 - _D1], 1) + np.array([0.0, 0.0, 4.0])             # (16 triangles, 3 vertices, xyz)
# ordinary triangles well outside the clump's box: the root is not the leaf
AROUND = [(x, y, z) for x in (-2.75, 2.75) for y in (-1.5, 0.0, 1.5) for z in (4.0, 5.0)]


def _write_big_leaf(d, n):
    verts = [CLUMP.reshape(-1, 3)]
    faces = [np.arange(48).reshape(16, 3)[np.arange(n) % 16]]
    for k, c in enumerate(AROUND):
        verts.append(np.array(c) + np.array([[-0.25, -0.25, 0.0], [0.25, -0.25, 0.0], [0.0, 0.25, 0.0]]))
        faces.append(np.array([[48 + 3 * k, 49 + 3 * k, 50 + 3 * k]]))
    _write_obj(os.path.join(d, f"leaf{n}.obj"), np.concatenate(verts), np.concatenate(faces))
    if not os.path.exists(os.path.join(d, "back.obj")):                # a second mesh behind: prims follow the clump's
        _write_obj(os.path.join(d, "back.obj"), [[-6, -6, 9], [6, -6, 9], [6, 6, 9], [-6, 6, 9]], [[0, 1, 2], [0, 2, 3]])
    return _write_scene(d, f"leaf{n}", [(f"leaf{n}.obj", (0, 0, 0)), ("back.obj", (0, 0, 0))], w=32, h=24, spp=2, bounces=3)


@pytest.fixture(scope="module")
def leaf_scenes(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("leaves"))
    return {n: _flatten(_write_big_leaf(d, n), os.path.join(d, f"leaf{n}.crscene")) for n in BIG_LEAVES}


def _big_leaf(path, n):
    """(label, boxes, centres, stored nodes, stored prims) of the clump mesh and the bounds of its leaf of n triangles"""
    meshes = mesh_inputs(path)
    label, bb, ct, nodes, prims = meshes[0]
    assert len(bb) == n + len(AROUND)
    leaf = (nodes["count_leaf"] & crscene.LEAF_BIT) != 0
    cnt = nodes["count_leaf"] & crscene.COUNT_MASK
    big = np.nonzero(leaf & (cnt == n))[0]
    assert len(big) == 1 and cnt[leaf].max() == n, (n, np.sort(cnt[leaf])[-4:])
    assert len(nodes) > 1 and not leaf[0]
    assert (prims[nodes["first"][big[0]]:nodes["first"][big[0]] + n] < n).all()        # exactly the clump's faces
    return meshes[0], nodes["bounds"][big[0]].astype(np.float64)


@pytest.mark.parametrize("n", BIG_LEAVES)
def test_big_leaf_host_tree(n, leaf_scenes):
    (label, bb, ct, nodes, prims), box = _big_leaf(leaf_scenes[n], n)
    check_tree(nodes, prims, len(bb))
    h_nodes, h_prims = crscene.build_bvh(bb, ct)
    same_tree(h_nodes, h_prims, nodes, prims)


@pytest.mark.gpu
@pytest.mark.parametrize("n", BIG_LEAVES)
def test_big_leaf_device_tree(n, leaf_scenes):
    (label, bb, ct, nodes, prims), box = _big_leaf(leaf_scenes[n], n)
    d_nodes, d_prims = crscene.build_bvh_gpu(bb, ct)
    same_tree(d_nodes, d_prims, nodes, prims)


def _unit(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def big_leaf_rays(o, box, rng, k=400):
    """rays that hit the clump, graze its leaf box (origins on its faces, directions along them, rays aimed at its edges) and miss
    it (parallel to an axis, just outside), plus the traced paths of a block of pixels and the adversarial classes"""
    lo, hi = box[0::2], box[1::2]
    centre = (lo + hi) / 2
    rays, cls = [], []

    def add(org, d, c):
        rays.append(np.concatenate([org, d], 1).astype(np.float32))
        cls.extend([c] * len(org))
    # hit: random points of random clump triangles, from a sphere around the box
    w = rng.dirichlet([1, 1, 1], k)
    tgt = np.einsum("kv,kvx->kx", w, CLUMP[rng.integers(0, 16, k)])
    org = centre + _unit(rng.normal(size=(k, 3))) * 3.0
    add(org, _unit(tgt - org), "hit")
    # graze: origins on a face of the box, directions random or along the face (that component +0 / -0)
    axis, side = rng.integers(0, 3, k), rng.integers(0, 2, k)
    org = lo + rng.uniform(0, 1, (k, 3)) * (hi - lo)
    org[np.arange(k), axis] = np.where(side == 1, hi[axis], lo[axis])
    d = _unit(rng.normal(size=(k, 3)))
    add(org, d, "graze")
    d[np.arange(k), axis] = np.where(rng.integers(0, 2, k) == 1, -0.0, 0.0)
    add(org, d, "graze")
    # graze: aimed from outside at points of the box's edges
    edge = lo + rng.uniform(0, 1, (k, 3)) * (hi - lo)
    a, b = rng.integers(0, 3, k), rng.integers(1, 3, k)
    b = (a + b) % 3
    edge[np.arange(k), a] = np.where(rng.integers(0, 2, k) == 1, hi[a], lo[a])
    edge[np.arange(k), b] = np.where(rng.integers(0, 2, k) == 1, hi[b], lo[b])
    org = centre + _unit(rng.normal(size=(k, 3))) * 4.0
    add(org, _unit(edge - org), "graze")
    # miss: along z (with a small y slope) at x just outside the box, from in front of it
    gap = rng.uniform(1e-4, 0.05, k) * (hi[0] - lo[0])
    x = np.where(rng.integers(0, 2, k) == 1, hi[0] + gap, lo[0] - gap)
    org = np.stack([x, rng.uniform(lo[1], hi[1], k), np.full(k, lo[2] - 2.0)], 1)
    d = np.stack([np.zeros(k), rng.uniform(-0.05, 0.05, k), np.ones(k)], 1)
    add(org, _unit(d), "miss")
    p = o.path_rays(8, 6, 24, 18, passes=(0, 1))
    add(p[:, :3], p[:, 3:], "path")
    a, ac, _ = adversarial_rays(o, rng, n=96)
    add(a[:, :3], a[:, 3:], "adversarial")
    return np.concatenate(rays), np.array(cls)


@pytest.mark.gpu
@pytest.mark.parametrize("n", BIG_LEAVES)
def test_big_leaf_trace_records_every_variant(n, leaf_scenes):
    path = leaf_scenes[n]
    _, box = _big_leaf(path, n)
    o = O.OracleScene(path)
    rays, cls = big_leaf_rays(o, box, np.random.default_rng(n))
    t = time.perf_counter()
    r1, c1 = o.closest_hit(rays, O.SEM_DEVICE)
    o.close()
    _note(f"big leaf {n}: {len(rays)} rays, oracle {time.perf_counter() - t:.1f} s, {c1['tri_tests']} triangle tests")
    hit_clump = (r1["inst"] >= 0) & (r1["poly"] >= 0) & (r1["poly"] < n)
    assert hit_clump[cls == "hit"].mean() > 0.9 and hit_clump[cls == "graze"].any() and not hit_clump[cls == "miss"].any()
    assert c1["tri_tests"] > 1000 * n                                              # many rays test the whole leaf
    g = crgpu.GpuScene(path)
    for kn in VARIANTS:
        rec, perm, misses, st = g.trace_rays(rays, **kn)
        check_records(g, rec, perm, misses, r1, f"leaf{n} {_name(kn)}")
        if kn.get("count"):
            check_counters(st, c1, len(rays), f"leaf{n} {_name(kn)}")
    g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n", BIG_LEAVES)
def test_big_leaf_frame_equals_device_semantics(n, leaf_scenes):
    _frame_vs_device_semantics(leaf_scenes[n], 32, 24, 2, 3, f"leaf{n}")


# ================================================================================================ D: tile sets past one launch
def _tile_sets():
    """name -> (W, H, rects): every set covers its frame, and its last rectangle is at least as large as the one before"""
    out = {}
    W, H = 256, 160
    y, x = np.mgrid[0:H, 0:W]
    out["1x1_256x160"] = (W, H, np.stack([x, y, x + 1, y + 1], -1).reshape(-1, 4))
    W, H = 320, 240
    y, x = np.mgrid[0:H // 2, 0:W]
    ones = np.stack([x, y, x + 1, y + 1], -1).reshape(-1, 4)
    y, x = np.mgrid[H // 2:H:4, 0:W]
    strips = np.stack([x, y, x + 1, y + 4], -1).reshape(-1, 4)
    out["1x1+1x4_320x240"] = (W, H, np.concatenate([ones, strips]))
    rng = np.random.default_rng(12)
    rects, y0 = [], 0
    while y0 < H:
        h = min(int(rng.choice([1, 1, 2])), H - y0)
        x0 = 0
        while x0 < W:
            w = min(int(rng.choice([1, 1, 2])), W - x0)
            rects.append((x0, y0, x0 + w, y0 + h))
            x0 += w
        y0 += h
    rects = np.array(rects)[rng.permutation(len(rects))]
    area = (rects[:, 2] - rects[:, 0]) * (rects[:, 3] - rects[:, 1])
    big = int(np.argmax(area))
    rects[[big, -1]] = rects[[-1, big]]
    out["ragged_320x240"] = (W, H, rects)
    return out


TILE_SETS = _tile_sets()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(TILE_SETS))
def test_tile_sets_past_one_pixel_list_launch(name):
    W, H, rects = TILE_SETS[name]
    assert 40000 <= len(rects) <= 70000
    path, spp = os.path.join(GOLDEN, "g_nodes.crscene"), 3
    g = crgpu.GpuScene(path, W, H, spp, 4)
    g.render_frame()
    ref = g.read().view(np.uint32).copy()
    g.close()

    def check(g, what):
        got = g.read().view(np.uint32)
        bad = np.nonzero((got != ref).any(axis=2))
        assert len(bad[0]) == 0, f"{name} {what}: {len(bad[0])} pixels differ from render_frame(), first rows {bad[0][:5]} cols {bad[1][:5]}"

    g = crgpu.GpuScene(path, W, H, spp, 4)
    st = g.render_tiles(rects)
    assert st["paths"] == W * H * spp
    check(g, "default budget")
    g.clear()
    g.render_tiles(rects)                                              # the same list: the pixel list is not rebuilt
    check(g, "second call, same list")
    g.clear()
    g.render_tiles(rects, 0, 1)
    g.render_tiles(rects, 1, spp - 1)
    check(g, "split pass ranges")
    g.clear()
    g.enable_stop(True)
    st = g.render_tiles(rects)
    assert not st["stopped"]
    check(g, "armed")
    g.close()
    g = crgpu.GpuScene(path, W, H, spp, 4)
    g.set_max_paths(1024)                                              # many pieces: the walk over list ranges
    g.render_tiles(rects)
    check(g, "1024 paths in flight")
    g.close()


# ================================================================================================ E: the gather past 65,535 tiles
@pytest.mark.gpu
def test_cli_gather_past_65535_tiles_per_peer(tmp_path):
    """cray_b200 -j 2 on a 512x288 frame in 1x1 tiles: each GPU owns 73,728 tiles, all packed, sent and unpacked by the NCCL
    gather; the frame must be the -j 1 frame bit for bit."""
    if crgpu.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    exe = os.path.join(ROOT, "c-ray_b200", "cray_b200")
    args = [exe, os.path.join(GOLDEN, "g_nodes.crscene"), "-d", "512x288", "-s", "2", "-t", "1x1", "-o", str(tmp_path / "o.png"), "-q"]
    frames = []
    for j in (1, 2):
        f32 = str(tmp_path / f"j{j}.f32")
        r = subprocess.run(args + ["-j", str(j), "--dump-f32", f32], cwd=str(tmp_path), stdout=subprocess.PIPE,
                           stderr=subprocess.STDOUT, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-2000:]
        frames.append(np.fromfile(f32, dtype=np.float32))
    assert len(frames[0]) == 512 * 288 * 3
    assert np.array_equal(frames[0].view(np.uint32), frames[1].view(np.uint32))


@pytest.mark.gpu
def test_ranked_gather_past_65535_tiles_per_peer():
    """The same through two torchrun ranks (bench.py, one process per GPU, the rank gather): the frame CRC of one rank."""
    if crgpu.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from test_gpu_parity import _bench
    common = ["--workload", "hdr", "--width", "512", "--height", "288", "--spp", "2", "--tile", "1", "--steps", "1", "--warmup", "1",
              "--no-cpu-baseline"]
    one, two = _bench(common, 1), _bench(common, 2)
    assert two["n_gpus"] == 2 and two["frame_crc32"] == one["frame_crc32"] == two["value_path_crc32"]
