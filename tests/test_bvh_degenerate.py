"""BVH builds of primitives that no split separates: centres at one point, extents that overflow to inf, centres that underflow
into one cluster.  The binned SAH puts every primitive of such a node into bin 0, every cost is NaN or inf, and the median fallback
(above 16 primitives) or the default split sends everything left.  The node then splits into an empty right leaf and a left child
with the same primitives and box, which decides the same way, down to the depth cap of 64: the tree can need more than the 2n - 1
nodes of a tree without empty leaves.

The judge is a plain restatement of the reference's build (bvh.c:96-296: buildBvhGeneric, buildBvhRecursive and the two-pointer
partition) in numpy float32, recursive, one node at a time, with an unbounded node list.  Before it judges anything it must
reproduce the stored BVHs of the golden scenes and the host builder's trees of test_bvh_build.synthetic_cases(), bit for bit.

CPU: crloader_build_bvh (room for 2n - 1 nodes: equal to the reference, or refuses and reports the size without writing past
2n - 1) and the scene loader (stores the whole tree) against the reference, serial and parallel.  The host builds run in a
subprocess, so that a build writing past its array fails a test instead of the test run.
GPU: crgpu_bvh_build under the same contract; scenes with such trees traced (every K2 variant, against the oracle), rendered
(against the oracle's device semantics) and rendered by the CLI with --gpu-bvh; and a scene edit that makes such a top level.
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
from conftest import GOLDEN, GOLDEN_SCENES, ROOT
from test_bvh_build import check_tree, mesh_inputs, same_tree, synthetic_cases

F32 = np.float32
FLT_MAX = F32(np.finfo(np.float32).max)
MAX_DEPTH, MAX_LEAF, BINS = 64, 16, 32
CRGPU_ERR_UNSUPPORTED = -4
GUARD = 64                                   # nodes past the caller's 2n - 1 that a build must leave untouched
GUARD_WORD = 0xA5A5A5A5


# ================================================================================================ the reference, restated
def _okey(v):
    """a total-order key of float32 values (+0 and -0 get the same key)"""
    b = (np.asarray(v, F32) + F32(0)).view(np.uint32).astype(np.uint64)
    return np.where(b & 0x80000000, ~b & 0xFFFFFFFF, b | 0x80000000)


def _bin_index(coord, lo, scale):
    """bvh.c:89-95 with (unsigned)float as x86-64 cvttss2si: truncate to 64 bits, keep the low 32; NaN and overflow give 0"""
    with np.errstate(all="ignore"):
        fi = (coord - lo) * scale
        fi = np.where(fi < 0, F32(0), fi)
        ok = (fi > F32(-9.2233720e18)) & (fi < F32(9.2233720e18))
        b = np.where(ok, fi, F32(0)).astype(np.int64) & 0xFFFFFFFF
    return np.minimum(b, BINS - 1)


def _half_area(mn, mx):
    """bbox.h:26 in float32, one rounding per operation: (..., 3) arrays"""
    with np.errstate(all="ignore"):
        e = (mx - mn).astype(F32)
        return e[..., 0] * (e[..., 1] + e[..., 2]) + e[..., 1] * e[..., 2]


def _fold(boxes, lo0, hi0):
    """bbox_extend folded over boxes in order from (lo0, hi0): MIN(a, b) = a < b ? a : b, so a tie takes the later box's value,
    which decides the sign of a zero bound.  Python floats hold float32 values exactly, so comparisons are the C ones."""
    lo, hi = list(lo0), list(hi0)
    for bmn, bmx in boxes:
        for k in range(3):
            lo[k] = lo[k] if lo[k] < bmn[k] else bmn[k]
            hi[k] = hi[k] if hi[k] > bmx[k] else bmx[k]
    return lo, hi


EMPTY_LO, EMPTY_HI = [float(FLT_MAX)] * 3, [float(-FLT_MAX)] * 3


class Reference:
    """buildBvhGeneric + buildBvhRecursive: nodes as BVH_NODE records, primitive order as int32"""

    def __init__(self, bboxes, centers):
        self.bb = np.ascontiguousarray(bboxes, F32).reshape(-1, 6)
        self.ct = np.ascontiguousarray(centers, F32).reshape(-1, 3)
        n = len(self.bb)
        self.prims = np.arange(n, dtype=np.int32)
        self.nodes = []                                          # [bounds minx maxx miny maxy minz maxz, first, count|leaf]
        if n == 0:
            return
        lo, hi = self._fold_prims(np.arange(n))
        self.nodes.append([[lo[0], hi[0], lo[1], hi[1], lo[2], hi[2]], 0, 0])
        self._build(0, 0, n, 0)

    def _fold_prims(self, idx):
        """the fold over primitives idx in order: extreme value, the last of its ties (vectorised by key: value, then position)"""
        pos = np.arange(len(idx), dtype=np.uint64)
        lo, hi = [], []
        for k in range(3):
            v = self.bb[idx, k]
            w = int(pos[np.argmin((_okey(v) << 32) | (0xFFFFFFFF - pos))]) if len(idx) else -1
            lo.append(min(float(FLT_MAX), float(v[w])) if w >= 0 else float(FLT_MAX))
            v = self.bb[idx, 3 + k]
            w = int(pos[np.argmax((_okey(v) << 32) | pos)]) if len(idx) else -1
            hi.append(max(float(-FLT_MAX), float(v[w])) if w >= 0 else float(-FLT_MAX))
        return lo, hi

    def _bins(self, idx, ids):
        """per bin of one axis: (lo, hi) of the fold over its primitives in array order, and the count (the same extreme value and
        last tie as _fold_prims, for all bins at once: segments of a stable sort by bin, reduced by key)"""
        out = [(EMPTY_LO, EMPTY_HI)] * BINS
        cnt = np.bincount(ids, minlength=BINS)
        order = np.argsort(ids, kind="stable")
        pos = np.arange(len(idx), dtype=np.uint64)[order]
        starts = np.r_[0, np.cumsum(cnt)][:-1][cnt > 0]
        full = np.nonzero(cnt)[0]
        bb = self.bb[idx[order]]
        lo, hi = np.empty((len(full), 3)), np.empty((len(full), 3))
        for k in range(3):
            w = np.minimum.reduceat((_okey(bb[:, k]) << 32) | (0xFFFFFFFF - pos), starts)
            lo[:, k] = np.minimum(self.bb[idx[(0xFFFFFFFF - (w & 0xFFFFFFFF)).astype(np.int64)], k], FLT_MAX)
            w = np.maximum.reduceat((_okey(bb[:, 3 + k]) << 32) | pos, starts)
            hi[:, k] = np.maximum(self.bb[idx[(w & 0xFFFFFFFF).astype(np.int64)], 3 + k], -FLT_MAX)
        for j, b in enumerate(full):
            out[b] = (lo[j].tolist(), hi[j].tolist())
        return out, cnt

    def _split(self, bounds, begin, end, depth):
        """bvh.c:137-243 for prims[begin:end): None for a leaf, else (first right position, left box, right box)"""
        count = end - begin
        if depth >= MAX_DEPTH or count < 2:
            return None
        idx = self.prims[begin:end]
        bins, counts, minCost, minBin = [], [], [float(FLT_MAX)] * 3, [1, 1, 1]
        for axis in range(3):
            lo = F32(bounds[2 * axis])
            with np.errstate(all="ignore"):
                scale = F32(BINS) / (F32(bounds[2 * axis + 1]) - lo)
            b, cnt = self._bins(idx, _bin_index(self.ct[idx, axis], lo, scale))
            bins.append(b)
            counts.append(cnt)
            # right to left: the cost of everything right of each split, then left to right
            rb, rc, cur, c = [], [], (EMPTY_LO, EMPTY_HI), 0
            for i in range(BINS - 1, 0, -1):
                c += int(cnt[i])
                cur = _fold([b[i]], *cur)
                rb.append(cur)
                rc.append(c)
            rb, rc = np.array(rb[::-1], F32), np.array([0] + rc[::-1])               # index i: bins i..31 (i >= 1)
            with np.errstate(all="ignore"):
                rcost = np.r_[F32(0), rc[1:].astype(F32) * _half_area(rb[:, 0], rb[:, 1])].astype(F32)
            lb, lc, cur, c = [], [], (EMPTY_LO, EMPTY_HI), 0
            for i in range(BINS - 1):
                c += int(cnt[i])
                cur = _fold([b[i]], *cur)
                lb.append(cur)
                lc.append(c)
            lb = np.array(lb, F32)
            with np.errstate(all="ignore"):
                cost = np.array(lc).astype(F32) * _half_area(lb[:, 0], lb[:, 1]) + rcost[1:]
            for i in range(BINS - 1):
                if float(cost[i]) < minCost[axis]:
                    minBin[axis], minCost[axis] = i + 1, float(cost[i])
        minAxis = 0
        if minCost[1] < minCost[0]:
            minAxis = 1
        if minCost[2] < minCost[minAxis]:
            minAxis = 2
        with np.errstate(all="ignore"):
            nb = np.array(bounds, F32)
            leafCost = float(_half_area(nb[0::2], nb[1::2]) * (F32(count) - F32(1.5)))
        if minCost[minAxis] > leafCost:
            if count <= MAX_LEAF:
                return None
            accum, best = 0, count                                   # the approximate median (bvh.c:196-205)
            for i in range(BINS - 1):
                accum += int(counts[minAxis][i])
                approx = abs(count // 2 - accum)
                if approx < best:
                    best, minBin[minAxis] = approx, i + 1
        split = minBin[minAxis]
        lo = F32(bounds[2 * minAxis])
        with np.errstate(all="ignore"):
            scale = F32(BINS) / (F32(bounds[2 * minAxis + 1]) - lo)
        # the two-pointer partition (bvh.c:97-135): the k-th primitive from the left that belongs right swaps places with the k-th
        # from the right that belongs left; the pointers meet where the left part ends
        left = _bin_index(self.ct[idx, minAxis], lo, scale) < split
        i = int(left.sum())
        if i <= 0:
            return None
        pos = np.arange(count)
        a, b = pos[:i][~left[:i]], pos[i:][left[i:]][::-1]
        p = idx.copy()
        p[a], p[b] = idx[b], idx[a]
        self.prims[begin:end] = p
        lb = _fold(bins[minAxis][:split], EMPTY_LO, EMPTY_HI)
        rb = _fold(bins[minAxis][split:], EMPTY_LO, EMPTY_HI)
        return begin + i, lb, rb

    def _build(self, node, begin, end, depth):
        s = self._split(self.nodes[node][0], begin, end, depth)
        if s is None:
            self.nodes[node][1:] = [begin, crscene.LEAF_BIT | (end - begin)]
            return
        mid, lb, rb = s
        left = len(self.nodes)                                       # children allocated as a pair, the left subtree first
        self.nodes.append([[lb[0][0], lb[1][0], lb[0][1], lb[1][1], lb[0][2], lb[1][2]], 0, 0])
        self.nodes.append([[rb[0][0], rb[1][0], rb[0][1], rb[1][1], rb[0][2], rb[1][2]], 0, 0])
        self.nodes[node][1:] = [left, 0]
        self._build(left, begin, mid, depth + 1)
        self._build(left + 1, mid, end, depth + 1)

    def arrays(self):
        out = np.zeros(len(self.nodes), crscene.BVH_NODE)
        if self.nodes:
            out["bounds"] = np.array([n[0] for n in self.nodes], F32)
            out["first"] = [n[1] for n in self.nodes]
            out["count_leaf"] = [n[2] for n in self.nodes]
        return out, self.prims.copy()


_REF = {}


def reference(name, bb, ct):
    if name not in _REF:
        _REF[name] = Reference(bb, ct).arrays()
    return _REF[name]


def depths(nodes):
    d = np.zeros(len(nodes), np.int64)
    for i in range(len(nodes)):                              # children come after their parent
        if not nodes["count_leaf"][i] & crscene.LEAF_BIT:
            d[nodes["first"][i]] = d[nodes["first"][i] + 1] = d[i] + 1
    return d


def check_tree_deep(nodes, prims, n):
    """check_tree, plus: depth <= 64, and every empty leaf carries the empty box"""
    check_tree(nodes, prims, n)
    assert depths(nodes).max() <= MAX_DEPTH
    leaf = (nodes["count_leaf"] & crscene.LEAF_BIT) != 0
    empty = leaf & ((nodes["count_leaf"] & crscene.COUNT_MASK) == 0)
    want = np.array([FLT_MAX, -FLT_MAX] * 3, F32).view(np.uint32)
    assert (nodes["bounds"][empty].view(np.uint32) == want).all()


def chain(nodes):
    """(empty leaves, deepest level) of a tree"""
    leaf = (nodes["count_leaf"] & crscene.LEAF_BIT) != 0
    return int((leaf & ((nodes["count_leaf"] & crscene.COUNT_MASK) == 0)).sum()), int(depths(nodes).max())


# ================================================================================================ inputs
def points(p):
    p = np.asarray(p, F32).reshape(-1, 3)
    return np.concatenate([p, p], 1), p.copy()


def ordinary(m, seed=1, half=0.05):
    rng = np.random.default_rng(seed)
    c = rng.uniform(-5, 5, (m, 3)).astype(F32)
    e = np.full((m, 3), half, F32)
    return np.concatenate([c - e, c + e], 1), c


def join(*parts):
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])


SPOT = (0.3, -0.2, 0.1)


def cases():
    out = {}
    for k in (16, 17, 64, 1000):
        out[f"coincident{k}"] = points(np.tile(SPOT, (k, 1)))
        for m in (300, 2000, 20000):
            out[f"coincident{k}_in{m}"] = join(ordinary(m), points(np.tile(SPOT, (k, 1))))
    out["far2"] = points([[-2e38, 0, 0], [2e38, 0, 0]])
    out["far17"] = points([[(-1) ** i * 2e38, i, 0] for i in range(17)])
    big = np.array([[-FLT_MAX, -1, -1, FLT_MAX, 1, 1]] * 3, F32)
    out["flt_max_bounds"] = join(ordinary(40, seed=3), (big, np.zeros((3, 3), F32)))
    out["underflow64"] = points(np.repeat((0.125 ** np.arange(64, dtype=np.float64))[:, None], 3, axis=1))
    return out


CASES = cases()
# 17 coincident points stay below TASK_MIN_PRIMS (2048), so their chain lies inside one task of the parallel build; 4,096 and 10,000
# do not, so the chain (and its empty right ranges) starts in the serial top phase
PARALLEL = {f"parallel{m}": join(ordinary(m, seed=5), points(np.tile(SPOT, (17, 1)))) for m in (8175, 8176, 8191, 12000)}
PARALLEL["coincident10000"] = points(np.tile(SPOT, (10000, 1)))
PARALLEL["parallel8192_4096"] = join(ordinary(8192, seed=6), points(np.tile(SPOT, (4096, 1))))


# ================================================================================================ host builds, in a subprocess
def _host_build(bb, ct):
    """crloader_build_bvh with room for 2n - 1 nodes and a guard behind them: (rc, node count, nodes, prims, guard intact)"""
    n = len(bb)
    buf = np.zeros(2 * n - 1 + GUARD, crscene.BVH_NODE)
    buf.view(np.uint32)[:] = GUARD_WORD
    prims = np.zeros(n, np.int32)
    cnt = C.c_uint32(0)
    L = crscene.loader()
    L.crloader_build_bvh.restype = C.c_int
    rc = L.crloader_build_bvh(np.ascontiguousarray(bb, F32).ctypes.data_as(C.c_void_p), np.ascontiguousarray(ct, F32).ctypes.data_as(C.c_void_p),
                              C.c_uint32(n), buf.ctypes.data_as(C.c_void_p), C.byref(cnt), prims.ctypes.data_as(C.c_void_p))
    guard_ok = bool((buf[2 * n - 1:].view(np.uint32) == GUARD_WORD).all())
    return rc, cnt.value, buf[:min(cnt.value, 2 * n - 1)].copy(), prims, guard_ok, L.crloader_last_error().decode() if rc else ""


def obj_of(bb):
    """an OBJ whose triangle i spans box i: (min, max, min), so a point box collapses onto one vertex"""
    lines = []
    for b in bb:
        lines.append("v %.9g %.9g %.9g" % tuple(b[:3]))
        lines.append("v %.9g %.9g %.9g" % tuple(b[3:]))
    lines.append("vn 0 0 -1")
    lines += ["f %d//1 %d//1 %d//1" % (2 * i + 1, 2 * i + 2, 2 * i + 1) for i in range(len(bb))]
    return "\n".join(lines) + "\n"


def scene_doc(prims, meshes, w=64, h=48, spp=2, bounces=4):
    return {"renderer": {"width": w, "height": h, "samples": spp, "bounces": bounces}, "camera": {"FOV": 70},
            "scene": {"ambientColor": {"down": [1, 1, 1], "up": [0.5, 0.7, 1.0]}, "primitives": prims, "meshes": meshes}}


def radius0_spheres(pos):
    return [{"type": "sphere", "radius": 0.0, "color": [0.5, 0.5, 0.5],
             "instances": [{"transforms": [{"type": "translate", "X": float(p[0]), "Y": float(p[1]), "Z": float(p[2])}]} for p in pos]}]


def _loaded_trees(path):
    """(mesh 0's boxes, centres, nodes, prims) and (top-level instance boxes, centres, nodes, prims) of a JSON scene"""
    flat = crscene.load_json(path)
    A = crscene.arrays(flat)
    top = int(flat.top_bvh)
    crscene.free(flat)
    out = {}
    if len(A["meshes"]):
        m = A["meshes"][0]
        polys = A["polys"][m["poly_offset"]:m["poly_offset"] + m["poly_count"]]
        bb, ct = crscene.prim_boxes(A["vertices"], polys)
        b = A["bvhs"][m["bvh"]]
        out["mesh"] = (bb, ct, A["bvh_nodes"][b["node_offset"]:b["node_offset"] + b["node_count"]],
                       A["prim_indices"][b["prim_offset"]:b["prim_offset"] + b["prim_count"]])
    inst = A["instances"]
    if (inst["kind"] != 1).all():                              # spheres placed by a translation: the +-radius box moved by it
        b = A["bvhs"][top]
        c = inst["A"][:, [3, 7, 11]].astype(F32)
        r = A["spheres"]["radius"][inst["object"]].astype(F32)[:, None]
        out["top"] = (np.concatenate([-r + c, r + c], 1), c, A["bvh_nodes"][b["node_offset"]:b["node_offset"] + b["node_count"]],
                      A["prim_indices"][b["prim_offset"]:b["prim_offset"] + b["prim_count"]])
    return out


def isolated_host_builds(src, dst):
    """run in a child process: every case of src (npz) through crloader_build_bvh and, for the mesh/instance forms, the loader"""
    d = np.load(src)
    res = {}
    work = os.path.dirname(dst)
    for name in sorted({k.split("/")[0] for k in d.files}):
        bb, ct = d[name + "/bb"], d[name + "/ct"]
        rc, cnt, nodes, prims, guard, err = _host_build(bb, ct)
        res.update({f"{name}/rc": rc, f"{name}/cnt": cnt, f"{name}/nodes": nodes, f"{name}/prims": prims, f"{name}/guard": guard,
                    f"{name}/err": err})
        if name + "/json" in d.files:
            kind = str(d[name + "/json"])
            if kind == "mesh":
                open(os.path.join(work, name + ".obj"), "w").write(obj_of(bb))
                doc = scene_doc([], [{"fileName": name + ".obj", "instances": [{"transforms": [{"type": "translate", "Z": 5}]}]}])
            else:
                doc = scene_doc(radius0_spheres(ct), [])
            path = os.path.join(work, name + ".json")
            open(path, "w").write(json.dumps(doc))
            for part, (lbb, lct, ln, lp) in _loaded_trees(path).items():
                if part == kind or kind == "instances" and part == "top":
                    res.update({f"{name}/lbb": lbb, f"{name}/lct": lct, f"{name}/lnodes": ln, f"{name}/lprims": lp})
    np.savez(dst, **res)


def host_builds(tmp_path, named, threads=None, json_kind=None):
    """{name: results} of isolated_host_builds for {name: (bb, ct)}"""
    src, dst = str(tmp_path / "in.npz"), str(tmp_path / "out.npz")
    arrs = {}
    for name, (bb, ct) in named.items():
        arrs[name + "/bb"], arrs[name + "/ct"] = bb, ct
        if json_kind:
            arrs[name + "/json"] = np.array(json_kind(name))
    np.savez(src, **arrs)
    env = dict(os.environ)
    if threads:
        env["CRLOADER_THREADS"] = str(threads)
    code = (f"import sys; sys.path[:0] = [{os.path.join(ROOT, 'c-ray_b200')!r}, {os.path.join(ROOT, 'tests')!r}]\n"
            f"import test_bvh_degenerate as T; T.isolated_host_builds({src!r}, {dst!r})")
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=str(tmp_path), stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=900)
    assert r.returncode == 0, f"host builds died (exit {r.returncode}):\n{r.stdout[-3000:]}"
    d = np.load(dst)
    return {name: {k.split("/", 1)[1]: d[k] for k in d.files if k.split("/")[0] == name} for name in named}


def check_host(name, bb, ct, got):
    nodes, prims = reference(name, bb, ct)
    n = len(bb)
    assert got["guard"], f"{name}: crloader_build_bvh wrote past the caller's 2n - 1 nodes"
    if len(nodes) <= 2 * n - 1:
        assert int(got["rc"]) == 0, f"{name}: crloader_build_bvh failed ({int(got['rc'])}) on a tree of {len(nodes)} nodes"
        same_tree(got["nodes"], got["prims"], nodes, prims)
    else:
        assert int(got["rc"]) != 0, f"{name}: the tree needs {len(nodes)} nodes, crloader_build_bvh has room for {2 * n - 1}"
        assert int(got["cnt"]) == len(nodes), f"{name}: reported {int(got['cnt'])} nodes needed, the tree has {len(nodes)}"
        assert f"needs {len(nodes)} nodes" in str(got["err"]), f"{name}: crloader_last_error() says {str(got['err'])!r}"
    if "lnodes" in got:
        lnodes, lprims = reference(name + "/loaded", got["lbb"], got["lct"])
        check_tree_deep(lnodes, lprims, n)
        same_tree(got["lnodes"], got["lprims"], lnodes, lprims)


# ================================================================================================ CPU: the reference itself
@pytest.mark.parametrize("name", GOLDEN_SCENES)
def test_reference_reproduces_the_golden_trees(name):
    for label, bb, ct, nodes, prims in mesh_inputs(os.path.join(GOLDEN, name + ".crscene")):
        r_nodes, r_prims = Reference(bb, ct).arrays()
        same_tree(r_nodes, r_prims, nodes, prims)


def test_reference_reproduces_the_synthetic_host_trees():
    for label, bb, ct in synthetic_cases():
        h_nodes, h_prims = crscene.build_bvh(bb, ct)
        r_nodes, r_prims = Reference(bb, ct).arrays()
        same_tree(r_nodes, r_prims, h_nodes, h_prims)


def test_reference_trees_of_the_degenerate_inputs():
    """what the inputs are for: 16 coincident points are a leaf, 17 make the 64-deep chain (alone and inside ordinary boxes, where
    the 20,017 tree fits in 2n - 1 nodes); far-apart pairs chain too; the underflowing centres end in a leaf of 42 at depth 64"""
    for name, (bb, ct) in CASES.items():
        nodes, prims = reference(name, bb, ct)
        check_tree_deep(nodes, prims, len(bb))
    assert len(reference("coincident16", *CASES["coincident16"])[0]) == 1
    for name in ("coincident17", "coincident64", "coincident1000", "far2", "far17", "coincident17_in300", "coincident17_in20000"):
        nodes, _ = reference(name, *CASES[name])
        assert chain(nodes)[1] == MAX_DEPTH, name
    assert len(reference("coincident17", *CASES["coincident17"])[0]) == 129
    assert len(reference("far2", *CASES["far2"])[0]) == 129
    nodes, _ = reference("coincident17_in20000", *CASES["coincident17_in20000"])
    assert len(nodes) <= 2 * 20017 - 1 and chain(nodes)[0] > 0
    nodes, _ = reference("underflow64", *CASES["underflow64"])
    leaf = (nodes["count_leaf"] & crscene.LEAF_BIT) != 0
    deep = leaf & (depths(nodes) == MAX_DEPTH)
    assert (nodes["count_leaf"][deep] & crscene.COUNT_MASK).max() > MAX_LEAF       # the underflowed cluster, never split


# ================================================================================================ CPU: the host builder and the loader
def test_host_builder_on_degenerate_inputs(tmp_path):
    got = host_builds(tmp_path, CASES, json_kind=lambda name: "instances" if name.startswith("far") else "mesh")
    for name, (bb, ct) in CASES.items():
        check_host(name, bb, ct, got[name])


@pytest.mark.parametrize("threads", [1, 8])
def test_host_builder_parallel_path(tmp_path, threads):
    """around PARALLEL_MIN_PRIMS (8192): with 8 threads the chain lies inside one task of the parallel build"""
    got = host_builds(tmp_path, PARALLEL, threads=threads, json_kind=lambda name: "mesh")
    for name, (bb, ct) in PARALLEL.items():
        check_host(name, bb, ct, got[name])


def test_loader_scenes_of_the_issue(tmp_path):
    """ordinary JSON scenes: a mesh of 300 triangles plus 17 collapsed onto one vertex, 17 radius-0 spheres at one point, two
    spheres at x = +-2e38: each loads and stores the reference's whole tree"""
    paths = write_scenes(str(tmp_path))
    code = (f"import sys, json; sys.path[:0] = [{os.path.join(ROOT, 'c-ray_b200')!r}, {os.path.join(ROOT, 'tests')!r}]\n"
            f"import numpy as np, test_bvh_degenerate as T\n"
            f"out = {{}}\n"
            f"for name, p in json.loads(sys.argv[1]).items():\n"
            f"    for part, v in T._loaded_trees(p).items():\n"
            f"        for k, a in zip(('bb', 'ct', 'nodes', 'prims'), v): out[f'{{name}}/{{part}}/{{k}}'] = a\n"
            f"np.savez(sys.argv[2], **out)\n")
    dst = str(tmp_path / "loaded.npz")
    r = subprocess.run([sys.executable, "-c", code, json.dumps(paths), dst], cwd=str(tmp_path), stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, f"loading died (exit {r.returncode}):\n{r.stdout[-3000:]}"
    d = np.load(dst)
    for name in paths:
        parts = sorted({k.split("/")[1] for k in d.files if k.startswith(name + "/")})
        for part in parts:
            if name != "collapsed_mesh" and part == "mesh":
                continue
            g = {k: d[f"{name}/{part}/{k}"] for k in ("bb", "ct", "nodes", "prims")}
            nodes, prims = Reference(g["bb"], g["ct"]).arrays()
            check_tree_deep(nodes, prims, len(g["bb"]))
            same_tree(g["nodes"], g["prims"], nodes, prims)
        want_chain = {"collapsed_mesh": "mesh", "collapsed_big": "mesh", "collapsed_many": "mesh", "coincident_spheres": "top", "far_spheres": "top"}[name]
        assert chain(d[f"{name}/{want_chain}/nodes"])[1] == MAX_DEPTH, name


# ================================================================================================ scenes for the GPU
def write_scenes(d):
    """{name: JSON path}: the scenes whose trees hold a 64-deep chain, each with a few visible spheres around the cluster"""
    os.makedirs(d, exist_ok=True)
    rng = np.random.default_rng(11)
    lit = [{"type": "sphere", "radius": 0.4, "color": [0.8, 0.3, 0.2], "instances": [{"transforms": [{"type": "translate", "X": -1.2, "Z": 6}]}]},
           {"type": "sphere", "radius": 0.5, "bsdf": "metal", "roughness": 0.2, "color": [0.7, 0.7, 0.9],
            "instances": [{"transforms": [{"type": "translate", "X": 1.3, "Y": 0.3, "Z": 7}]}]}]
    out = {}

    def mesh(name, m, clusters=1):
        """m ordinary triangles around (0, 0, 5) plus, per cluster, 17 collapsed onto one vertex (the first in the middle of the view)"""
        c = rng.uniform(-1.5, 1.5, (m, 3)) * [1, 1, 0.5]
        v = np.repeat(c, 3, axis=0) + rng.normal(0, 0.08, (3 * m, 3))
        spots = [(0.05, -0.03, 0.0)] + [tuple(x) for x in np.round(rng.uniform(-1.4, 1.4, (clusters - 1, 3)) * [1, 1, 0.5], 4)]
        lines = ["v %.6f %.6f %.6f" % tuple(p) for p in v] + ["v %.6f %.6f %.6f" % p for p in spots] + ["vn 0 0 -1"]
        lines += ["f %d//1 %d//1 %d//1" % (3 * i + 1, 3 * i + 2, 3 * i + 3) for i in range(m)]
        for k in range(clusters):
            lines += ["f {0}//1 {0}//1 {0}//1".format(3 * m + 1 + k)] * 17
        open(os.path.join(d, name + ".obj"), "w").write("\n".join(lines) + "\n")
        return [{"fileName": name + ".obj", "instances": [{"transforms": [{"type": "translate", "Z": 5}]}]}]

    docs = {"collapsed_mesh": scene_doc(lit, mesh("collapsed_mesh", 300)),
            "collapsed_big": scene_doc(lit, mesh("collapsed_big", 1100)),
            "collapsed_many": scene_doc(lit, mesh("collapsed_many", 1024, clusters=12)),
            "coincident_spheres": scene_doc(lit + radius0_spheres([[0.2, 0.1, 5.0]] * 17), []),
            "far_spheres": scene_doc(lit + radius0_spheres([[-2e38, 0, 5], [2e38, 0, 5]]), [])}
    for name, doc in docs.items():
        out[name] = os.path.join(d, name + ".json")
        open(out[name], "w").write(json.dumps(doc))
    return out


# ================================================================================================ GPU: the device builder
def _device_build(bb, ct):
    n = len(bb)
    buf = np.zeros(2 * n - 1 + GUARD, crscene.BVH_NODE)
    buf.view(np.uint32)[:] = GUARD_WORD
    prims = np.zeros(n, np.int32)
    cnt = C.c_uint32(0)
    G = crgpu.lib()
    G.crgpu_bvh_build.restype = C.c_int
    rc = G.crgpu_bvh_build(np.ascontiguousarray(bb, F32).ctypes.data_as(C.c_void_p), np.ascontiguousarray(ct, F32).ctypes.data_as(C.c_void_p),
                           C.c_uint32(n), C.c_int(0), buf.ctypes.data_as(C.c_void_p), C.byref(cnt), prims.ctypes.data_as(C.c_void_p))
    return rc, cnt.value, buf, prims


@pytest.mark.gpu
def test_device_builder_on_degenerate_inputs():
    for name, (bb, ct) in {**CASES, **PARALLEL}.items():
        nodes, prims = reference(name, bb, ct)
        n = len(bb)
        rc, cnt, buf, got = _device_build(bb, ct)
        assert (buf[2 * n - 1:].view(np.uint32) == GUARD_WORD).all(), f"{name}: crgpu_bvh_build wrote past the caller's 2n - 1 nodes"
        if len(nodes) <= 2 * n - 1:
            assert rc == 0, f"{name}: crgpu_bvh_build failed ({rc}) on a tree of {len(nodes)} nodes"
            same_tree(buf[:cnt], got, nodes, prims)
        else:
            assert rc == CRGPU_ERR_UNSUPPORTED, f"{name}: rc {rc} for a tree of {len(nodes)} nodes (room for {2 * n - 1})"
            assert cnt == len(nodes), f"{name}: reported {cnt} nodes needed, the tree has {len(nodes)}"
            assert (buf[:2 * n - 1].view(np.uint32) == GUARD_WORD).all(), f"{name}: a refused build wrote nodes"


# ================================================================================================ GPU: end to end
@pytest.fixture(scope="module")
def chain_scenes(tmp_path_factory):
    from test_gpu_trace import _flatten
    d = str(tmp_path_factory.mktemp("chain"))
    js = write_scenes(d)
    return d, js, {n: _flatten(p, os.path.join(d, n + ".crscene")) for n, p in js.items()}


def cluster_rays(o, target, n=3000, seed=3):
    """rays from around the scene aimed at the cluster (and just beside it), plus the adversarial rays of the trace tests"""
    from test_gpu_trace import adversarial_rays
    rng = np.random.default_rng(seed)
    t = np.asarray(target, np.float64)
    org = t + rng.normal(size=(n, 3)) * [3.0, 3.0, 2.0]
    org[: n // 2] = t + rng.uniform(-0.3, 0.3, (n // 2, 3)) * [1, 1, 0] - [0, 0, 5]    # from near the camera
    aim = t + rng.normal(size=(n, 3)) * np.where(rng.random((n, 1)) < 0.5, 0.0, 0.05)
    d = aim - org
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    a, _, _ = adversarial_rays(o, rng, n=256)
    return np.concatenate([np.concatenate([org, d], 1).astype(F32), a]).astype(F32)


CLUSTER = {"collapsed_mesh": (0.05, -0.03, 5.0), "collapsed_big": (0.05, -0.03, 5.0), "coincident_spheres": (0.2, 0.1, 5.0),
           "far_spheres": (0.0, 0.0, 5.0)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CLUSTER))
def test_chain_scene_traces_as_the_oracle(name, chain_scenes):
    import oracle_lib as O
    from test_gpu_trace import VARIANTS, _name, check_counters, check_records
    path = chain_scenes[2][name]
    o = O.OracleScene(path)
    rays = cluster_rays(o, CLUSTER[name])
    r1, c1 = o.closest_hit(rays, O.SEM_DEVICE)
    o.close()
    if name == "far_spheres":            # t is NaN wherever the +-2e38 spheres decide it: any NaN matches any NaN
        r1["t"][np.isnan(r1["t"])] = np.nan
    g = crgpu.GpuScene(path)
    try:
        for kn in VARIANTS:
            rec, perm, misses, st = g.trace_rays(rays, **kn)
            if name == "far_spheres":
                assert (np.isnan(rec["t"]) == np.isnan(r1["t"])).all(), f"{name} {_name(kn)}: NaN distances differ"
                rec["t"][np.isnan(rec["t"])] = np.nan
            check_records(g, rec, perm, misses, r1, f"{name} {_name(kn)}")
            if kn.get("count"):
                check_counters(st, c1, len(rays), f"{name} {_name(kn)}")
    finally:
        g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["collapsed_mesh", "collapsed_big", "coincident_spheres"])
def test_chain_scene_frame_equals_device_semantics(name, chain_scenes):
    from test_gpu_scale import _frame_vs_device_semantics
    _frame_vs_device_semantics(chain_scenes[2][name], 64, 48, 2, 4, name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["collapsed_big", "collapsed_many"])
def test_cli_with_device_bvh_renders_the_collapsed_mesh(name, chain_scenes):
    """cray_b200 --gpu-bvh on meshes of more than 1,024 triangles (the hook's threshold) with collapsed faces: 1,117 triangles with one
    cluster, whose tree fits in 2n - 1 nodes and is built on the device, and 1,228 with twelve, whose tree does not, so the device
    build refuses and the loader builds it on the host.  Either way the frame is the host-built scene's, bit for bit."""
    d, js, _ = chain_scenes
    _, _, nodes, _ = _loaded_trees(js[name])["mesh"]
    exe = os.path.join(ROOT, "c-ray_b200", "cray_b200")
    outs = []
    for extra in ([], ["--gpu-bvh"]):
        f32 = os.path.join(d, f"cli_{name}{len(outs)}.f32")
        r = subprocess.run([exe, js[name], "-d", "64x48", "-s", "4", "-b", "4", "--dump-f32", f32, "-o", os.path.join(d, "o.png"), "-q"]
                           + extra, cwd=d, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
        assert r.returncode == 0, r.stdout[-2000:]
        refused = extra and len(nodes) > 2 * MESH_TRIANGLES[name] - 1
        assert ("device BVH build failed" in r.stdout) == bool(refused), r.stdout[-2000:]
        if refused:
            assert f"needs {len(nodes)} nodes" in r.stdout and "building on the host" in r.stdout, r.stdout[-2000:]
        outs.append(np.fromfile(f32, dtype=np.float32))
    assert np.array_equal(outs[0].view(np.uint32), outs[1].view(np.uint32))
    assert (len(nodes) > 2 * MESH_TRIANGLES[name] - 1) == (name == "collapsed_many")


MESH_TRIANGLES = {"collapsed_big": 1100 + 17, "collapsed_many": 1024 + 12 * 17}


def edit_doc(cluster, spread, radius):
    """17 radius-0 spheres at `cluster` (one object), the spread spheres of the given radius (another) and a lit sphere"""
    doc = scene_doc(radius0_spheres(cluster), [])
    doc["scene"]["primitives"].append({"type": "sphere", "radius": radius, "color": [0.3, 0.6, 0.3],
                                       "instances": [{"transforms": [{"type": "translate", "X": float(p[0]), "Y": float(p[1]), "Z": float(p[2])}]}
                                                     for p in spread]})
    doc["scene"]["primitives"].append({"type": "sphere", "radius": 0.5, "color": [0.8, 0.3, 0.2],
                                       "instances": [{"transforms": [{"type": "translate", "X": 0.4, "Z": 6}]}]})
    return doc


def top_boxes(instances, radius):
    """the instance boxes of edit_doc's scenes, as the loader computes them for translated spheres"""
    c = instances["A"][:, [3, 7, 11]].astype(F32)
    r = np.zeros((len(c), 1), F32)
    r[17:-1], r[-1] = radius, 0.5
    return np.concatenate([-r + c, r + c], 1), c


@pytest.mark.gpu
@pytest.mark.parametrize("spread_count,radius,fits", [(23, 0.0, False), (600, 0.05, True)])
def test_moving_instances_onto_one_point(spread_count, radius, fits):
    """17 spread-out radius-0 spheres moved onto one point among other spheres.  The edit is accepted exactly when the reference's
    new top level fits in 2n - 1 nodes, and then the scene equals the edited JSON loaded fresh (frame, records, P/T/S/I); when it
    does not fit the edit is refused with CRGPU_ERR_UNSUPPORTED and the scene renders and traces as before."""
    from test_gpu_scene_edit import Loaded, assert_same_as_fresh, full, ray_set, traced
    rng = np.random.default_rng(spread_count)
    before_pos = np.round(rng.uniform(-2, 2, (17, 3)) + [0, 0, 6], 3)
    spread = np.round(rng.uniform(-2, 2, (spread_count, 3)) + [0, 0, 6], 3)
    cfg = (64, 48, 2, 4)
    a, b = Loaded(edit_doc(before_pos, spread, radius), *cfg), Loaded(edit_doc([[0.2, 0.1, 5.0]] * 17, spread, radius), *cfg)
    g = a.upload()
    try:
        rays = ray_set(b.camera)
        before_img, before_tr = full(g), traced(g, rays)
        nodes, _ = Reference(*top_boxes(b.instances, radius)).arrays()
        n = len(b.instances)
        assert chain(nodes)[1] == MAX_DEPTH and (len(nodes) <= 2 * n - 1) == fits
        inst = np.ascontiguousarray(b.instances)
        rc = crgpu.lib().crgpu_scene_set_instances(g.handle, inst.ctypes.data, n)
        assert (rc == 0) == fits, f"set_instances returned {rc} for a top level of {len(nodes)} nodes ({n} instances)"
        if fits:
            assert_same_as_fresh(g, b, rays)
        else:
            assert rc == CRGPU_ERR_UNSUPPORTED, rc
            img, tr = full(g), traced(g, rays)
            assert img.tobytes() == before_img.tobytes(), "a refused edit changed the frame"
            assert tr[0].tobytes() == before_tr[0].tobytes() and tr[1:] == before_tr[1:], "a refused edit changed the traversal"
    finally:
        g.close()
        a.free()
        b.free()
