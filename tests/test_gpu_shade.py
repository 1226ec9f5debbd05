"""GPU tests of the shading step that renders every frame — K4 + K3 (k_bucket, k_shade), the direction sort K4b and the tail
kernel (k_tail) — path state by path state, against the oracle in device semantics.

crgpu_shade_rays loads path states into the wave buffers and runs one bounce through the frame's own launch functions (K2 -> K4 ->
K3 -> K4b), or the tail kernel, which runs every path to its end.  The oracle's cro_path_step runs the same pathTrace loop body as
cro_render.  In semantics 1 it evaluates every libm call as the device does (the fp64 function rounded once to fp32, DESIGN.md §2),
so every field must be bit-identical: K2's record, alive, the next ray, weight, RNG state, L and the has-L bit.  A NaN equals any
NaN (CUDA and x86 differ in NaN payloads); -0 and +0 differ.  The one exemption is a state the oracle flags: a libm result within a
few fp64 ulps of an fp32 rounding boundary, which the device's fp64 routines may round the other way.  Flagged counts are printed and
must stay below 1e-5 of the states.

The states are the states of real paths at every bounce (golden, bundled and synthetic scenes), the same states made adversarial
(special weights, L poison, depths at the Russian-roulette and last-bounce edges, RNG states whose next draws are exactly 0 or 1),
in every K3 launch variant, both node interpreters, every direction-sort mode and batch sizes around the warp, block and grid.
The last part renders whole frames and requires the oracle's semantics-1 frame bit for bit outside pixels with a flagged sample.
"""
import ctypes as C
import json
import os

import numpy as np
import pytest

import crgpu
import oracle_lib as O
from conftest import GOLDEN, GOLDEN_FLAT, SUMMARY_LINES
from test_gpu_shade_order import _write_edge_scenes
from test_gpu_trace import _flat_arrays, _flatten, _write_synthetic
from test_oracle import _sweeps, same_bits

pytestmark = pytest.mark.gpu
TAIL_FROM, TAIL_MAX = 6, 16384            # CRG_TAIL_FROM (crgpu_api.cu), CRG_TAIL_MAX (crgpu_shade.cu)
BUNDLED = ["hdr", "scene", "refraction", "venus", "alphanode", "fence", "glowmetal", "statues", "uvsphere"]
# every K3 launch variant of the hit and miss kernels
LAUNCH = [dict(minb=m, split=s, prefetch=p) for m in (2, 3, 4) for s in (0, 1) for p in (0, 1)]
FLAG_SHARE = 1e-5                         # the near-tie exemption may cover at most this share of what a test compares


class Tally:
    """states (or samples) a test compared and how many of them the near-tie flag exempted"""
    def __init__(self, what):
        self.what, self.states, self.flagged = what, 0, 0

    def add(self, n, flagged):
        self.states += int(n)
        self.flagged += int(flagged)

    def check(self):
        line = f"{self.what}: {self.flagged} of {self.states} states / samples flagged"
        print(line)
        SUMMARY_LINES.append(line)
        assert self.states > 0, line
        assert self.flagged <= max(1, self.states * FLAG_SHARE), line


# ------------------------------------------------------------------------------------------------ scenes
NODE_DTYPE = np.dtype([("kind", "<i4"), ("in", "<i4", 3), ("f", "<f4", 8), ("tex", "<i4"), ("options", "<u4"), ("pad", "<u4", 2)])
TEX_DTYPE = np.dtype([("width", "<u4"), ("height", "<u4"), ("channels", "<u4"), ("is_float", "<u4"), ("has_alpha", "<u4"),
                      ("pad", "<u4"), ("data_offset", "<u8")])
MAT_DTYPE = np.dtype([("emission", "<f4", 4), ("IOR", "<f4"), ("bsdf", "<i4"), ("pad", "<u4", 2)])
SPHERE_DTYPE = np.dtype([("radius", "<f4"), ("ray_offset", "<f4"), ("material", "<u4"), ("pad", "<u4")])
CRS_IMG_NO_BILINEAR = 0x02                # include/crscene.h


def _view(ptr, count, dtype):
    return np.frombuffer((C.c_uint8 * (count * dtype.itemsize)).from_address(ptr), dtype=dtype)


def _write_deep(out):
    """g_legacy with two node graphs of its own (no JSON scene nests this deep):
    * its spheres: mix(red, blue, alpha(image with alpha)) — the only read of uv is through the alpha node, so the sphere-uv skip
      must know that an alpha node reads uv;
    * everything else: diffuse(checker(red, blue, grayscale(checker(black, grey, grayscale(checker(black, grey,
      grayscale(nearest-texel image))))))) — the image sits at the last level of the hot interpreter (NodeEval<0>), and on the mesh without uvs
      the checkers switch on the sign of p.x * p.y * p.z exactly when the level below is not black, so that image decides the
      top colour."""
    L = crgpu.lib()
    L.crscene_save.argtypes = [C.POINTER(crgpu.FlatScene), C.c_char_p]
    f = crgpu.FlatScene()
    assert L.crscene_load(C.byref(f), os.path.join(GOLDEN, "g_legacy.crscene").encode()) == 0
    nodes = list(_view(f.nodes, f.node_count, NODE_DTYPE).copy())
    texs = _view(f.textures, f.texture_count, TEX_DTYPE)
    alpha_tex = int(np.nonzero((texs["has_alpha"] != 0) & (texs["channels"] == 4))[0][0])

    def add(kind, ins=(-1, -1, -1), fs=(), tex=-1, options=0):
        n = np.zeros((), NODE_DTYPE)
        n["kind"] = kind
        n["in"] = list(ins) + [-1] * (3 - len(ins))
        n["f"][:len(fs)] = fs
        n["tex"] = tex
        n["options"] = options
        nodes.append(n)
        return len(nodes) - 1
    black, grey = add(32, fs=(0, 0, 0, 1)), add(32, fs=(0.05, 0.05, 0.05, 1))
    red, blue = add(32, fs=(0.9, 0.2, 0.2, 1)), add(32, fs=(0.2, 0.3, 0.9, 1))
    level = add(33, tex=0, options=CRS_IMG_NO_BILINEAR)     # 8-bit texels: none of the 256 levels squares to a near tie
    for top in (False, False, True):
        g = add(65, (level,))
        level = add(34, (red, blue, g) if top else (black, grey, g))
    deep = add(1, (level,))
    mix = add(5, (add(1, (red,)), add(1, (blue,)), add(66, (add(33, tex=alpha_tex),))))
    mats = _view(f.materials, f.material_count, MAT_DTYPE).copy()          # the loaded scene is read-only memory
    sphere_mats = set(_view(f.spheres, f.sphere_count, SPHERE_DTYPE)["material"].tolist())
    for i in range(f.material_count):
        mats["bsdf"][i] = mix if i in sphere_mats else deep
    arr = np.array(nodes, NODE_DTYPE)
    keep = f.nodes, f.node_count, f.materials
    f.nodes, f.node_count, f.materials = arr.ctypes.data, len(arr), mats.ctypes.data
    rc = L.crscene_save(C.byref(f), out.encode())
    f.nodes, f.node_count, f.materials = keep
    L.crscene_free(C.byref(f))
    assert rc == 0
    return out


def _write_noalpha(out):
    """g_nodes with its 8-bit RGBA texture marked has_alpha = 0 (a scene flattened from elsewhere may say so; this repository's
    loader never does) and every material mix(red, blue, alpha(checker(image, image))): the alpha node reads the image COLOUR's
    alpha lane through the checker, i.e. cr_texel, which must give 1 for a texture without alpha, like the oracle."""
    L = crgpu.lib()
    L.crscene_save.argtypes = [C.POINTER(crgpu.FlatScene), C.c_char_p]
    f = crgpu.FlatScene()
    assert L.crscene_load(C.byref(f), os.path.join(GOLDEN, "g_nodes.crscene").encode()) == 0
    nodes = list(_view(f.nodes, f.node_count, NODE_DTYPE).copy())
    texs = _view(f.textures, f.texture_count, TEX_DTYPE).copy()
    rgba = np.nonzero((texs["channels"] == 4) & (texs["is_float"] == 0))[0]
    assert len(rgba)
    texs["has_alpha"][rgba] = 0

    def add(kind, ins=(-1, -1, -1), fs=(), tex=-1, options=0):
        n = np.zeros((), NODE_DTYPE)
        n["kind"], n["in"], n["tex"], n["options"] = kind, list(ins) + [-1] * (3 - len(ins)), tex, options
        n["f"][:len(fs)] = fs
        nodes.append(n)
        return len(nodes) - 1
    t = int(rgba[0])
    red, blue = add(32, fs=(0.875, 0.25, 0.25, 1)), add(32, fs=(0.25, 0.375, 0.875, 1))
    ck = add(34, (add(33, tex=t), add(33, tex=t, options=CRS_IMG_NO_BILINEAR), add(64, fs=(7.0,))))
    mix = add(5, (add(1, (red,)), add(1, (blue,)), add(66, (ck,))))
    mats = _view(f.materials, f.material_count, MAT_DTYPE).copy()
    mats["bsdf"] = mix
    arr = np.array(nodes, NODE_DTYPE)
    keep = f.nodes, f.node_count, f.materials, f.textures
    f.nodes, f.node_count, f.materials, f.textures = arr.ctypes.data, len(arr), mats.ctypes.data, texs.ctypes.data
    rc = L.crscene_save(C.byref(f), out.encode())
    f.nodes, f.node_count, f.materials, f.textures = keep
    L.crscene_free(C.byref(f))
    assert rc == 0
    return out


# spheres of the JSON shading scene: (x, y, z, radius, material); the aimed states below find them by position
SHADING_SPHERES = [
    (-3.0, 0.0, 0.0, 0.5, {"type": "diffuse", "color": {"path": "rgb.png", "lerp": True, "transform": True}}),      # 7 px wide, bilinear, sRGB
    (-2.0, 0.0, 0.0, 0.5, {"type": "diffuse", "color": {"path": "rgba.png", "lerp": False, "transform": False}}),   # 16 px wide, nearest, linear
    (-1.0, 0.0, 0.0, 0.5, {"type": "metal", "color": {"path": "rgb.png", "lerp": False}, "roughness": {"path": "gray.png", "lerp": True}}),
    (0.0, 0.0, 0.0, 0.5, {"type": "glass", "color": [1, 1, 1], "roughness": 0.0, "IOR": 1.5}),
    (1.0, 0.0, 0.0, 0.5, {"type": "glass", "color": [0.9, 1, 0.9], "roughness": 0.3, "IOR": 1.5}),
    (2.0, 0.0, 0.0, 0.5, {"type": "glass", "color": [1, 1, 1], "roughness": 0.0, "IOR": 1.0}),
    (3.0, 0.0, 0.0, 0.5, {"type": "plastic", "color": {"path": "rgba.png", "lerp": True}}),
    (-3.0, 1.2, 0.0, 0.5, {"type": "diffuse", "color": [0.5, 0.5, 0.5]}),                                              # Russian roulette p = 0.5
    (-2.0, 1.2, 0.0, 0.5, {"type": "diffuse", "color": [0, 0, 0]}),                                                    # p = 0
    (-1.0, 1.2, 0.0, 0.5, {"type": "mix", "A": {"type": "diffuse", "color": [0.9, 0.1, 0.1]},
                           "B": {"type": "metal", "color": [0.9, 0.9, 0.9], "roughness": 0.0}, "factor": 0.5}),          # lerp 0.5
    (0.0, 1.2, 0.0, 0.5, {"type": "mix", "A": {"type": "diffuse", "color": [0.9, 0.1, 0.1]}, "B": {"type": "transparent", "color": [1, 1, 1]},
                          "factor": 0.0}),
    (1.0, 1.2, 0.0, 0.5, {"type": "mix", "A": {"type": "diffuse", "color": [0.9, 0.1, 0.1]}, "B": {"type": "transparent", "color": [1, 1, 1]},
                          "factor": 1.0}),
    (2.0, 1.2, 0.0, 0.5, {"type": "add", "A": {"type": "diffuse", "color": [0.2, 0.3, 0.4]}, "B": {"type": "metal", "color": [0.5, 0.5, 0.5], "roughness": 0.2}}),
    (3.0, 1.2, 0.0, 0.5, {"type": "diffuse", "color": {"type": "checkerboard", "size": 9}}),
] + [(-3.0 + k, 2.4, 0.0, 0.5, {"type": "emissive", "color": {"type": "blackbody", "degrees": t}, "strength": 2})
     for k, t in enumerate((1899, 1900, 1901, 6599, 6600, 6601, 40000, 4000000))]


def _write_shading(d):
    """A JSON scene of the shading paths no bundled scene isolates (SHADING_SPHERES), two textured quads — one with texture
    coordinates at 0, 1, just outside [0, 1] and up to 3e9 (cr_wrap's 64-bit branch and the (size_t) conversion's limits), one
    without any — and a gradient background with an offset.  (Isotropic has no JSON path; g_f4 holds the one node graph that does.)"""
    import shutil
    os.makedirs(d, exist_ok=True)
    for a in ("rgb.png", "rgba.png", "gray.png"):
        shutil.copy(os.path.join(GOLDEN, "assets", a), os.path.join(d, a))
    open(os.path.join(d, "tex.mtl"), "w").write("newmtl t\nKd 1 1 1\nmap_Kd rgb.png\nnewmtl u\nKd 1 1 1\nmap_Kd rgba.png\n")
    open(os.path.join(d, "uvquad.obj"), "w").write(
        "mtllib tex.mtl\nv -1 -1 0\nv 1 -1 0\nv 1 1 0\nv -1 1 0\nvt -0.0000001 0\nvt 1.0000001 1\nvt 3e9 -3e9\nvt 1 0\n"
        "vn 0 0 -1\nusemtl t\nf 1/1/1 2/4/1 3/2/1\nf 1/1/1 3/2/1 4/3/1\n")
    open(os.path.join(d, "flatquad.obj"), "w").write(
        "mtllib tex.mtl\nv -1 -1 0\nv 1 -1 0\nv 1 1 0\nv -1 1 0\nvn 0 0 -1\nusemtl u\nf 1//1 2//1 3//1\nf 1//1 3//1 4//1\n")
    def absolute(m):                      # node-graph texture paths resolve against the working directory, as in the reference
        if isinstance(m, dict):
            return {k: (os.path.join(d, v) if k == "path" else absolute(v)) for k, v in m.items()}
        return m
    prims = [{"type": "sphere", "radius": r, "material": absolute(m), "instances": [{"transforms": [{"type": "translate", "X": x, "Y": y, "Z": z}]}]}
             for x, y, z, r, m in SHADING_SPHERES]
    meshes = [{"fileName": "uvquad.obj", "instances": [{"transforms": [{"type": "translate", "X": -1.5, "Y": -1.5, "Z": 0.5}]}]},
              {"fileName": "flatquad.obj", "instances": [{"transforms": [{"type": "translate", "X": 1.5, "Y": -1.5, "Z": 0.5}]}]}]
    sc = {"renderer": {"width": 64, "height": 40, "samples": 4, "bounces": 8},
          "camera": {"FOV": 80, "transforms": [{"type": "translate", "X": 0, "Y": 0.4, "Z": -4.5}]},
          "scene": {"ambientColor": {"down": [0.6, 0.5, 0.4], "up": [0.5, 0.7, 1.0], "offset": 30}, "primitives": prims, "meshes": meshes}}
    p = os.path.join(d, "syn_shading.json")
    open(p, "w").write(json.dumps(sc))
    return p


@pytest.fixture(scope="module")
def scenes(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("shade_scenes"))
    out = {n: os.path.join(GOLDEN, n + ".crscene") for n in GOLDEN_FLAT}
    for n in BUNDLED:
        p = O.bundled_scene(n, d)
        if p:
            out[n] = p
    for n, p in _write_synthetic(os.path.join(d, "syn")).items():
        out[n] = _flatten(p, os.path.join(d, n + ".crscene"))
    out["syn_deep"] = _write_deep(os.path.join(d, "syn_deep.crscene"))
    out["syn_noalpha"] = _write_noalpha(os.path.join(d, "syn_noalpha.crscene"))
    out["syn_shading"] = _flatten(_write_shading(os.path.join(d, "shading")), os.path.join(d, "syn_shading.crscene"))
    os.makedirs(os.path.join(d, "edge"))
    for n, p in _write_edge_scenes(os.path.join(d, "edge")).items():
        out[n] = _flatten(p, os.path.join(d, n + ".crscene"))
    return out


# bundled scenes at small sizes: the states of a block of pixels
CONFIG = {"hdr": (96, 54, 2, 32), "scene": (80, 50, 2, 4), "refraction": (64, 36, 2, 512), "venus": (40, 64, 2, 25),
          "alphanode": (96, 60, 2, 0), "fence": (96, 60, 2, 0), "glowmetal": (96, 60, 2, 0), "statues": (96, 60, 2, 0),
          "uvsphere": (96, 60, 2, 0)}


def open_oracle(name, path):
    W, H, spp, b = CONFIG.get(name, (0, 0, 0, 0))
    return O.OracleScene(path, W, H, spp, b), (W, H, spp, b)


def open_gpu(name, path):
    W, H, spp, b = CONFIG.get(name, (0, 0, 0, 0))
    return crgpu.GpuScene(path, W, H, spp, b)


def path_states(o, block=(32, 24), max_states=1 << 16):
    """{depth: states} of every path of a block of pixels, from the oracle in device semantics"""
    W, H = o.W, o.H
    bw, bh = min(W, block[0]), min(H, block[1])
    x0, y0 = (W - bw) // 2, (H - bh) // 2
    cur = o.camera_states(x0, y0, x0 + bw, y0 + bh, passes=(0, min(2, o.s.prefs.sample_count)))[:max_states]
    cur["pad"] = 0
    out = {}
    for depth in range(o.s.prefs.bounces):
        if len(cur) == 0:
            break
        out[depth] = cur.copy()
        r = o.path_step(cur, depth)
        cur = r["next"][r["alive"] != 0]
    return out


# ------------------------------------------------------------------------------------------------ comparison
def expected_key(rec):
    return np.where(rec["inst"] >= 0, np.minimum(rec["material"] + 1, 255), 0).astype(np.uint32)


def host_dir_bin(o, d, p, mode):
    """cr_dir_bin (crgpu_shade.cu) for modes 1-3, in fp32"""
    key = (np.signbit(d[:, 0]).astype(np.uint32) | (np.signbit(d[:, 1]).astype(np.uint32) << 1) | (np.signbit(d[:, 2]).astype(np.uint32) << 2))
    if mode == 2:
        a = np.abs(d)
        major = np.where((a[:, 0] >= a[:, 1]) & (a[:, 0] >= a[:, 2]), 0, np.where(a[:, 1] >= a[:, 2], 1, 2)).astype(np.uint32)
        key |= major << 3
    elif mode == 3:
        f = _flat_arrays(o.s)
        top = f["bvh"][f["top"]]
        b = f["node"][top["node_offset"]]["bounds"] if top["node_count"] >= 1 else np.array([0, 1, 0, 1, 0, 1], np.float32)
        lo, hi = b[0::2].astype(np.float32), b[1::2].astype(np.float32)
        e = hi - lo
        inv = np.where((e > 0) & (e < np.float32(3.0e38)), np.float32(1) / np.where(e > 0, e, np.float32(1)), np.float32(0)).astype(np.float32)
        with np.errstate(all="ignore"):
            fr = ((p - lo) * inv).astype(np.float32)
            cell = lambda v, k, m: np.fmin(np.fmax(v * np.float32(k), np.float32(0)), np.float32(m)).astype(np.uint32)
            key |= (cell(fr[:, 0], 4, 3) << 3) | (cell(fr[:, 2], 4, 3) << 5) | (cell(fr[:, 1], 2, 1) << 7)
    return key


def check_step(o, res, perm2, surv, exp, tally, what, dirmode=0, tail=False):
    """device results vs oracle semantics-1 step results, bit for bit outside states whose step the oracle flagged (both sides
    start from the same input state, so only a near tie inside this step can separate them)"""
    n = len(exp)
    flag = exp["flag"] != 0
    ok = ~flag
    tally.add(n, flag.sum())

    def bad(mask, field):
        idx = np.nonzero(mask & ok)[0]
        assert len(idx) == 0, f"{what}: {field} differs on {len(idx)} of {n} states, first {idx[:6]}"

    if not tail:
        r, e = res["rec"], exp["rec"]
        bad(r["inst"] != e["inst"], "hit instance")
        bad(~same_bits(r["t"], e["t"]), "hit distance")
        bad(r["poly"] != e["poly"], "hit poly")
        mesh = e["poly"] >= 0
        bad(mesh & (~same_bits(r["u"], e["u"]) | ~same_bits(r["v"], e["v"])), "hit u/v")
        bad(r["key"] != expected_key(e), "shading key")
    alive = exp["alive"] != 0
    bad((res["alive"] != 0) != alive, "alive")
    a = alive & (res["alive"] != 0)
    g, x = res["next"], exp["next"]
    for f in ("o", "d", "weight"):
        bad(a & ~same_bits(g[f], x[f]).all(axis=1), f"next {f}")
    bad(a & (g["rng"] != x["rng"]), "rng state")
    bad(a & (g["has_l"] != x["has_l"]), "has-L")
    with_l = ~alive | (x["has_l"] != 0)
    bad(with_l & ~same_bits(g["L"], x["L"]).all(axis=1), "L")
    assert surv == int((res["alive"] != 0).sum()), what
    if not tail:
        slots = np.sort(res["slot"][res["alive"] != 0])
        assert np.array_equal(slots, np.arange(surv, dtype=np.uint32)), f"{what}: survivor slots are not 0..{surv}"
    if dirmode and surv and not tail:
        assert np.array_equal(np.sort(perm2), np.arange(surv, dtype=np.uint32)), f"{what}: perm2 is not a permutation"
        live = np.nonzero(res["alive"] != 0)[0]
        key_of_slot = np.zeros(surv, np.uint32)
        key_of_slot[res["slot"][live]] = res["dir_key"][live]
        assert (np.diff(key_of_slot[perm2].astype(np.int64)) >= 0).all(), f"{what}: perm2 is not in key order"
        octant = host_dir_bin(o, g["d"][live], g["o"][live], 1)
        assert np.array_equal(res["dir_key"][live] & 7, octant), f"{what}: direction octant"
        if dirmode in (1, 2, 3):
            hk = host_dir_bin(o, g["d"][live], g["o"][live], dirmode)
            assert np.array_equal(res["dir_key"][live], hk), f"{what}: direction key differs from the host bin"
    return int(flag.sum())


def run_step(g, o, states, tally, depth, max_depth, what, exp=None, **opts):
    """one device step vs the oracle's (exp: the oracle's results when already computed); returns (device, oracle) results"""
    tail = opts.get("tail", 0)
    if exp is None:
        exp = o.path_step(states, depth, max_depth, bounces=(1 << 30) if tail else 1)
    res, perm2, surv, box = g.shade_rays(states, depth, max_depth, **opts)
    check_step(o, res, perm2, surv, exp, tally, what, opts.get("dirmode", 0), bool(tail))
    return res, exp


# ------------------------------------------------------------------------------------------------ the libm stand-ins
def test_device_libm_matches_device_semantics():
    """crgpu_math.cuh's stand-ins on the device equal the oracle's semantics 1 bit for bit wherever the oracle does not flag a near
    tie: the same sweeps the CPU suite checks against 80-bit evaluation, plus schlick's pow5 and both halves of sincos."""
    total = flagged = 0
    sweeps = _sweeps()
    trig = [s for s in sweeps if s[0] == "sin"][0][1]
    rng = np.random.default_rng(3)
    p5 = np.concatenate([trig, rng.uniform(0, 2, 20000).astype(np.float32)])
    jobs = [(fn, x, y, fn) for fn, x, y in sweeps] + [("pow5", p5, None, "pow5"), ("sincos_sin", trig, None, "sin"), ("sincos_cos", trig, None, "cos")]
    for dev_fn, x, y, ora_fn in jobs:
        got = crgpu.libm_eval(dev_fn, x, y)
        exp, flag = O.libm(ora_fn, O.SEM_DEVICE, x, y)
        bad = np.nonzero(~same_bits(got, exp) & ~flag)[0]
        assert len(bad) == 0, (dev_fn, x[bad[:5]], None if y is None else y[bad[:5]], got[bad[:5]], exp[bad[:5]])
        total += len(x)
        flagged += int(flag.sum())
    tally = Tally("device libm vs semantics 1")
    tally.add(total, flagged)
    tally.check()


# ------------------------------------------------------------------------------------------------ real path states
SCENES = GOLDEN_FLAT + BUNDLED + ["syn_ties", "syn_materials", "syn_single", "syn_onetri", "syn_deep", "syn_noalpha", "syn_shading", "syn_allmiss", "syn_nomiss"]


@pytest.mark.parametrize("name", SCENES)
def test_real_path_states(name, scenes):
    """Every bounce of the paths of a block of pixels: the default launch at every depth; every K3 launch variant, the complete
    interpreter and every direction-sort mode at the first bounces, at depth 4 (Russian roulette starts) and at the last bounce;
    the tail kernel from bounce CRG_TAIL_FROM on."""
    if name not in scenes:
        pytest.skip(f"{name}: bundled scenes need scenes/_built or oracle/_ref/input")
    o, _ = open_oracle(name, scenes[name])
    g = open_gpu(name, scenes[name])
    B = o.s.prefs.bounces
    per_depth = path_states(o)
    full = {0, 1, 4, 5, B - 1}
    n_states = 0
    tally = Tally(f"real path states, {name}")
    for depth, st in sorted(per_depth.items()):
        n_states += len(st)
        if depth > 40 and depth not in full:
            continue
        variants = [dict()]
        if depth in full:
            variants = LAUNCH + [dict(complete_interpreter=1), dict(complete_interpreter=1, split=0)] + [dict(dirmode=m) for m in (1, 2, 3, 4, 4)]
        exp = o.path_step(st, depth, B)
        for kn in variants:
            run_step(g, o, st, tally, depth, B, f"{name} depth {depth} {kn}", exp=exp, **kn)
        if depth >= TAIL_FROM and len(st) <= TAIL_MAX and (depth in full or depth == TAIL_FROM):
            exp = o.path_step(st, depth, B, bounces=1 << 30)
            for kn in (dict(tail=1), dict(tail=1, complete_interpreter=1)):
                run_step(g, o, st, tally, depth, B, f"{name} tail from {depth} {kn}", exp=exp, **kn)
    assert n_states > 0
    tally.check()
    g.close()
    o.close()


# ------------------------------------------------------------------------------------------------ adversarial states
MULT, INC = 6364136223846793005, 1
MULT_INV = pow(MULT, -1, 1 << 64)


def state_with_draw(u32, k, rng):
    """a PCG state whose k-th next output (k >= 1) is u32: the output function is inverted with rot = 0 and the LCG run back"""
    t = [(u32 >> i) & 1 for i in range(32)]
    x = [0] * 64
    for b in range(27):
        x[b] = int(rng.integers(0, 2))
    for kbit in range(58, 26, -1):                    # y = x ^ (x >> 18); output bits = y[27..58]
        x[kbit] = t[kbit - 27] ^ (x[kbit + 18] if kbit + 18 < 64 else 0)
    s = sum(b << i for i, b in enumerate(x))
    for _ in range(k - 1):
        s = ((s - INC) * MULT_INV) % (1 << 64)
    return s


def pcg_draws(state, k):
    out = []
    for _ in range(k):
        old = state
        state = (old * MULT + INC) % (1 << 64)
        xs = (((old >> 18) ^ old) >> 27) & 0xFFFFFFFF
        rot = old >> 59
        out.append(((xs >> rot) | (xs << ((-rot) & 31))) & 0xFFFFFFFF)
    return out


def test_rng_inversion():
    rng = np.random.default_rng(1)
    for u, k in ((0xFFFFFFFF, 1), (0, 3), (0x12345678, 5), (0xFFFFFF80, 2)):
        s = state_with_draw(u, k, rng)
        assert pcg_draws(s, k)[-1] == u


def adversarial(o, st, rng, depth):
    """variants of real states: special weights, L inputs with and without has-L, and RNG states whose 1st / 2nd / 3rd draw is
    exactly 0.0f or 1.0f (the Russian-roulette draw of a diffuse bounce is the 3rd, a glass / plastic / mix decision the 1st)"""
    out = []
    w_special = np.array([0.0, -0.0, 1e-45, -1e-40, -0.5, 1e30, -1e30, np.inf, -np.inf, np.nan], np.float32)
    k = min(len(st), 64)
    base = st[rng.choice(len(st), k, replace=False)]
    for w in w_special:
        s = base.copy()
        s["weight"][:, rng.integers(0, 3)] = w
        out.append(s)
        s = base.copy()
        s["weight"] = w
        out.append(s)
    for L, has in ((np.nan, 0), (np.float32(-1.5e38), 0), (1.25, 1), (-0.0, 1), (np.inf, 1), (0.0, 1)):
        s = base.copy()
        s["L"] = L
        s["has_l"] = has
        out.append(s)
    for u in (0xFFFFFFFF, 0xFFFFFF80, 0):              # draws of exactly 1.0f (both) and 0.0f
        for kk in (1, 2, 3):
            s = base.copy()
            s["rng"] = np.array([state_with_draw(u, kk, rng) for _ in range(len(s))], np.uint64)
            out.append(s)
    return np.concatenate(out)


@pytest.mark.parametrize("name", ["g_nodes", "g_f4", "g_single", "glowmetal", "refraction", "hdr", "uvsphere", "fence"])
def test_adversarial_states(name, scenes):
    """Real states made adversarial, at depths 0, 3, 4, maxDepth - 1 and (tail) CRG_TAIL_FROM and beyond."""
    if name not in scenes:
        pytest.skip(f"{name}: bundled scenes need scenes/_built or oracle/_ref/input")
    o, _ = open_oracle(name, scenes[name])
    g = open_gpu(name, scenes[name])
    per_depth = path_states(o, block=(16, 16))
    st = np.concatenate(list(per_depth.values()))
    rng = np.random.default_rng(sum(map(ord, name)))
    adv = adversarial(o, st, rng, 0)
    tally = Tally(f"adversarial states, {name}")
    B = max(o.s.prefs.bounces, 1)
    for depth, md in ((0, B), (3, max(B, 8)), (4, max(B, 8)), (B - 1, B), (4, 5), (0, 1)):
        if depth >= md:
            continue
        exp = o.path_step(adv, depth, md)
        for kn in (dict(), dict(split=0), dict(minb=4, prefetch=1), dict(dirmode=2)):
            run_step(g, o, adv, tally, depth, md, f"{name} adversarial depth {depth}/{md} {kn}", exp=exp, **kn)
    for depth, md in ((TAIL_FROM, max(B, TAIL_FROM + 8)), (TAIL_FROM + 3, max(B, TAIL_FROM + 4))):
        run_step(g, o, adv, tally, depth, md, f"{name} adversarial tail {depth}/{md}", tail=1)
    tally.check()
    g.close()
    o.close()


# ------------------------------------------------------------------------------------------------ aimed states
def aimed_states(rng):
    """States aimed at computed points of the JSON shading scene (syn_shading), each with ten RNG states, and what they reach:
    * every sphere head-on, at both poles (d = -y / +y through the pole: asin(+-1)), on the seam (z = +0 and z = -0 at x = -r:
      atan2(+-0, -1) = +-pi) and from its centre (back faces: the hit point is reached from inside);
    * the plain glass sphere from inside at (0.9 r, 0, 0) along +y: 64 degrees of incidence, total internal reflection;
    * the textured quad at its vertices and edge midpoints: texture coordinates exactly 0 and 1, -1e-7 and 1 + 1e-7, and 3e9
      (cr_wrap's 64-bit branch and the (size_t) conversion of a large coordinate); the quad without coordinates likewise (uv = -1);
    * background directions from far outside the world: +-y with x and z +0 / -0, subnormal components, all-subnormal (its
      length underflows), and large unnormalised vectors;
    * RNG states whose 1st, 2nd or 3rd draw is exactly 0.5f, 1.0f or 0.0f: draw == lerp on the mix with factor 0.5 (1st draw),
      draw == probability in Russian roulette on the grey diffuse sphere (p = 0.5, 3rd draw), p = 0 at draw 0 on the black one
      (1/p = inf), mix factor 0 at draw 0 and factor 1 at draw 1, and total internal reflection at draw 1.0f (deviation 3)."""
    o, d = [], []

    def ray(org, dirn):
        o.append(org)
        d.append(dirn)
    for x, y, z, r, _ in SHADING_SPHERES:
        c = np.array([x, y, z], np.float64)
        ray(c + (0, 0, -3 * r), (0, 0, 1))
        ray(c + (0, 3 * r, 0), (0, -1, 0))
        ray(c - (0, 3 * r, 0), (0, 1, 0))
        ray(c + (-3 * r, 0, 0), (1, 0, 0))
        ray(c + (-3 * r, 0, 0), (1, 0, -0.0))
        for v in rng.normal(size=(4, 3)):
            ray(c, v / np.linalg.norm(v))
    ray((0.45, 0.0, 0.0), (0, 1, 0))                                     # inside the IOR 1.5 glass sphere at the origin
    for qx in (-1.5, 1.5):                                               # the two quads (z = 0.5)
        for px, py in ((-1, -1), (1, -1), (1, 1), (-1, 1), (0, -1), (1, 0), (0, 1), (-1, 0), (0, 0), (0.999, 0.999), (-0.999, 0.5)):
            ray((qx + px, -1.5 + py, -2.0), (0, 0, 1))
    far = (100.0, 100.0, 100.0)
    for v in ((0, 1, 0), (0, -1, 0), (-0.0, 1, 0), (0, 1, -0.0), (-0.0, -1, -0.0), (1e-45, 1, 0), (0, 1e-45, 1), (1e-40, -1e-40, 1),
              (1e-45, 1e-45, 1e-45), (1e30, 2e30, -3e30), (3e38, 0, 0), (-1e-3, 5e3, 2e2), (0, 0, 1), (0, 0, -1), (1, 0, 0)):
        ray(far, v)
    n = len(o)
    base = np.zeros(n, crgpu.PATH_STATE_DTYPE)
    base["o"] = np.array(o, np.float32)
    base["d"] = np.array(d, np.float32)
    base["weight"] = 1.0
    out = []
    for u, k in [(None, 0)] + [(u, k) for u in (1 << 31, 0xFFFFFFFF, 0) for k in (1, 2, 3)]:
        st = base.copy()
        st["rng"] = np.array([int(rng.integers(0, 1 << 63)) if u is None else state_with_draw(u, k, rng) for _ in range(n)], np.uint64)
        out.append(st)
    return np.concatenate(out)


def test_aimed_states(scenes):
    """aimed_states() in every K3 launch variant, both interpreters and every sort mode, at depth 0, at depth 4 (Russian roulette),
    at the last bounce, and through the tail kernel."""
    name = "syn_shading"
    o = O.OracleScene(scenes[name])
    g = crgpu.GpuScene(scenes[name])
    st = aimed_states(np.random.default_rng(17))
    B = o.s.prefs.bounces
    tally = Tally("aimed states")
    reached = o.path_step(st, 0)
    assert (reached["rec"]["inst"] < 0).sum() >= 15 * 10 and (reached["rec"]["poly"] >= 0).sum() >= 22 * 10
    for depth in (0, 4, B - 1):
        exp = o.path_step(st, depth, B)
        for kn in LAUNCH + [dict(complete_interpreter=1), dict(complete_interpreter=1, split=0)] + [dict(dirmode=m) for m in (1, 2, 3, 4)]:
            run_step(g, o, st, tally, depth, B, f"{name} aimed depth {depth} {kn}", exp=exp, **kn)
    for kn in (dict(tail=1), dict(tail=1, complete_interpreter=1)):
        run_step(g, o, st, tally, TAIL_FROM, B + TAIL_FROM, f"{name} aimed tail {kn}", **kn)
    tally.check()
    g.close()
    o.close()


# ------------------------------------------------------------------------------------------------ batch sizes
def _pool(o, n):
    st = np.concatenate(list(path_states(o, block=(48, 32)).values()))
    return st[np.resize(np.arange(len(st)), n)]


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 255, 256, 257, 132 * 8 * 256 + 77])
def test_batch_sizes(n, scenes):
    """Empty, single, warp-, block- and grid-edge batches (132 SMs x 8 blocks x 256 threads: the grid-stride loop and the
    prefetch guard)."""
    name = "hdr" if "hdr" in scenes else "g_nodes"
    o, _ = open_oracle(name, scenes[name])
    g = open_gpu(name, scenes[name])
    st = _pool(o, n)
    tally = Tally(f"batch of {n}")
    exp = o.path_step(st, 1)
    for kn in (dict(), dict(split=0, prefetch=1), dict(prefetch=1), dict(dirmode=1)):
        run_step(g, o, st, tally, 1, o.s.prefs.bounces, f"{name} n={n} {kn}", exp=exp, **kn)
    if n:
        tally.check()
    g.close()
    o.close()


def test_all_misses_and_no_misses(scenes):
    name = "g_legacy"
    o, _ = open_oracle(name, scenes[name])
    g = open_gpu(name, scenes[name])
    st = _pool(o, 4096)
    r = o.path_step(st, 1)
    tally = Tally("all misses and no misses")
    for sel, what in ((r["rec"]["inst"] < 0, "all misses"), (r["rec"]["inst"] >= 0, "no misses")):
        s = st[sel]
        assert len(s)
        exp = o.path_step(s, 1)
        for kn in LAUNCH:
            run_step(g, o, s, tally, 1, o.s.prefs.bounces, f"{name} {what} {kn}", exp=exp, **kn)
    tally.check()
    g.close()
    o.close()


def test_tail_limits(scenes):
    """The tail kernel runs CRG_TAIL_MAX paths to their end, and leaves CRG_TAIL_MAX + 1 untouched: the live count stays, and so
    do the states and L."""
    name = "refraction" if "refraction" in scenes else "g_nodes"
    o, _ = open_oracle(name, scenes[name])
    g = open_gpu(name, scenes[name])
    st = _pool(o, TAIL_MAX + 1)
    st["L"] = np.float32(7.5)
    md = max(o.s.prefs.bounces, TAIL_FROM + 4)
    tally = Tally("tail limits")
    run_step(g, o, st[:TAIL_MAX], tally, TAIL_FROM, md, f"{name} tail n={TAIL_MAX}", tail=1)
    tally.check()
    res, _, surv, _ = g.shade_rays(st, TAIL_FROM, md, tail=1)
    assert surv == TAIL_MAX + 1 and (res["alive"] == 1).all()
    for f in ("o", "d", "weight", "rng", "has_l"):
        assert res["next"][f].tobytes() == st[f].tobytes(), f
    assert (res["next"]["L"] == np.float32(7.5)).all()
    g.close()
    o.close()


# ------------------------------------------------------------------------------------------------ whole frames
FRAMES = [(n, 0, 0, 0, 0) for n in GOLDEN_FLAT] + [(n, 0, 0, 0, 0) for n in ("syn_ties", "syn_materials", "syn_single", "syn_onetri", "syn_deep", "syn_noalpha", "syn_shading", "syn_allmiss", "syn_nomiss")] + \
         [("hdr", 240, 135, 16, 32), ("scene", 320, 200, 16, 4), ("refraction", 240, 135, 8, 512), ("venus", 100, 160, 16, 25),
          ("alphanode", 96, 60, 8, 0), ("fence", 96, 60, 8, 0), ("glowmetal", 96, 60, 8, 0), ("statues", 96, 60, 8, 0),
          ("uvsphere", 96, 60, 8, 0)]


@pytest.mark.parametrize("name,W,H,spp,b", FRAMES)
def test_frame_equals_device_semantics(name, W, H, spp, b, scenes):
    """The GPU frame equals the oracle's semantics-1 frame bit for bit, except in pixels with a flagged sample."""
    if name not in scenes:
        pytest.skip(f"{name}: bundled scenes need scenes/_built or oracle/_ref/input")
    g = crgpu.GpuScene(scenes[name], W, H, spp, b)
    g.render_frame()
    img = g.read()
    g.close()
    o = O.OracleScene(scenes[name], W, H, spp, b)
    ref, flagged = o.render_sem(O.SEM_DEVICE)
    samples = int(o.W * o.H * o.s.prefs.sample_count)
    o.close()
    differ = (~same_bits(img, ref)).any(axis=2)
    tally = Tally(f"frame {name}")
    tally.add(samples, flagged.sum())
    tally.check()
    bad = np.nonzero(differ & (flagged == 0))
    assert len(bad[0]) == 0, f"{name}: {len(bad[0])} unflagged pixels differ, first rows {bad[0][:5]} cols {bad[1][:5]}"
