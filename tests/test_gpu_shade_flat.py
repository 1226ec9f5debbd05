"""The flat hit launch of K3: materials of a fixed form, folded at upload and sampled without the node interpreter.

A material is flat when its graph is a leaf (diffuse, metal, glass, emissive, or plastic over a diffuse) whose inputs are constants
or one image colour, alone or under the loader's legacy wrapper Mix(Transparent(constant), leaf, Alpha(colour)).  K4 puts their
buckets right behind the misses and K3 shades them in a launch of their own; every other hit goes to the interpreter.

* CPU: which materials of every bundled, golden and synthetic scene are flat, against an independent reading of the node graphs
  and against what the scenes are known to hold.
* GPU: path states through crgpu_shade_rays with the flat launch (generic_only = 0) and without it (generic_only = 1), bit for bit
  against each other and against the oracle in device semantics, at every bounce and in sort modes 0 and 4; wrapper states whose
  alpha draw lands below, above and exactly on an image alpha; a scene that mixes flat and generic materials in one bounce; one
  with more than 254 materials (the overflow key 255 is generic); and whole frames with CRGPU_SHADE_GENERIC_ONLY=1.
"""
import ctypes as C
import os

import numpy as np
import pytest

import crgpu
import oracle_lib as O
from conftest import GOLDEN, GOLDEN_FLAT
from test_gpu_shade import (MAT_DTYPE, NODE_DTYPE, SHADING_SPHERES, SPHERE_DTYPE, TEX_DTYPE, Tally, _view, check_step, open_gpu,
                            open_oracle, path_states, scenes, state_with_draw)      # noqa: F401  (scenes is a fixture)
from test_gpu_trace import _frames
from test_oracle import same_bits

CRS_IMG_NO_BILINEAR = 0x02
# include/crscene.h node kinds
DIFFUSE, METAL, GLASS, PLASTIC, MIX, ADD, TRANSPARENT, EMISSIVE = 1, 2, 3, 4, 5, 6, 7, 8
COLOR_CONSTANT, COLOR_IMAGE, VALUE_CONSTANT, VALUE_ALPHA = 32, 33, 64, 66
# crgpu_prepared_materials: kinds and flags
FLAT_KIND = {DIFFUSE: 1, METAL: 2, GLASS: 3, EMISSIVE: 4, PLASTIC: 5}
WRAPPED, ALPHA_IMG, COL_IMG = 1, 2, 4


# ------------------------------------------------------------------------------------------------ classification (CPU)
def _load(path):
    L = crgpu.lib()
    f = crgpu.FlatScene()
    assert L.crscene_load(C.byref(f), path.encode()) == 0, path
    return L, f


def device_classes(path):
    """(kinds, flags) per material, as crgpu_prepare folded them"""
    L, f = _load(path)
    L.crgpu_prepare.argtypes = [C.POINTER(crgpu.FlatScene), C.POINTER(C.c_void_p)]
    L.crgpu_prepared_free.argtypes = [C.c_void_p]
    L.crgpu_prepared_materials.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    p = C.c_void_p()
    rc = L.crgpu_prepare(C.byref(f), C.byref(p))
    n = f.material_count
    L.crscene_free(C.byref(f))
    assert rc == 0, path
    kinds, flags, count = np.zeros(n, np.uint32), np.zeros(n, np.uint32), C.c_uint32()
    rc = L.crgpu_prepared_materials(p, kinds.ctypes.data, flags.ctypes.data, n, C.byref(count))
    L.crgpu_prepared_free(p)
    assert rc == 0 and count.value == n
    return kinds, flags


def expected_classes(path):
    """the same split read off the node graphs here: (kind, flags) per material"""
    L, f = _load(path)
    nodes = _view(f.nodes, f.node_count, NODE_DTYPE).copy()
    mats = _view(f.materials, f.material_count, MAT_DTYPE).copy()
    L.crscene_free(C.byref(f))

    def kind(i):
        return int(nodes[i]["kind"]) if 0 <= i < len(nodes) else -1

    def inp(i, k):
        return int(nodes[i]["in"][k])

    def colour(i):                        # 0 = constant, COL_IMG = image, None = anything else
        return {COLOR_CONSTANT: 0, COLOR_IMAGE: COL_IMG}.get(kind(i))

    def leaf(i):
        k = kind(i)
        c = colour(inp(i, 0)) if k in (DIFFUSE, METAL, GLASS, EMISSIVE) else None
        if k == DIFFUSE or (k in (METAL, EMISSIVE) and kind(inp(i, 1)) == VALUE_CONSTANT) or \
           (k == GLASS and kind(inp(i, 1)) == VALUE_CONSTANT and kind(inp(i, 2)) == VALUE_CONSTANT):
            return None if c is None else (FLAT_KIND[k], c)
        if k == PLASTIC and kind(inp(i, 1)) == COLOR_CONSTANT and kind(inp(i, 2)) == DIFFUSE:
            c = colour(inp(inp(i, 2), 0))
            return None if c is None else (FLAT_KIND[k], c)
        return None

    out = []
    for root in mats["bsdf"]:
        root, fl = int(root), 0
        if kind(root) == MIX:
            t, a = inp(root, 0), inp(root, 2)
            if not (kind(t) == TRANSPARENT and kind(inp(t, 0)) == COLOR_CONSTANT and kind(a) == VALUE_ALPHA and colour(inp(a, 0)) is not None):
                out.append((0, 0))
                continue
            fl = WRAPPED | (ALPHA_IMG if colour(inp(a, 0)) else 0)
            root = inp(root, 1)
        r = leaf(root)
        out.append((0, 0) if r is None else (r[0], fl | r[1]))
    return np.array([k for k, _ in out], np.uint32), np.array([fl for _, fl in out], np.uint32)


CLASS_SCENES = GOLDEN_FLAT + ["hdr", "scene", "refraction", "venus", "alphanode", "fence", "glowmetal", "statues", "uvsphere",
                              "syn_ties", "syn_materials", "syn_single", "syn_onetri", "syn_deep", "syn_noalpha", "syn_shading", "syn_wrap"]


@pytest.mark.parametrize("name", CLASS_SCENES)
def test_flat_classification(name, scenes, flat_scenes):
    if name not in flat_scenes:
        pytest.skip(f"{name}: bundled scenes need scenes/_built or oracle/_ref/input")
    path = flat_scenes[name]
    kinds, flags = device_classes(path)
    ek, ef = expected_classes(path)
    assert np.array_equal(kinds, ek) and np.array_equal(flags * (kinds != 0), ef), (name, kinds, flags, ek, ef)
    flat = kinds != 0
    print(f"{name}: {flat.sum()} flat, {(~flat).sum()} generic materials")
    if name == "hdr":                     # every legacy material is flat, the gridplane's image-backed wrapper too
        assert flat.all() and (flags == WRAPPED | ALPHA_IMG | COL_IMG).any()
    if name in ("hdr", "venus", "refraction", "scene", "syn_materials"):
        assert flat.all() and (flags & WRAPPED).all()
    if name in ("syn_deep", "syn_noalpha"):
        assert not flat.any()
    if name == "syn_shading":
        L, f = _load(path)
        sm = _view(f.spheres, f.sphere_count, SPHERE_DTYPE)["material"].copy()
        L.crscene_free(C.byref(f))
        assert len(sm) == len(SHADING_SPHERES)
        generic = [2, 9, 10, 11, 12, 13] + list(range(14, len(SHADING_SPHERES)))   # image roughness, mix, add, checker, blackbody
        flat_ones = [0, 1, 3, 4, 5, 7, 8]                                           # image / constant diffuse, glass
        assert not flat[sm[generic]].any() and flat[sm[flat_ones]].all()
        assert (kinds[sm[[3, 4, 5]]] == FLAT_KIND[GLASS]).all() and (flags[sm[[0, 1]]] & COL_IMG).all()
    if name == "syn_wrap":
        assert flat.any() and not flat.all()


# ------------------------------------------------------------------------------------------------ scenes
ALPHA_BYTE = 77                           # the alpha of syn_wrap's one-texel texture: 77/255, strictly inside (0, 1)


def _write_wrap(out):
    """g_legacy with a one-texel RGBA texture (alpha 77/255) and its materials dealt round-robin over: the wrapper over a diffuse
    whose colour is that image (nearest texel; the same image node feeds the alpha, as the loader builds it), the same with bilinear
    filtering, the wrapper with a constant alpha 0.5 over a rough metal, the wrapper over a plastic over that image, and a generic
    ADD — flat and generic materials in one bounce."""
    L = crgpu.lib()
    L.crscene_save.argtypes = [C.POINTER(crgpu.FlatScene), C.c_char_p]
    f = crgpu.FlatScene()
    assert L.crscene_load(C.byref(f), os.path.join(GOLDEN, "g_legacy.crscene").encode()) == 0
    nodes = list(_view(f.nodes, f.node_count, NODE_DTYPE).copy())
    texs = _view(f.textures, f.texture_count, TEX_DTYPE).copy()
    data = np.frombuffer((C.c_uint8 * f.texdata_bytes).from_address(f.texdata), np.uint8) if f.texdata_bytes else np.zeros(0, np.uint8)
    off = (len(data) + 15) & ~15
    newdata = np.zeros(off + 16, np.uint8)
    newdata[:len(data)] = data
    newdata[off:off + 4] = (200, 100, 50, ALPHA_BYTE)
    t = np.zeros(1, TEX_DTYPE)
    t["width"], t["height"], t["channels"], t["is_float"], t["has_alpha"], t["data_offset"] = 1, 1, 4, 0, 1, off
    texs = np.concatenate([texs, t])
    tex = len(texs) - 1

    def add(kind, ins=(-1, -1, -1), fs=(), tex=-1, options=0):
        n = np.zeros((), NODE_DTYPE)
        n["kind"], n["in"], n["tex"], n["options"] = kind, list(ins) + [-1] * (3 - len(ins)), tex, options
        n["f"][:len(fs)] = fs
        nodes.append(n)
        return len(nodes) - 1
    white = add(COLOR_CONSTANT, fs=(1, 1, 1, 1))

    def wrap(base, alpha_colour):
        return add(MIX, (add(TRANSPARENT, (white,)), base, add(VALUE_ALPHA, (alpha_colour,))))
    img_n = add(COLOR_IMAGE, tex=tex, options=CRS_IMG_NO_BILINEAR)
    img_b = add(COLOR_IMAGE, tex=tex)
    grey = add(COLOR_CONSTANT, fs=(0.7, 0.7, 0.7, 0.5))
    graphs = [wrap(add(DIFFUSE, (img_n,)), img_n),
              wrap(add(DIFFUSE, (img_b,)), img_b),
              wrap(add(METAL, (grey, add(VALUE_CONSTANT, fs=(0.25,)))), grey),
              wrap(add(PLASTIC, (img_n, add(COLOR_CONSTANT, fs=(0.1, 0.2, 0.3, 1)), add(DIFFUSE, (img_n,)))), img_n),
              add(ADD, (add(DIFFUSE, (grey,)), add(METAL, (img_b, add(VALUE_CONSTANT, fs=(0.0,))))))]
    mats = _view(f.materials, f.material_count, MAT_DTYPE).copy()
    mats["bsdf"] = [graphs[i % len(graphs)] for i in range(f.material_count)]
    mats["IOR"] = 1.45
    arr = np.array(nodes, NODE_DTYPE)
    keep = f.nodes, f.node_count, f.materials, f.textures, f.texture_count, f.texdata, f.texdata_bytes
    f.nodes, f.node_count, f.materials = arr.ctypes.data, len(arr), mats.ctypes.data
    f.textures, f.texture_count, f.texdata, f.texdata_bytes = texs.ctypes.data, len(texs), newdata.ctypes.data, len(newdata)
    rc = L.crscene_save(C.byref(f), out.encode())
    f.nodes, f.node_count, f.materials, f.textures, f.texture_count, f.texdata, f.texdata_bytes = keep
    L.crscene_free(C.byref(f))
    assert rc == 0
    return out


@pytest.fixture(scope="module")
def flat_scenes(scenes, tmp_path_factory):
    out = dict(scenes)
    out["syn_wrap"] = _write_wrap(str(tmp_path_factory.mktemp("flat") / "syn_wrap.crscene"))
    return out


# ------------------------------------------------------------------------------------------------ path states (GPU)
def same_results(a, b, what):
    """two device runs of the same states: the same record, survivors, next states and L, bit for bit"""
    for f in ("inst", "poly", "key"):
        assert np.array_equal(a["rec"][f], b["rec"][f]), f"{what}: record {f}"
    assert same_bits(a["rec"]["t"], b["rec"]["t"]).all(), f"{what}: record t"
    assert np.array_equal(a["alive"], b["alive"]), f"{what}: alive"
    live = a["alive"] != 0
    for f in ("o", "d", "weight"):
        assert same_bits(a["next"][f][live], b["next"][f][live]).all(), f"{what}: next {f}"
    for f in ("rng", "has_l"):
        assert np.array_equal(a["next"][f][live], b["next"][f][live]), f"{what}: next {f}"
    with_l = ~live | (a["next"]["has_l"] != 0)
    assert same_bits(a["next"]["L"][with_l], b["next"]["L"][with_l]).all(), f"{what}: L"


def both_paths(g, o, st, tally, depth, md, what, exp, **kn):
    """the flat launch and the interpreter alone, each against the oracle and against each other"""
    out = []
    for go in (0, 1):
        res, perm2, surv, _ = g.shade_rays(st, depth, md, generic_only=go, **kn)
        check_step(o, res, perm2, surv, exp, tally, f"{what} generic_only={go}", kn.get("dirmode", 0))
        out.append(res)
    same_results(out[0], out[1], what)


PATH_SCENES = GOLDEN_FLAT + ["hdr", "scene", "refraction", "venus", "glowmetal", "uvsphere", "syn_materials", "syn_shading", "syn_deep",
                             "syn_noalpha", "syn_wrap"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", PATH_SCENES)
def test_flat_launch_path_states(name, flat_scenes):
    """Every bounce of the paths of a block of pixels, in sort modes 0 and 4, with the hit kernels at 2 blocks per SM; at the first
    bounces, at depth 4 and at the last bounce also at 3 and 4 blocks per SM and with the L2 prefetch."""
    if name not in flat_scenes:
        pytest.skip(f"{name}: bundled scenes need scenes/_built or oracle/_ref/input")
    o, _ = open_oracle(name, flat_scenes[name])
    g = open_gpu(name, flat_scenes[name])
    B = o.s.prefs.bounces
    full = {0, 1, 4, B - 1}
    tally = Tally(f"flat launch, {name}")
    for depth, st in sorted(path_states(o).items()):
        if depth > 40 and depth not in full:
            continue
        exp = o.path_step(st, depth, B)
        variants = [dict(dirmode=0), dict(dirmode=4)]
        if depth in full:
            variants += [dict(minb=3), dict(minb=4, prefetch=1), dict(minb=4, dirmode=4)]
        for kn in variants:
            both_paths(g, o, st, tally, depth, B, f"{name} depth {depth} {kn}", exp, **kn)
    tally.check()
    g.close()
    o.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["hdr", "g_legacy", "syn_shading", "syn_wrap"])
def test_flat_launch_adversarial_states(name, flat_scenes):
    """the adversarial states of the interpreter's tests (special weights, poisoned L, draws of exactly 0, 0.5 and 1)"""
    from test_gpu_shade import adversarial
    if name not in flat_scenes:
        pytest.skip(f"{name}: bundled scenes need scenes/_built or oracle/_ref/input")
    o, _ = open_oracle(name, flat_scenes[name])
    g = open_gpu(name, flat_scenes[name])
    st = np.concatenate(list(path_states(o, block=(16, 16)).values()))
    rng = np.random.default_rng(sum(map(ord, name)) + 1)
    adv = adversarial(o, st, rng, 0)
    for u in (1 << 31,):                  # first, second and third draws of exactly 0.5
        for k in (1, 2, 3):
            s = st[rng.choice(len(st), min(len(st), 64), replace=False)].copy()
            s["rng"] = np.array([state_with_draw(u, k, rng) for _ in range(len(s))], np.uint64)
            adv = np.concatenate([adv, s])
    tally = Tally(f"flat launch adversarial, {name}")
    B = max(o.s.prefs.bounces, 1)
    for depth, md in ((0, B), (4, max(B, 8)), (B - 1, B)):
        exp = o.path_step(adv, depth, md)
        for kn in (dict(), dict(dirmode=4)):
            both_paths(g, o, adv, tally, depth, md, f"{name} adversarial depth {depth}/{md} {kn}", exp, **kn)
    tally.check()
    g.close()
    o.close()


@pytest.mark.gpu
def test_flat_launch_aimed_states(flat_scenes):
    """the aimed states of syn_shading: poles, seams, back faces, total internal reflection, quad vertices and edges"""
    from test_gpu_shade import aimed_states
    name = "syn_shading"
    o = O.OracleScene(flat_scenes[name])
    g = crgpu.GpuScene(flat_scenes[name])
    st = aimed_states(np.random.default_rng(23))
    B = o.s.prefs.bounces
    tally = Tally("flat launch aimed states")
    for depth in (0, 4, B - 1):
        exp = o.path_step(st, depth, B)
        for kn in (dict(), dict(dirmode=4), dict(minb=4)):
            both_paths(g, o, st, tally, depth, B, f"{name} aimed depth {depth} {kn}", exp, **kn)
    tally.check()
    g.close()
    o.close()


@pytest.mark.gpu
def test_wrapper_alpha_draw_edges(flat_scenes):
    """syn_wrap's hits with RNG states whose first draw (the wrapper's) is exactly the image alpha 77/255, and just below and above:
    draw > alpha takes the transparent branch, so the draw equal to the alpha takes the leaf."""
    name = "syn_wrap"
    o = O.OracleScene(flat_scenes[name])
    g = crgpu.GpuScene(flat_scenes[name])
    st = np.concatenate(list(path_states(o, block=(24, 24)).values()))
    hits = o.path_step(st, 0)["rec"]["inst"] >= 0
    base = st[hits][:2048]
    assert len(base) >= 256
    alpha = np.float32(ALPHA_BYTE) / np.float32(255)
    u = int(float(alpha) * 2.0 ** 32)
    assert np.float32(2.3283064365386963e-10) * np.float32(u) == alpha        # the draw of u is the alpha itself
    rng = np.random.default_rng(5)
    states = []
    for uu in (u, u - 512, u + 512, u - 1, u + 1):
        s = base.copy()
        s["rng"] = np.array([state_with_draw(uu, 1, rng) for _ in range(len(s))], np.uint64)
        states.append(s)
    states = np.concatenate(states)
    tally = Tally("wrapper alpha draws")
    B = o.s.prefs.bounces
    for depth in (0, 4, B - 1):
        exp = o.path_step(states, depth, B)
        for kn in (dict(), dict(dirmode=4), dict(minb=3)):
            both_paths(g, o, states, tally, depth, B, f"{name} alpha draws depth {depth} {kn}", exp, **kn)
    tally.check()
    g.close()
    o.close()


@pytest.mark.gpu
def test_generic_only_frames_are_bit_identical(flat_scenes):
    """CRGPU_SHADE_GENERIC_ONLY=1 (every hit through the interpreter, buckets in key order) renders the default frame bit for bit,
    and so does the flat kernel at 3 and 4 blocks per SM"""
    jobs = [[n, flat_scenes[n], 0, 0, 0, 0, 0] for n in ("g_nodes", "g_legacy", "syn_materials", "syn_shading", "syn_wrap")]
    if "hdr" in flat_scenes:
        jobs.append(["hdr", flat_scenes["hdr"], 240, 135, 16, 32, 240 * 135 * 4])
    if "venus" in flat_scenes:
        jobs.append(["venus", flat_scenes["venus"], 100, 160, 16, 25, 0])
    base = _frames({}, jobs)
    bad = []
    for env in ({"CRGPU_SHADE_GENERIC_ONLY": "1"}, {"CRGPU_SHADE_FLAT_MINB": "3"}, {"CRGPU_SHADE_FLAT_MINB": "4"},
                {"CRGPU_SHADE_GENERIC_ONLY": "1", "CRGPU_TRACE_SORT": "4"}):
        got = _frames(env, jobs)
        bad += [(env, k) for k in base if got[k] != base[k]]
    assert not bad, bad
