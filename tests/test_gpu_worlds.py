"""Seeded random worlds through every comparison the suite has: loader and oracle against the reference, K2 ray by ray, K3 and the
tail kernel state by state, whole frames, tile sets, pass splits and scene edits against the oracle in device semantics.

The worlds are the loader fuzz's (test_loader._fuzz_scene, and a share of _odd_scene's wrong-typed, defaulted and degenerate
inputs), re-placed by a transform generator of their own: mirrors on one, two and three axes, anisotropic scales up to 1:1000,
uniform scales of 1e-3 and 1e3, rotations by multiples of 90 degrees (the loader's cosf / sinf of the fp32 angle leave entries
of about 4e-8 where a real quarter turn has 0; sign-flip scales give the exact 0, -0 and +-1 entries of a half turn), odd angles
and compositions about all three axes, and one mesh and one sphere each instanced at 1e-3 and at 1e3 (the last instance sets
the object's ray offset).  Every mesh has texture coordinates on all of its faces or on none, as the device upload requires.
Images are 24-96 pixels a side, 1-8 samples and 0-40 bounces, so the oracle's CPU time stays small.

world(seed, d, variant=True) draws the same objects and instance counts with other instance transforms and another camera:
the target of the edit tests, which take a world to its variant with crgpu_scene_set_camera / crgpu_scene_set_instances.

CPU: the generator's determinism and coverage, the device's refusals (only node graphs nested deeper than the interpreters
take, and ADD nodes nested deeper than its stack, may be refused), and every world's loader export and oracle frame against the
strict reference bit for bit.  GPU: everything else.
"""
import contextlib
import ctypes as C
import json
import os
import random
import re
import subprocess

import numpy as np
import pytest

import crgpu
import crscene
import oracle_lib as O
from conftest import SUMMARY_LINES
from test_gpu_scene_edit import Loaded, assert_same_as_fresh, edit, full, ray_set
from test_gpu_shade import FLAG_SHARE, LAUNCH, TAIL_FROM, TAIL_MAX, Tally, path_states, run_step
from test_gpu_trace import VARIANTS, _flat_arrays, _flatten, _name, adversarial_rays, check_counters, check_records
from test_loader import REF, _fuzz_scene, _odd_scene, _write_obj, assert_same_scene, load_crscene
from test_oracle import same_bits

SEEDS = range(48)
MIN_RENDERED = 40
# the only reasons crgpu_prepare may give for a world the loader accepts (crgpu_api.cu check_bsdf)
REFUSAL = re.compile(r"(color|value) node \d+ nests deeper than \d+|ADD nodes nest deeper than \d+")


# ------------------------------------------------------------------------------------------------ generator
def _scale(x, y, z):
    return {"type": "scale", "X": x, "Y": y, "Z": z}


def _rotation(rng, exact):
    axis = rng.choice("XYZ")
    deg = rng.choice([90, 180, 270, -90]) if exact else round(rng.uniform(-180, 180), 2)
    return {"type": "rotate" + axis, "degrees": deg}


XF_KINDS = ["plain", "mirror1", "mirror2", "mirror3", "aniso", "aniso", "tiny", "huge", "quarter", "odd", "all_axes", "half_exact"]


def _instance_transforms(rng, kind=None):
    """(kind, transform list) of one instance; the loader composes translate * rotate * scale whatever the list order"""
    kind = kind or rng.choice(XF_KINDS)
    m = lambda: round(rng.uniform(0.4, 1.6), 3)
    out = []
    if kind.startswith("mirror"):
        k = int(kind[-1])
        neg = set(rng.sample(range(3), k))
        s = [(-1 if a in neg else 1) * m() for a in range(3)]
        out.append({"type": "scaleUniform", "scale": -m()} if k == 3 and rng.random() < 0.3 else _scale(*s))
    elif kind == "aniso":                     # up to 1:1000 between axes
        b = round(rng.uniform(0.5, 2.0), 3)
        s = [b, b * 10 ** -rng.uniform(0, 3), b * rng.choice([1e-3, 10 ** -rng.uniform(0, 3)])]
        rng.shuffle(s)
        out.append(_scale(*[float("%.4g" % (v * rng.choice([1, 1, 1, -1]))) for v in s]))
    elif kind in ("tiny", "huge"):
        out.append({"type": "scaleUniform", "scale": 1e-3 if kind == "tiny" else 1e3})
    elif kind == "half_exact":                # a half turn as two sign flips: entries exactly +-1, +0 and -0
        a = rng.randrange(3)
        out.append(_scale(*[1 if i == a else -1 for i in range(3)]))
    if kind == "quarter" or (kind != "plain" and rng.random() < 0.4):
        out.append(_rotation(rng, True))
    if kind == "odd" or (kind != "plain" and rng.random() < 0.3):
        out.append(_rotation(rng, False))
    if kind == "all_axes":
        out += [{"type": "rotate" + a, "degrees": rng.choice([90, 180, 270, round(rng.uniform(-180, 180), 2)])} for a in "XYZ"]
    if kind == "huge":                        # far out, so that the camera stays outside it
        out.append({"type": "translate", "X": round(rng.uniform(-2000, 2000), 1), "Y": round(rng.uniform(-2000, 2000), 1),
                    "Z": round(rng.uniform(3000, 6000), 1)})
    else:
        out.append({"type": "translate", "X": round(rng.uniform(-3, 3), 3), "Y": round(rng.uniform(-2, 2), 3),
                    "Z": round(rng.uniform(-1, 4), 3)})
    return kind, out


def _consistent_texcoords(path):
    """Give every face of an OBJ with `vt` lines a texture coordinate on every vertex (the loader fuzz leaves some empty)."""
    lines = open(path).read().split("\n")
    nt = sum(ln.startswith("vt ") for ln in lines)
    if not nt:
        return
    def fill(tok):
        v, t, n = tok.split("/")
        return "%s/%s/%s" % (v, t or str(int(v) % nt + 1), n)
    out = [("f " + " ".join(fill(t) for t in ln.split()[1:])) if ln.startswith("f ") else ln for ln in lines]
    open(path, "w").write("\n".join(out))


def world(seed, d, variant=False, mirrors=True):
    """Write world `seed` (JSON + OBJ/MTL + PNG/HDR) into d and return its JSON document.  The objects, materials, images and
    instance counts depend on the seed alone; variant=True redraws the instance transforms and the camera.  mirrors=False gives
    the world's mirror-free twin: every scale factor made positive, nothing else changed."""
    os.makedirs(d, exist_ok=True)
    rng = random.Random(5000 + seed)
    odd = seed % 4 == 3
    sc = _odd_scene(rng, d) if odd else _fuzz_scene(rng, d)
    scene = sc["scene"]
    for m in scene.get("meshes", []):
        _consistent_texcoords(os.path.join(d, m["fileName"]))
        mtl = os.path.join(d, m["fileName"][:-4] + ".mtl")
        if isinstance(m.get("material"), list) and os.path.exists(mtl):
            # a list shorter than the MTL leaves materials without a graph: a NULL bsdf the reference dereferences when a ray
            # hits one, and the device refuses the scene; here every material gets one
            n = open(mtl).read().count("newmtl ")
            m["material"] = [m["material"][k % len(m["material"])] for k in range(max(n, len(m["material"])))]
    prims = scene["primitives"]
    if not odd and rng.random() < 0.3:
        prims.append({"type": "sphere", "radius": rng.choice([0, -1.0]), "bsdf": "glass", "color": [0.9, 0.9, 1.0],
                      "instances": [{} for _ in range(rng.randrange(1, 3))]})
    mixed = []
    if rng.random() < 0.5:                    # one sphere and one mesh, each at 1e-3 and at 1e3
        mixed.append({"type": "sphere", "radius": round(rng.uniform(0.2, 1.0), 3), "bsdf": rng.choice(["glass", "metal", "lambertian"]),
                      "color": [0.8, 0.7, 0.6], "instances": [{}, {}]})
        prims.append(mixed[-1])
        _write_obj(rng, os.path.join(d, "mixed.obj"), None, False, rng.random() < 0.5, [])
        mixed.append({"fileName": "mixed.obj", "bsdf": "plastic", "instances": [{}, {}]})
        scene.setdefault("meshes", []).append(mixed[-1])
    if not any(p.get("instances") for p in prims) and not any(m.get("instances") for m in scene.get("meshes", [])):
        prims.append({"type": "sphere", "radius": 1, "instances": [{}], "color": [1, 0, 0], "bsdf": "metal"})
    ren = {k: v for k, v in sc.get("renderer", {}).items() if k.lower() not in ("width", "height", "samples", "bounces")}
    ren.update(width=rng.randrange(24, 97), height=rng.randrange(24, 97), samples=rng.randrange(1, 9), bounces=rng.randrange(0, 41))
    sc["renderer"] = ren

    trng = random.Random(9000 + 2 * seed + int(variant))
    objects = list(prims) + list(scene.get("meshes", []))
    for ob in objects:
        for inst in ob.get("instances", []):
            inst["transforms"] = _instance_transforms(trng)[1]
    order = (seed // 2 + int(variant)) % 2            # the variant swaps which of the two instances comes last
    for ob, o in zip(mixed, (order, 1 - order)):
        for inst, k in zip(ob["instances"], ("tiny", "huge") if o == 0 else ("huge", "tiny")):
            inst["transforms"] = _instance_transforms(trng, k)[1]
    if not mirrors:
        for ob in objects:
            for inst in ob.get("instances", []):
                for t in inst["transforms"]:
                    for k in ("X", "Y", "Z", "scale"):
                        if t["type"].startswith("scale") and k in t:
                            t[k] = abs(t[k])
    cam = sc.setdefault("camera", {})
    cam["transforms"] = [{"type": "rotateX", "degrees": round(trng.uniform(-12, 12), 2)},
                         {"type": "rotateY", "degrees": round(trng.uniform(-15, 15), 2)},
                         {"type": "translate", "X": round(trng.uniform(-1, 1), 3), "Y": round(trng.uniform(-1, 1), 3),
                          "Z": round(-trng.uniform(6, 12), 3)}]
    open(os.path.join(d, "world.json"), "w").write(json.dumps(sc, indent=1))
    return sc


@contextlib.contextmanager
def _in_dir(d):
    """node-graph texture paths resolve against the working directory, as in the reference"""
    here = os.getcwd()
    os.chdir(d)
    try:
        yield
    finally:
        os.chdir(here)


class World:
    """A generated world: its directory, JSON document and .crscene, and why the device refuses it (None: it does not)."""

    def __init__(self, root, seed, variant=False, mirrors=True):
        self.seed, self.variant = seed, variant
        self.dir = os.path.join(root, "w%d%s%s" % (seed, "v" if variant else "", "" if mirrors else "m"))
        self.doc = world(seed, self.dir, variant, mirrors)
        self.json = os.path.join(self.dir, "world.json")
        self.path = os.path.join(self.dir, "world.crscene")
        with _in_dir(self.dir):
            _flatten(self.json, self.path)
        self.refusal = prepare_error(self.path)
        r = self.doc["renderer"]
        self.cfg = (r["width"], r["height"], r["samples"], r["bounces"])

    def loaded(self):
        """test_gpu_scene_edit.Loaded of this world at its own size"""
        return Loaded(self.doc, *self.cfg, cwd=self.dir, asset_path=self.dir)


def prepare_error(path):
    """crgpu_last_error of crgpu_prepare on a flat scene, or None when the device takes it (no device needed)"""
    L = crgpu.lib()
    L.crgpu_prepare.argtypes = [C.POINTER(crgpu.FlatScene), C.POINTER(C.c_void_p)]
    L.crgpu_prepared_free.argtypes = [C.c_void_p]
    f = crgpu.FlatScene()
    assert L.crscene_load(C.byref(f), path.encode()) == 0, path
    p = C.c_void_p()
    rc = L.crgpu_prepare(C.byref(f), C.byref(p))
    L.crscene_free(C.byref(f))
    if rc == 0:
        L.crgpu_prepared_free(p)
        return None
    return L.crgpu_last_error().decode(errors="replace")


_WORLDS = {}


@pytest.fixture(scope="module")
def worlds(tmp_path_factory):
    """(seed, variant, mirrors) -> World, built on first use"""
    root = str(tmp_path_factory.mktemp("worlds"))

    def get(seed, variant=False, mirrors=True):
        if (seed, variant, mirrors) not in _WORLDS:
            _WORLDS[(seed, variant, mirrors)] = World(root, seed, variant, mirrors)
        return _WORLDS[(seed, variant, mirrors)]
    yield get
    _WORLDS.clear()


def accepted(worlds, seed):
    """the world of a GPU test; the test skips without a CUDA device, and for a world the device refuses"""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    w = worlds(seed)
    if w.refusal:
        pytest.skip(f"world {seed} is refused by the device: {w.refusal}")
    return w


# ------------------------------------------------------------------------------------------------ generator (CPU)
def _mat(inst):
    return inst["A"].reshape(4, 4)[:3, :3].astype(np.float64)


def test_world_generator(worlds, tmp_path):
    """Every seed loads into a .crscene; a second run writes the same bytes; the variant keeps objects and instance counts and
    moves the instances; the worlds reach every transform class; texture coordinates are all-or-none per mesh; the world box
    stays far inside fp32's range; the device refuses only for the documented reasons, and at least 40 worlds reach it."""
    seen = dict(det_neg=0, two_flips=0, aniso_1000=0, tiny=0, huge=0, exact_half=0, quarter=0, radius_0=0, radius_neg=0,
                mixed_small_last=0, mixed_big_last=0, smooth_mesh=0, flat_mesh=0, uv_mesh=0, odd_tiles=0)
    refused = {}
    for seed in SEEDS:
        w = worlds(seed)
        d = str(tmp_path / ("again%d" % seed))
        assert json.dumps(world(seed, d)).replace(d, w.dir) == json.dumps(w.doc), seed
        for name in sorted(os.listdir(d)):
            if name != "world.json":
                assert open(os.path.join(d, name), "rb").read() == open(os.path.join(w.dir, name), "rb").read(), (seed, name)
        W, H, spp, b = w.cfg
        assert 24 <= W <= 96 and 24 <= H <= 96 and 1 <= spp <= 8 and 0 <= b <= 40
        f = crgpu.FlatScene()
        assert crgpu.lib().crscene_load(C.byref(f), w.path.encode()) == 0
        A = crscene.arrays(f)
        v = worlds(seed, True)
        fv = crgpu.FlatScene()
        assert crgpu.lib().crscene_load(C.byref(fv), v.path.encode()) == 0
        B = crscene.arrays(fv)
        for key in ("polys", "vertices", "normals", "texcoords", "materials", "nodes", "textures", "texdata"):
            assert A[key].tobytes() == B[key].tobytes(), (seed, key)
        assert np.array_equal(A["instances"][["kind", "object"]], B["instances"][["kind", "object"]]), seed
        assert A["spheres"]["radius"].tobytes() == B["spheres"]["radius"].tobytes()
        assert A["instances"]["A"].tobytes() != B["instances"]["A"].tobytes(), seed
        assert json.dumps(w.doc["renderer"]) == json.dumps(v.doc["renderer"]) and w.doc["camera"] != v.doc["camera"]
        for inst in A["instances"]:
            M = _mat(inst)
            sv = np.linalg.svd(M, compute_uv=False)
            seen["det_neg"] += np.linalg.det(M) < 0
            seen["aniso_1000"] += sv[0] / sv[-1] >= 500
            seen["tiny"] += np.allclose(sv, 1e-3, rtol=1e-5)
            seen["huge"] += np.allclose(sv, 1e3, rtol=1e-5)
            exact = np.isin(M, (-1.0, 0.0, 1.0)).all()
            seen["exact_half"] += exact and np.signbit(M).any() and np.linalg.det(M) > 0
            seen["two_flips"] += exact and (np.diag(M) < 0).sum() == 2
            seen["quarter"] += ((M != 0) & (np.abs(M) < 1e-6 * np.abs(M).max())).any()     # cosf(fp32 pi / 2) and the like
        rad = A["spheres"]["radius"]
        obj_inst = A["instances"][A["instances"]["kind"] == 0]["object"]
        seen["radius_0"] += int((rad[obj_inst] == 0).sum())
        seen["radius_neg"] += int((rad[obj_inst] < 0).sum())
        if any(m["fileName"] == "mixed.obj" for m in w.doc["scene"].get("meshes", [])):
            last = [i for i in A["instances"] if i["kind"] == 0 and rad[i["object"]] == w.doc["scene"]["primitives"][-1]["radius"]]
            big = np.linalg.svd(_mat(last[-1]), compute_uv=False)[0] > 1
            seen["mixed_big_last" if big else "mixed_small_last"] += 1
        for m in A["meshes"]:
            p = A["polys"][m["poly_offset"]:m["poly_offset"] + m["poly_count"]]
            with_t = p["t"] >= 0
            assert with_t.all() or not with_t.any(), (seed, "a mesh mixes faces with and without texture coordinates")
            seen["uv_mesh"] += bool(with_t.all() and m["texcoord_count"])
            seen["smooth_mesh"] += bool(p["has_normals"].any())
            seen["flat_mesh"] += bool(not p["has_normals"].all())
        seen["odd_tiles"] += W % f.prefs.tile_width != 0 or H % f.prefs.tile_height != 0
        if f.top_bvh < f.bvh_count and A["bvhs"][f.top_bvh]["node_count"]:
            box = A["bvh_nodes"][A["bvhs"][f.top_bvh]["node_offset"]]["bounds"]
            assert np.isfinite(box).all() and np.abs(box).max() < 1e5, (seed, box)
        crgpu.lib().crscene_free(C.byref(f))
        crgpu.lib().crscene_free(C.byref(fv))
        if w.refusal:
            assert REFUSAL.search(w.refusal), (seed, w.refusal)
            why = REFUSAL.search(w.refusal).group(0).split()[0]
            refused[why] = refused.get(why, 0) + 1
    rendered = len(SEEDS) - sum(refused.values())
    line = (f"random worlds: {len(SEEDS)} seeds, {rendered} reach the device, {sum(refused.values())} refused "
            f"({', '.join(f'{k} nesting {v}' for k, v in sorted(refused.items())) or 'none'}); instances: "
            + " ".join(f"{k} {int(v)}" for k, v in seen.items()))
    print(line)
    SUMMARY_LINES.append(line)
    assert rendered >= MIN_RENDERED, line
    for k, v in seen.items():
        assert v >= 2, (k, line)


# ------------------------------------------------------------------------------------------------ reference anchor (CPU)
def _ref(w, *args, timeout=120):
    return subprocess.run([REF, args[0], "world.json", *args[1:]], cwd=w.dir, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                          text=True, errors="replace", timeout=timeout)


def mirrored(path):
    """whether some instance of a flat scene has a transform of negative determinant"""
    f = crgpu.FlatScene()
    assert crgpu.lib().crscene_load(C.byref(f), path.encode()) == 0
    dets = [np.linalg.det(_mat(i)) for i in crscene.arrays(f)["instances"]]
    crgpu.lib().crscene_free(C.byref(f))
    return min(dets, default=1.0) < 0


@pytest.mark.parametrize("seed", SEEDS)
def test_world_matches_reference(seed, worlds):
    """The loader's flat scene is the strict reference's export, and the oracle's semantics-0 frame is the reference's frame,
    bit for bit: what the GPU is compared with below is tied to the reference on every world.  The reference refuses a transform
    whose determinant is not positive (inverseMatrix, transforms.c:264-267: "No inverse for given transform!", then exits), so a
    mirrored world must be refused there and its mirror-free twin is compared instead; the loader, the oracle and the device
    take mirrors as the matrices they are."""
    if not os.path.exists(REF):
        pytest.skip("oracle/_ref/cray_ref_strict is only built where /root/reference exists")
    w = worlds(seed)
    if mirrored(w.path):
        r = _ref(w, "export", "0", "0", "0", "0", "ref.crscene")
        assert r.returncode != 0 and "No inverse for given transform" in r.stdout, r.stdout[-2000:]
        w = worlds(seed, mirrors=False)
        assert not mirrored(w.path)
    r = _ref(w, "export", "0", "0", "0", "0", "ref.crscene")
    assert r.returncode == 0, r.stdout[-2000:]
    mine, ref = load_crscene(w.path), load_crscene(os.path.join(w.dir, "ref.crscene"))
    assert_same_scene(mine, ref)
    crgpu.lib().crscene_free(C.byref(mine))
    crgpu.lib().crscene_free(C.byref(ref))
    r = _ref(w, "render", "0", "0", "0", "0", str(os.cpu_count() or 1), "0", "0", "ref.f32", timeout=600)
    assert r.returncode == 0, r.stdout[-2000:]
    o = O.OracleScene(w.path)
    img = o.render(threads=os.cpu_count())
    o.close()
    want = np.fromfile(os.path.join(w.dir, "ref.f32"), dtype=np.float32).reshape(img.shape)
    differ = (~same_bits(img, want)).any(axis=2)
    assert not differ.any(), f"world {seed}: {int(differ.sum())} pixels differ from the reference, first rows {np.nonzero(differ)[0][:5]}"


# ------------------------------------------------------------------------------------------------ GPU
# what the GPU tests compared, over all worlds: the per-test near-tie bound is checked in each test, the totals are reported last
TOTALS = {k: Tally(f"random worlds, {k}") for k in ("K2 rays", "K3 states", "aimed states", "frame samples")}
# K3 options that rotate with the seed at depths 0, 1, 4 and B - 1
ROTATE = LAUNCH + [dict(complete_interpreter=1)] + [dict(dirmode=m) for m in (1, 2, 3, 4)]


def _bounded(tally):
    assert tally.flagged <= max(1, tally.states * FLAG_SHARE), f"{tally.what}: {tally.flagged} of {tally.states} flagged"
    TOTALS[tally.what.split(", ")[1]].add(tally.states, tally.flagged)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", SEEDS)
def test_world_trace_records(seed, worlds):
    """K2 on the paths of a pixel block and on test_gpu_trace.adversarial_rays: records bit for bit against the oracle in device
    semantics in the default launch, the instrumented launch (P/T/S/I counts exact) and one more variant rotating with the seed."""
    w = accepted(worlds, seed)
    o = O.OracleScene(w.path)
    bw, bh = min(o.W, 48), min(o.H, 32)
    x0, y0 = (o.W - bw) // 2, (o.H - bh) // 2
    p = o.path_rays(x0, y0, x0 + bw, y0 + bh, passes=(0, min(2, o.s.prefs.sample_count)))
    a, _, _ = adversarial_rays(o, np.random.default_rng(seed))
    rays = np.concatenate([p, a]).astype(np.float32)
    r1, c1 = o.closest_hit(rays, O.SEM_DEVICE)
    o.close()
    g = crgpu.GpuScene(w.path)
    extra = [v for v in VARIANTS if v and v != dict(count=1)]
    for kn in (dict(), dict(count=1), extra[seed % len(extra)]):
        rec, perm, misses, st = g.trace_rays(rays, **kn)
        check_records(g, rec, perm, misses, r1, f"world {seed} {_name(kn)}")
        if kn.get("count"):
            check_counters(st, c1, len(rays), f"world {seed} {_name(kn)}")
    g.close()
    TOTALS["K2 rays"].add(len(rays), 0)


def _sphere_instances(o):
    """(A 3x4, radius) of the sphere instances whose transform is mirrored or not a uniform scale, radius not 0"""
    f = _flat_arrays(o.s)
    rad = np.frombuffer((C.c_uint8 * (16 * o.s.sphere_count)).from_address(o.s.spheres), dtype=crscene.SPHERE)["radius"] \
        if o.s.sphere_count else np.zeros(0, np.float32)
    out = []
    for inst in f["inst"]:
        if inst["kind"] != 0 or rad[inst["object"]] == 0:
            continue
        M = _mat(inst)
        sv = np.linalg.svd(M, compute_uv=False)
        if np.linalg.det(M) < 0 or sv[0] > sv[-1] * (1 + 1e-3):
            out.append((inst["A"].reshape(4, 4)[:3].astype(np.float64), abs(float(rad[inst["object"]]))))
    return out


def aimed_sphere_states(o, rng, per=4, draws=4):
    """States aimed at the mirrored and anisotropic spheres, built in object space and carried out by the instance matrix: at the
    centre and grazing (0.999 r off the centre line), from outside and from inside, with `draws` RNG states each"""
    org, dirs = [], []
    for A, r in _sphere_instances(o)[:32]:
        for _ in range(per):
            u = rng.normal(size=3)
            u /= np.linalg.norm(u)
            wv = np.cross(u, rng.normal(size=3))
            wv /= np.linalg.norm(wv)
            for po in (-3 * r * u, 0.999 * r * wv - 3 * r * u, 0 * u, 0.999 * r * wv):
                org.append(A[:, :3] @ po + A[:, 3])
                dw = A[:, :3] @ u
                dirs.append(dw / np.linalg.norm(dw))
    base = np.zeros(len(org), crgpu.PATH_STATE_DTYPE)
    if not len(org):
        return base
    base["o"], base["d"], base["weight"] = np.array(org, np.float32), np.array(dirs, np.float32), 1.0
    out = []
    for _ in range(draws):
        st = base.copy()
        st["rng"] = rng.integers(0, 1 << 63, len(st), dtype=np.uint64)
        out.append(st)
    return np.concatenate(out)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", SEEDS)
def test_world_path_states(seed, worlds):
    """K3 and the tail kernel on every bounce of the paths of a pixel block: the default launch at every depth, an option rotating
    with the seed at depths 0, 1, 4 and B - 1, the tail kernel from CRG_TAIL_FROM; and states aimed at the mirrored and
    anisotropic spheres, which meet normals that point inward or are not of unit length."""
    w = accepted(worlds, seed)
    o = O.OracleScene(w.path)
    g = crgpu.GpuScene(w.path)
    B = o.s.prefs.bounces
    tally = Tally(f"world {seed}, K3 states")
    for depth, st in sorted(path_states(o).items()):
        exp = o.path_step(st, depth, B)
        variants = [dict()]
        if depth in (0, 1, 4, B - 1):
            variants.append(ROTATE[(seed + depth) % len(ROTATE)])
        for kn in variants:
            run_step(g, o, st, tally, depth, B, f"world {seed} depth {depth} {kn}", exp=exp, **kn)
        if depth == TAIL_FROM and len(st) <= TAIL_MAX:
            run_step(g, o, st, tally, depth, B, f"world {seed} tail from {depth}", tail=1, complete_interpreter=seed % 2)
    _bounded(tally)
    aimed = aimed_sphere_states(o, np.random.default_rng(seed))
    if len(aimed):
        tally = Tally(f"world {seed}, aimed states")
        md = max(B, 2)
        for depth in (0, md - 1):
            exp = o.path_step(aimed, depth, md)
            for kn in (dict(), dict(complete_interpreter=1), ROTATE[seed % len(ROTATE)]):
                run_step(g, o, aimed, tally, depth, md, f"world {seed} aimed depth {depth} {kn}", exp=exp, **kn)
        run_step(g, o, aimed, tally, TAIL_FROM, md + TAIL_FROM, f"world {seed} aimed tail", tail=1)
        _bounded(tally)
    g.close()
    o.close()


@pytest.mark.gpu
@pytest.mark.parametrize("seed", SEEDS)
def test_world_frames(seed, worlds):
    """render_frame equals the oracle's semantics-1 frame bit for bit outside pixels with a flagged sample; every third world also
    renders as the tile set of its own tile size and as that tile set split into two pass ranges, with the same bits."""
    w = accepted(worlds, seed)
    g = crgpu.GpuScene(w.path)
    g.render_frame()
    img = g.read().copy()
    o = O.OracleScene(w.path)
    ref, flagged = o.render_sem(O.SEM_DEVICE)
    tw, th, spp = o.s.prefs.tile_width, o.s.prefs.tile_height, o.s.prefs.sample_count
    o.close()
    tally = Tally(f"world {seed}, frame samples")
    tally.add(img.shape[0] * img.shape[1] * spp, flagged.sum())
    _bounded(tally)
    bad = np.nonzero((~same_bits(img, ref)).any(axis=2) & (flagged == 0))
    assert len(bad[0]) == 0, f"world {seed}: {len(bad[0])} unflagged pixels differ, first rows {bad[0][:5]} cols {bad[1][:5]}"
    if seed % 3 == 0:
        rects = [(x, y, min(x + tw, g.W), min(y + th, g.H)) for y in range(0, g.H, th) for x in range(0, g.W, tw)]
        g.clear()
        g.render_tiles(rects)
        assert g.read().tobytes() == img.tobytes(), f"world {seed}: {len(rects)} tiles of {tw}x{th}"
        if spp > 1:
            g.clear()
            g.render_tiles(rects, 0, spp // 2)
            g.render_tiles(rects, spp // 2, spp - spp // 2)
            assert g.read().tobytes() == img.tobytes(), f"world {seed}: tiles in passes [0, {spp // 2}) + [{spp // 2}, {spp})"
    g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("seed", SEEDS)
def test_world_edit_to_variant(seed, worlds):
    """A world edited with its variant's camera and instances renders and traces (records and P/T/S/I counts) as the variant
    loaded fresh, on the camera's rays and the variant's adversarial rays; editing back gives the world's own frame."""
    w = accepted(worlds, seed)
    v = worlds(seed, True)
    assert not v.refusal
    a, b = w.loaded(), v.loaded()
    assert len(a.instances) and np.array_equal(a.instances[["kind", "object"]], b.instances[["kind", "object"]])
    o = O.OracleScene(v.path)
    adv, _, _ = adversarial_rays(o, np.random.default_rng(seed), n=256)
    o.close()
    rays = np.concatenate([ray_set(b.camera, n=4096, seed=seed), adv]).astype(np.float32)
    fresh = a.upload()
    want = full(fresh)
    fresh.close()
    g = a.upload()
    try:
        edit(g, b)
        assert_same_as_fresh(g, b, rays)
        edit(g, a)
        assert full(g).tobytes() == want.tobytes(), f"world {seed}: editing back does not give the world's frame"
    finally:
        g.close()
        a.free()
        b.free()


@pytest.mark.gpu
def test_world_totals():
    """what the GPU tests above compared over all worlds, and the share of it the near-tie flag exempted"""
    if not sum(t.states for t in TOTALS.values()):
        pytest.skip("no GPU test of this file ran")
    for t in TOTALS.values():
        line = f"{t.what}: {t.flagged} of {t.states} flagged"
        print(line)
        SUMMARY_LINES.append(line)
