"""Scene loader (c-ray_b200/host/loader/, include/crloader.h) against the reference's own loader.

The loader must produce, for the same JSON + assets, the flat scene that the unmodified reference produces when its
world is flattened (oracle/ref_harness.c `export`): same instances and matrices, same hash-consed node graph, same
BVH node for node, same primitive order, same decoded textures — bit for bit, because the GPU hot path's parity with
the reference starts from identical inputs.

Three layers:
  * committed fixtures: tests/golden/*.json vs the *.crscene the strict reference exported (always run);
  * the reference's bundled scenes (hdr, venus, refraction, scene) vs scenes/_built/*.crscene (when built here);
  * differential fuzzing: random scenes written to a temp dir, loaded by both loaders (when oracle/_ref exists).
Known, documented tolerances (reference reads uninitialised memory there): malloc slack in the global vertex buffer
(slots past the parsed `v` lines), the unused bits of interior BVH nodes, and prefs.thread_count.
"""
import ctypes as C
import json
import math
import os
import random
import struct
import subprocess
import zlib

import numpy as np
import pytest

from conftest import GOLDEN, BUILT, GOLDEN_SCENES, ROOT
import crgpu
import crscene

REF = os.path.join(ROOT, "oracle", "_ref", "cray_ref_strict")
REF_INPUT = os.path.join(ROOT, "oracle", "_ref")


def load_crscene(path):
    L = crgpu.lib()
    s = crgpu.FlatScene()
    L.crscene_load.argtypes = [C.POINTER(crgpu.FlatScene), C.c_char_p]
    assert L.crscene_load(C.byref(s), os.fsencode(path)) == 0, path
    return s


def assert_same_scene(mine, ref, undefined_meshes=()):
    """Field-by-field, array-by-array equality (bitwise for floats) with the documented tolerances."""
    for name, _ in crgpu.FlatScene._fields_:
        if name in ("prefs", "camera", "owner") or name in [s[0] for s in crscene._SECTIONS]:
            continue
        if name == "bvh_node_count" and undefined_meshes:
            continue
        assert getattr(mine, name) == getattr(ref, name), name
    for name, _ in type(mine.prefs)._fields_:
        if name != "thread_count":
            assert getattr(mine.prefs, name) == getattr(ref.prefs, name), "prefs." + name
    assert bytes(mine.camera) == bytes(ref.camera), "camera"
    A, B = crscene.arrays(mine), crscene.arrays(ref)
    skip_bvh = set()
    for m in undefined_meshes:
        skip_bvh.add(int(B["meshes"][m]["bvh"]))
    if undefined_meshes:
        skip_bvh.add(int(ref.top_bvh))
    for key in A:
        a, b = A[key], B[key]
        if key == "bvhs" and skip_bvh:
            keep = [i for i in range(len(b)) if i not in skip_bvh]
            assert np.array_equal(a[keep]["prim_count"], b[keep]["prim_count"])
            continue
        if key in ("bvh_nodes", "prim_indices") and skip_bvh:
            off, cnt = ("node_offset", "node_count") if key == "bvh_nodes" else ("prim_offset", "prim_count")
            for i in range(len(B["bvhs"])):
                if i in skip_bvh:
                    continue
                sa = a[A["bvhs"][i][off]:A["bvhs"][i][off] + A["bvhs"][i][cnt]]
                sb = b[B["bvhs"][i][off]:B["bvhs"][i][off] + B["bvhs"][i][cnt]]
                _assert_array(key, sa, sb, B)
            continue
        if key == "meshes" and undefined_meshes:
            a, b = a.copy(), b.copy()
            for m in undefined_meshes:
                a[m]["ray_offset"] = b[m]["ray_offset"] = 0
        assert a.shape == b.shape, (key, a.shape, b.shape)
        _assert_array(key, a, b, B)


def _assert_array(key, a, b, B):
    assert a.shape == b.shape, (key, a.shape, b.shape)
    if key == "bvh_nodes":
        leaf = (b["count_leaf"] & crscene.LEAF_BIT) != 0
        # interior nodes: the reference never writes primCount / the top bit (bvh.c:227-228), the loader writes 0
        bc = np.where(leaf, b["count_leaf"] & (crscene.COUNT_MASK | crscene.LEAF_BIT), 0)
        assert a["bounds"].tobytes() == b["bounds"].tobytes(), "bvh bounds"
        assert np.array_equal(a["first"], b["first"]), "bvh child / first primitive"
        assert np.array_equal(a["count_leaf"], bc), "bvh leaf flag / count"
    elif key in ("vertices", "normals", "texcoords"):
        field = {"vertices": "v", "normals": "n", "texcoords": "t"}[key]
        idx = np.unique(B["polys"][field])
        idx = idx[(idx >= 0) & (idx < len(a))]
        if key == "vertices":
            # slots past a file's parsed `v` lines are malloc garbage in the reference (wavefront.c:139-141): faces that
            # reach them through the inflated negative-index base are excluded by the caller (undefined_meshes)
            bad = ~np.isfinite(b[idx]).all(axis=1)
            idx = idx[~bad]
        same = (a[idx].view(np.uint32) == b[idx].view(np.uint32)).all(axis=1)
        assert same.all() or key == "vertices" and _only_slack(a, b, idx[~same]), key
    else:
        assert a.tobytes() == b.tobytes(), key


def _only_slack(a, b, idx):
    """True when every differing vertex slot is one the loader left at zero (never parsed from a `v` line)."""
    return bool((a[idx] == 0).all())


# ------------------------------------------------------------------------------------------------ fixtures
def test_loader_exports_declared_symbols():
    import re
    text = open(os.path.join(ROOT, "include", "crloader.h")).read()
    names = sorted(set(re.findall(r"\b(crloader_\w+)\s*\(", text)))
    assert names == ["crloader_build_bvh", "crloader_last_error", "crloader_load_json", "crloader_load_json_buf", "crloader_set_bvh_builder"]
    L = C.CDLL(crscene.LOADER_PATH)
    for n in names:
        getattr(L, n)


@pytest.mark.parametrize("name", GOLDEN_SCENES)
def test_golden_scene_matches_reference_export(name, monkeypatch):
    monkeypatch.chdir(GOLDEN)            # JSON texture paths are cwd-relative in the reference (sceneloader.c:783,826)
    mine = crscene.load_json(name + ".json")
    ref = load_crscene(os.path.join(GOLDEN, name + ".crscene"))
    # g_legacy's third mesh (assets/mixed.obj) has a face "-3/-2/-1": with the reference's inflated vertex count it lands
    # on an unparsed slot, i.e. the reference builds that mesh's BVH from uninitialised memory
    undefined = (2,) if name == "g_legacy" else ()
    assert_same_scene(mine, ref, undefined)
    crscene.free(mine)


@pytest.mark.parametrize("name", ["hdr", "venus", "refraction", "scene", "alphanode", "fence", "glowmetal", "statues", "uvsphere"])
def test_bundled_scene_matches_reference_export(name, monkeypatch):
    src = os.path.join(REF_INPUT, "input", name + ".json")
    exported = os.path.join(BUILT, name + ".crscene")
    if not (os.path.exists(src) and os.path.exists(exported)):
        pytest.skip("bundled scenes are copied/exported by build() only where /root/reference exists")
    monkeypatch.chdir(REF_INPUT)
    mine = crscene.load_json(os.path.join("input", name + ".json"))
    ref = load_crscene(exported)
    assert_same_scene(mine, ref)
    crscene.free(mine)


# ------------------------------------------------------------------------------------------------ error paths
def test_loader_errors(tmp_path):
    with pytest.raises(RuntimeError, match="cannot read"):
        crscene.load_json(str(tmp_path / "nope.json"))
    bad = tmp_path / "bad.json"
    bad.write_text('{"renderer": {"width": 4,}')
    with pytest.raises(RuntimeError, match="syntax"):
        crscene.load_json(str(bad))
    nocam = tmp_path / "nocam.json"
    nocam.write_text('{"renderer": {"width": 4, "height": 4}, "scene": {}}')
    with pytest.raises(RuntimeError, match="camera"):
        crscene.load_json(str(nocam))
    (tmp_path / "tri.obj").write_text("v 0 0 0\nv 1 0 0\nv 0 1 0\nf 1 2 3\n")   # the reference segfaults on this syntax
    sc = tmp_path / "face.json"
    sc.write_text(json.dumps({"renderer": {"width": 4, "height": 4}, "camera": {},
                              "scene": {"meshes": [{"fileName": "tri.obj", "instances": [{}]}]}}))
    with pytest.raises(RuntimeError, match="v/vt/vn"):
        crscene.load_json(str(sc))


def test_mesh_without_polygons_is_rejected(tmp_path):
    """An OBJ with vertices but no faces: the loader refuses the instance, so the traversal's empty-BVH case (bvh.c:362-365,
    which resets the instance of an earlier hit) is not reachable from a scene file.  Should the loader ever accept such a
    mesh, tests/test_gpu_trace.py has to cover that case."""
    (tmp_path / "empty.obj").write_text("v 0 0 0\nv 1 0 0\nv 0 1 0\n")
    sc = tmp_path / "empty.json"
    sc.write_text(json.dumps({"renderer": {"width": 4, "height": 4}, "camera": {},
                              "scene": {"meshes": [{"fileName": "empty.obj", "instances": [{}]}]}}))
    with pytest.raises(RuntimeError, match="without polygons"):
        crscene.load_json(str(sc))


def test_loader_defaults_and_clamps(tmp_path):
    """parsePrefs / parseCamera defaults (sceneloader.c:190-208, :539-545) and clamps."""
    p = tmp_path / "min.json"
    p.write_text(json.dumps({"renderer": {"samples": -3, "bounces": -1, "tileWidth": 0, "WIDTH": 33, "height": 17,
                                          "tileOrder": "whatever"},
                             "camera": {"FOV": 400}, "scene": {}}))
    s = crscene.load_json(str(p))
    assert (s.prefs.sample_count, s.prefs.bounces, s.prefs.tile_width, s.prefs.tile_height) == (1, 1, 1, 32)
    assert (s.prefs.image_width, s.prefs.image_height, s.prefs.tile_order) == (33, 17, 3)   # keys are case-insensitive
    assert abs(s.camera.sensor_x) > 1e6                                                      # FOV clamps to 180: 2*tanf(pi/2)
    assert s.instance_count == 0 and s.bvh_count == 1 and s.node_count == 4                  # gray background + 2 values
    crscene.free(s)


# ------------------------------------------------------------------------------------------------ image decoders
def _png(w, h, ctype, depth, rows, palette=None, trns=None, filters=None):
    def chunk(tag, data):
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)
    bpp = max(1, {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}[ctype] * depth // 8)
    raw, prev = bytearray(), bytes(len(rows[0]))
    for y, row in enumerate(rows):
        f = filters[y % len(filters)] if filters else 0
        out = bytearray()
        for i, v in enumerate(row):
            a = row[i - bpp] if i >= bpp else 0
            b = prev[i]
            c = prev[i - bpp] if i >= bpp else 0
            if f == 0: pred = 0
            elif f == 1: pred = a
            elif f == 2: pred = b
            elif f == 3: pred = (a + b) // 2
            else:
                pa, pb, pc = abs(b - c), abs(a - c), abs(a + b - 2 * c)
                pred = a if pa <= pb and pa <= pc else (b if pb <= pc else c)
            out.append((v - pred) & 255)
        raw.append(f)
        raw.extend(out)
        prev = bytes(row)
    data = b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, ctype, 0, 0, 0))
    if palette: data += chunk(b"PLTE", bytes(palette))
    if trns: data += chunk(b"tRNS", bytes(trns))
    z = zlib.compress(bytes(raw), 6)
    half = len(z) // 2                                 # two IDAT chunks: the stream must be concatenated
    return data + chunk(b"IDAT", z[:half]) + chunk(b"IDAT", z[half:]) + chunk(b"IEND", b"")


def _decode(tmp_path, name, blob):
    """Decode an image through the loader by hanging it on a diffuse sphere; returns (crs_texture row, pixel bytes)."""
    (tmp_path / name).write_bytes(blob)
    sc = tmp_path / (name + ".json")
    sc.write_text(json.dumps({"renderer": {"width": 4, "height": 4}, "camera": {}, "scene": {"primitives": [
        {"type": "sphere", "radius": 1, "instances": [{}],
         "material": {"type": "diffuse", "color": {"type": "image", "path": str(tmp_path / name)}}}]}}))
    s = crscene.load_json(str(sc))
    A = crscene.arrays(s)
    assert len(A["textures"]) == 1
    t = A["textures"][0]
    n = int(t["width"]) * int(t["height"]) * int(t["channels"]) * (4 if t["is_float"] else 1)
    px = A["texdata"][int(t["data_offset"]):int(t["data_offset"]) + n].copy()
    crscene.free(s)
    return t, px


@pytest.mark.parametrize("ctype,depth", [(0, 8), (2, 8), (4, 8), (6, 8), (0, 16), (2, 16), (6, 16), (3, 8), (3, 4), (0, 1), (0, 2), (0, 4)])
def test_png_decoder(tmp_path, ctype, depth):
    rng = random.Random(ctype * 100 + depth)
    w, h = 13, 7
    chans = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}[ctype]
    palette = [rng.randrange(256) for _ in range(3 * (1 << min(depth, 4)))] if ctype == 3 else None
    maxv = (1 << depth) - 1
    samples = [[[rng.randrange(len(palette) // 3) if ctype == 3 else rng.randrange(maxv + 1) for _ in range(chans)]
                for _ in range(w)] for _ in range(h)]
    rows = []
    for y in range(h):
        flat = [v for px in samples[y] for v in px]
        if depth == 16:
            rows.append(bytes(b for v in flat for b in (v >> 8, v & 255)))
        elif depth == 8:
            rows.append(bytes(flat))
        else:
            bits, acc, n = bytearray(), 0, 0
            for v in flat:
                acc = (acc << depth) | v
                n += depth
                if n == 8:
                    bits.append(acc); acc = n = 0
            if n:
                bits.append(acc << (8 - n))
            rows.append(bytes(bits))
    t, px = _decode(tmp_path, "t.png", _png(w, h, ctype, depth, rows, palette, filters=[0, 1, 2, 3, 4]))
    assert (t["width"], t["height"], t["is_float"]) == (w, h, 0)
    if ctype == 3:
        expect = [c for y in range(h) for x in range(w) for c in palette[3 * samples[y][x][0]:3 * samples[y][x][0] + 3]]
        assert t["channels"] == 3
    else:
        assert t["channels"] == chans
        if depth == 16:
            expect = [v >> 8 for y in range(h) for x in range(w) for v in samples[y][x]]
        elif depth == 8:
            expect = [v for y in range(h) for x in range(w) for v in samples[y][x]]
        else:                                           # stb scales low bit depths to 0..255: v * (255 / maxv)
            expect = [v * (255 // maxv) for y in range(h) for x in range(w) for v in samples[y][x]]
    assert t["has_alpha"] == (1 if t["channels"] > 3 else 0)
    assert px.tolist() == expect


def test_png_palette_transparency(tmp_path):
    palette = [10, 20, 30, 40, 50, 60, 70, 80, 90]
    rows = [bytes([0, 1, 2, 1])]
    t, px = _decode(tmp_path, "p.png", _png(4, 1, 3, 8, rows, palette, trns=[0, 128]))
    assert t["channels"] == 4 and t["has_alpha"] == 1
    assert px.tolist() == [10, 20, 30, 0, 40, 50, 60, 128, 70, 80, 90, 255, 40, 50, 60, 128]


def _hdr(w, h, pix, rle):
    out = bytearray(b"#?RADIANCE\nFORMAT=32-bit_rle_rgbe\n\n" + f"-Y {h} +X {w}\n".encode())
    for y in range(h):
        row = pix[y]
        if not rle:
            for p in row: out.extend(bytes(p))
            continue
        out.extend(bytes([2, 2, w >> 8, w & 255]))
        for c in range(4):
            vals = [p[c] for p in row]
            i = 0
            while i < w:
                run = 1
                while i + run < w and run < 127 and vals[i + run] == vals[i]: run += 1
                if run >= 3:
                    out.extend(bytes([128 + run, vals[i]])); i += run
                else:
                    j = i
                    while j < w and j - i < 128 and not (j + 2 < w and vals[j] == vals[j + 1] == vals[j + 2]): j += 1
                    j = max(j, i + 1)
                    out.extend(bytes([j - i] + vals[i:j])); i = j
    return bytes(out)


@pytest.mark.parametrize("rle", [False, True])
def test_hdr_decoder(tmp_path, rle):
    rng = random.Random(7)
    w, h = 40, 5
    pix = [[[rng.randrange(256), rng.randrange(4) * 60, 17, rng.choice([0, 120, 128, 131])] for _ in range(w)] for _ in range(h)]
    t, px = _decode(tmp_path, "e.hdr", _hdr(w, h, pix, rle))
    assert (t["width"], t["height"], t["channels"], t["is_float"], t["has_alpha"]) == (w, h, 3, 1, 0)
    got = px.view(np.float32).reshape(h, w, 3)
    for y in range(h):
        for x in range(w):
            r, g, b, e = pix[y][x]
            f = np.float32(math.ldexp(1.0, e - 136)) if e else np.float32(0)
            assert got[y, x].tolist() == [np.float32(r) * f, np.float32(g) * f, np.float32(b) * f] if e else [0, 0, 0]


# ------------------------------------------------------------------------------------------------ differential fuzz
def _rand_color(rng):
    return [round(rng.random(), 3) for _ in range(3)]


def _rand_transforms(rng):
    out = []
    for _ in range(rng.randrange(0, 5)):
        k = rng.choice(["translate", "rotateX", "rotateY", "rotateZ", "scale", "scaleUniform"])
        if k == "translate":
            t = {"type": k}
            for ax in "XYZ":
                if rng.random() < 0.8: t[ax] = round(rng.uniform(-3, 3), 3)
            if len(t) == 1: t["X"] = 0.5
        elif k.startswith("rotate"):
            t = {"type": k, "degrees": round(rng.uniform(-180, 180), 2)} if rng.random() < 0.7 else {"type": k, "radians": round(rng.uniform(-3, 3), 3)}
        elif k == "scale":
            t = {"type": k, "X": round(rng.uniform(0.2, 2), 3), "Y": round(rng.uniform(0.2, 2), 3)}
        else:
            t = {"type": k, "scale": round(rng.uniform(0.2, 2.5), 3)}
        out.append(t)
    return out


def _rand_texnode(rng, images):
    r = rng.random()
    if r < 0.35: return _rand_color(rng) + ([round(rng.random(), 2)] if rng.random() < 0.3 else [])
    if r < 0.5: return {"r": 0.2, "g": round(rng.random(), 2), "b": 0.9}
    if r < 0.6: return {"type": "checkerboard", "size": rng.choice([2, 5, 12.5])}
    if r < 0.7: return {"type": "blackbody", "degrees": rng.choice([1500, 3200, 6600, 9000])}
    if r < 0.8: return {"blackbody": rng.choice([1900, 5000, 12000])}
    node = {"type": "image", "path": rng.choice(images)}
    if rng.random() < 0.5: node["lerp"] = rng.random() < 0.5
    if rng.random() < 0.5: node["transform"] = rng.random() < 0.5
    return node


def _rand_valnode(rng, images):
    return round(rng.random(), 3) if rng.random() < 0.7 else _rand_texnode(rng, images)


def _rand_bsdf(rng, images, depth=0):
    kinds = ["diffuse", "metal", "glass", "plastic", "transparent", "emissive"] + (["mix", "add"] if depth < 2 else [])
    k = rng.choice(kinds)
    n = {"type": k}
    if k in ("mix", "add"):
        n["A"] = _rand_bsdf(rng, images, depth + 1)
        n["B"] = _rand_bsdf(rng, images, depth + 1) if rng.random() < 0.85 else n["A"]
        if k == "mix" and rng.random() < 0.8: n["factor"] = _rand_valnode(rng, images)
        return n
    if rng.random() < 0.9: n["color"] = _rand_texnode(rng, images)
    if k in ("metal", "glass") and rng.random() < 0.7: n["roughness"] = _rand_valnode(rng, images)
    if k == "glass" and rng.random() < 0.6: n["IOR"] = rng.choice([1.1, 1.45, 1.5])
    if k == "emissive" and rng.random() < 0.7: n["strength"] = rng.choice([1, 4.5, 20])
    return n


def _write_obj(rng, path, mtl_name, with_uv, with_n, images):
    nv = rng.randrange(8, 120)
    lines = [f"mtllib {mtl_name}", "o fuzz"] if mtl_name else ["o fuzz"]
    verts = [[rng.uniform(-1, 1) for _ in range(3)] for _ in range(nv)]
    if rng.random() < 0.2:                                  # degenerate extent on one axis: exercises the NaN bins
        for v in verts: v[1] = 0.25
    lines += ["v %.5f %.5f %.5f" % tuple(v) for v in verts]
    nt = rng.randrange(3, 20) if with_uv else 0
    lines += ["vt %.4f %.4f" % (rng.uniform(-1, 2), rng.uniform(-1, 2)) for _ in range(nt)]
    nn = rng.randrange(2, 12) if with_n else 0
    for _ in range(nn):
        v = [rng.gauss(0, 1) for _ in range(3)]
        l = math.sqrt(sum(c * c for c in v)) or 1.0
        lines.append("vn %.5f %.5f %.5f" % tuple(c / l for c in v))
    mats = ["m%d" % i for i in range(rng.randrange(1, 4))] if mtl_name else []
    for _ in range(rng.randrange(4, 200)):
        if mats and rng.random() < 0.15: lines.append("usemtl " + rng.choice(mats + ["unknown"]))
        if rng.random() < 0.05: lines.append("# comment"), lines.append("")
        k = 4 if rng.random() < 0.25 else 3
        base = rng.randrange(nv)
        idx = [(base + rng.randrange(0, 6) * j) % nv + 1 for j in range(k)]
        face = "f " + " ".join("%d/%s/%d" % (i, rng.randrange(1, nt + 1) if nt and rng.random() < 0.9 else "",
                                             rng.randrange(1, nn + 1) if nn else 0) for i in idx)
        # now and then the same face many times over: identical centroids defeat the SAH, which exercises the
        # approximate-median fallback and the "nothing went left" leaf (bvh.c:196-209, :238-240)
        lines += [face] * (rng.choice([20, 45]) if rng.random() < 0.03 else 1)
    open(path, "w").write("\n".join(lines) + "\n")
    if mtl_name:
        out = ["# fuzz"]
        for m in mats:
            out += ["newmtl " + m, "Kd %.3f %.3f %.3f" % tuple(_rand_color(rng)), "Ks %.3f %.3f %.3f" % tuple(_rand_color(rng))]
            if rng.random() < 0.3: out.append("Ke %.2f %.2f %.2f" % (rng.random() * 3, rng.random(), rng.random() * 2))
            if rng.random() < 0.5: out.append("illum %d" % rng.choice([2, 5, 7]))
            if rng.random() < 0.5: out.append("Ni %.2f" % rng.uniform(1, 2))
            out += ["Ns 96.0", "d 1.0"]
            if rng.random() < 0.4: out.append("map_Kd " + os.path.basename(rng.choice(images)))
            if rng.random() < 0.2: out.append("map_Ns " + os.path.basename(rng.choice(images)))
        open(os.path.join(os.path.dirname(path), mtl_name), "w").write("\n".join(out) + "\n")


def _fuzz_scene(rng, d):
    images = []
    for i, ch in enumerate([1, 3, 4]):
        w, h = rng.randrange(2, 9), rng.randrange(2, 9)
        rows = [bytes(rng.randrange(256) for _ in range(w * ch)) for _ in range(h)]
        p = os.path.join(d, "tex%d.png" % i)
        open(p, "wb").write(_png(w, h, {1: 0, 3: 2, 4: 6}[ch], 8, rows, filters=[rng.randrange(5)]))
        images.append(p)
    pix = [[[rng.randrange(256), rng.randrange(256), rng.randrange(256), rng.randrange(120, 136)] for _ in range(16)] for _ in range(8)]
    open(os.path.join(d, "env.hdr"), "wb").write(_hdr(16, 8, pix, rng.random() < 0.5))
    prims, meshes = [], []
    for _ in range(rng.randrange(0, 6)):
        s = {"type": "sphere", "radius": round(rng.uniform(0.1, 1.5), 3),
             "instances": [{"transforms": _rand_transforms(rng)} for _ in range(rng.randrange(0, 4))]}
        if rng.random() < 0.5:
            s["material"] = _rand_bsdf(rng, images)
        else:
            s["bsdf"] = rng.choice(["lambertian", "metal", "glass", "plastic", "emissive", "bogus"])
            s["color"] = _rand_color(rng)
            if rng.random() < 0.5: s["roughness"] = round(rng.random(), 2)
            if rng.random() < 0.5: s["IOR"] = 1.33
            if rng.random() < 0.5: s["intensity"] = 7.5
        prims.append(s)
    for m in range(rng.randrange(0, 4)):
        name = "mesh%d.obj" % m
        has_mtl = rng.random() < 0.7
        _write_obj(rng, os.path.join(d, name), "mesh%d.mtl" % m if has_mtl else None, rng.random() < 0.6, rng.random() < 0.7, images)
        e = {"fileName": name, "instances": [{"transforms": _rand_transforms(rng)} for _ in range(rng.randrange(0, 4))]}
        r = rng.random()
        if r < 0.3: e["material"] = _rand_bsdf(rng, images)
        elif r < 0.45: e["material"] = [_rand_bsdf(rng, images)]
        else:
            e["bsdf"] = rng.choice(["lambertian", "metal", "glass", "plastic", "emissive"])
            if rng.random() < 0.5: e["roughness"] = round(rng.random(), 2)
            if rng.random() < 0.5: e["IOR"] = 1.6
            if rng.random() < 0.5: e["intensity"] = 3.0
        meshes.append(e)
    amb = rng.choice([{"hdr": "env.hdr", "offset": rng.choice([0, 45, -120])}, {"down": _rand_color(rng), "up": _rand_color(rng)},
                      {"hdr": "missing.hdr", "down": [1, 1, 1], "up": {"r": 0.1, "g": 0.2, "b": 0.9}}, {}])
    cam = {"FOV": rng.choice([20, 55.5, 90, 170]), "transforms": _rand_transforms(rng)}
    if rng.random() < 0.5: cam["focalDistance"] = round(rng.uniform(0.5, 9), 2)
    if rng.random() < 0.5: cam["fstops"] = rng.choice([0, 1.4, 6.5])
    return {"renderer": {"samples": rng.randrange(1, 50), "bounces": rng.randrange(0, 40), "width": rng.randrange(8, 300),
                         "height": rng.randrange(8, 200), "tileWidth": rng.choice([8, 32, 64]), "tileHeight": rng.choice([8, 32]),
                         "tileOrder": rng.choice(["random", "topToBottom", "fromMiddle", "toMiddle", "normal"])},
            "display": {}, "camera": cam, "scene": {"ambientColor": amb, "primitives": prims, "meshes": meshes}}


@pytest.mark.parametrize("seed", range(40))
def test_fuzz_against_live_reference(seed, tmp_path, monkeypatch):
    if not os.path.exists(REF):
        pytest.skip("oracle/_ref/cray_ref_strict is only built where /root/reference exists")
    rng = random.Random(1000 + seed)
    d = str(tmp_path)
    scene = _fuzz_scene(rng, d)
    if not scene["scene"]["primitives"] and not any(m["instances"] for m in scene["scene"]["meshes"]):
        scene["scene"]["primitives"] = [{"type": "sphere", "radius": 1, "instances": [{}], "color": [1, 0, 0], "bsdf": "metal"}]
    open(os.path.join(d, "fuzz.json"), "w").write(json.dumps(scene, indent=1))
    monkeypatch.chdir(d)
    r = subprocess.run([REF, "export", "fuzz.json", "0", "0", "0", "0", "ref.crscene"], cwd=d, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=120)
    assert r.returncode == 0, r.stdout[-2000:]
    mine = crscene.load_json("fuzz.json")
    ref = load_crscene(os.path.join(d, "ref.crscene"))
    assert_same_scene(mine, ref)
    crscene.free(mine)


def _big_scene(d, rng, tris=60000):
    """One mesh big enough (> 1 MB of text, > 8192 triangles) to take the loader's multi-threaded parse and BVH build."""
    lines = ["mtllib big.mtl", "o big"]
    nv = tris // 2 + 3
    for i in range(nv):
        a = i * 0.001
        # a band of vertices with y exactly +0 / -0 (Blender writes "-0.000000"): the builder's min/max keep the LAST of two
        # equal values, so the sign of a zero bound depends on visiting order — the threaded build must reproduce it
        y = rng.choice(["0.000000", "-0.000000"]) if 1000 <= i < 9000 else "%.6f" % rng.uniform(-1, 1)
        lines.append("v %.6f %s %.6f" % (math.cos(a * 7) * (1 + a), y, math.sin(a * 5) * (1 + 0.5 * a)))
    lines += ["vt %.5f %.5f" % (rng.random(), rng.random()) for _ in range(64)]
    lines += ["vn 0 1 0", "vn 0.6 0.8 0"]
    for i in range(tris):
        if i % 5000 == 0: lines.append("usemtl m%d" % ((i // 5000) % 3))
        a = rng.randrange(nv - 2)
        if i % 7 == 0:
            lines.append("f %d/%d/1 %d/%d/2 %d/%d/1 %d/%d/2" % (a + 1, i % 64 + 1, a + 2, (i + 1) % 64 + 1, a + 3, (i + 2) % 64 + 1, (a + 40) % nv + 1, 1))
        else:
            lines.append("f %d//1 %d//2 %d//1" % (a + 1, a + 2, (a + 17) % nv + 1))
    open(os.path.join(d, "big.obj"), "w").write("\n".join(lines) + "\n")
    open(os.path.join(d, "big.mtl"), "w").write("newmtl m0\nKd 0.8 0.1 0.1\nnewmtl m1\nKd 0.1 0.8 0.1\nillum 5\nnewmtl m2\nKd 0.1 0.1 0.8\nillum 7\nNi 1.4\n")
    scene = {"renderer": {"width": 64, "height": 48, "samples": 2, "bounces": 3}, "camera": {"FOV": 60},
             "scene": {"ambientColor": {"down": [1, 1, 1], "up": [0.2, 0.3, 1]},
                       "meshes": [{"fileName": "big.obj", "bsdf": "plastic",
                                   "instances": [{"transforms": [{"type": "translate", "Z": 6}]},
                                                 {"transforms": [{"type": "rotateY", "degrees": 30}, {"type": "translate", "X": 4, "Z": 9}]}]}]}}
    open(os.path.join(d, "big.json"), "w").write(json.dumps(scene))


def test_large_mesh_same_for_any_thread_count(tmp_path, monkeypatch):
    d = str(tmp_path)
    _big_scene(d, random.Random(5))
    assert os.path.getsize(os.path.join(d, "big.obj")) > (1 << 20)
    monkeypatch.chdir(d)
    scenes = []
    for threads in ("1", "2", "7"):
        monkeypatch.setenv("CRLOADER_THREADS", threads)
        scenes.append(crscene.load_json("big.json"))
    assert scenes[0].poly_count > 60000 and scenes[0].bvh_node_count > 10000
    for other in scenes[1:]:
        A, B = crscene.arrays(scenes[0]), crscene.arrays(other)
        for key in A:
            assert A[key].tobytes() == B[key].tobytes(), key
    if os.path.exists(REF):                                  # and the same as the reference's serial build
        r = subprocess.run([REF, "export", "big.json", "0", "0", "0", "0", "ref.crscene"], cwd=d, stdout=subprocess.PIPE,
                           stderr=subprocess.STDOUT, text=True, timeout=300)
        assert r.returncode == 0, r.stdout[-2000:]
        assert_same_scene(scenes[2], load_crscene(os.path.join(d, "ref.crscene")))
    for s_ in scenes:
        crscene.free(s_)


def test_texture_that_fails_late_falls_back_to_ordered_loading(tmp_path, monkeypatch):
    """Textures are decoded on background threads; a file whose header is fine but whose deflate stream is corrupt is only
    known to be bad after the node graph has been built with it.  The loader must then redo the load in order, ending with
    the graph without an image node (a NULL texture makes no node, image.c:51) — same bytes with or without background decoding."""
    d = str(tmp_path)
    good = _png(5, 4, 2, 8, [bytes(range(15))] * 4)
    bad = bytearray(_png(64, 64, 6, 8, [bytes((x * 7 + y) & 255 for x in range(256)) for y in range(64)]))
    idat = bad.index(b"IDAT") + 4
    for i in range(idat + 2, idat + 40): bad[i] ^= 0x5a                   # keep chunk structure and CRC field layout, break the deflate data
    open(os.path.join(d, "good.png"), "wb").write(good)
    open(os.path.join(d, "bad.png"), "wb").write(bytes(bad))
    scene = {"renderer": {"width": 8, "height": 8}, "camera": {}, "scene": {"primitives": [
        {"type": "sphere", "radius": 1, "instances": [{}], "material": {"type": "diffuse", "color": {"type": "image", "path": "good.png"}}},
        {"type": "sphere", "radius": 1, "instances": [{}], "material": {"type": "metal", "color": {"type": "image", "path": "bad.png"}, "roughness": 0.3}}]}}
    open(os.path.join(d, "s.json"), "w").write(json.dumps(scene))
    monkeypatch.chdir(d)
    a = crscene.load_json("s.json")
    monkeypatch.setenv("CRLOADER_SYNC_TEXTURES", "1")
    b = crscene.load_json("s.json")
    A, B = crscene.arrays(a), crscene.arrays(b)
    assert a.texture_count == 1 and a.node_count == b.node_count
    for key in A:
        assert A[key].tobytes() == B[key].tobytes(), key
    if os.path.exists(REF):
        r = subprocess.run([REF, "export", "s.json", "0", "0", "0", "0", "ref.crscene"], cwd=d, stdout=subprocess.PIPE,
                           stderr=subprocess.STDOUT, text=True, errors="replace", timeout=60)
        # the reference itself aborts on this input ("free(): invalid pointer": loadTextureFromBuffer destroys a texture that
        # lives in the node pool, textureloader.c:78-84) — compare only if a build of it survives
        if r.returncode == 0:
            assert_same_scene(a, load_crscene(os.path.join(d, "ref.crscene")))
    crscene.free(a); crscene.free(b)


# ---- odd but legal inputs: wrong-typed values, missing fields, key case, no-op / unknown transforms, NULL node inputs -------
def _odd_transforms(rng):
    out=[]
    for _ in range(rng.randrange(0,6)):
        out.append(rng.choice([
            {"type":"translate"},                       # no coords -> NOP
            {"type":"translate","x":1.5},              # lower-case keys (case-insensitive lookup)
            {"type":"rotateX"},                         # no angle -> NOP
            {"type":"rotateY","degrees":"90"},         # string, not number -> invalid
            {"type":"rotateZ","radians":0.7,"degrees":33},   # degrees wins
            {"type":"scale","Z":2.0},                  # others default to 1
            {"type":"scale"},                           # invalid -> NOP
            {"type":"scaleUniform"},                    # invalid
            {"type":"scaleUniform","scale":0.3},
            {"type":"shear","X":1},                    # unknown type
            {"type":"translate","X":-0.0,"Y":1e-30,"Z":1e20},
            {"type":"rotateX","degrees":720.5},
        ]))
    return out
def _odd_scene(rng, d):
    images=[]
    rows=[bytes(rng.randrange(256) for _ in range(4*3)) for _ in range(3)]
    p=os.path.join(d,"t.png"); open(p,"wb").write(_png(4,3,2,8,rows)); images.append(p)
    prims=[]
    for _ in range(rng.randrange(1,6)):
        s={"type":"sphere"}
        if rng.random()<0.8: s["radius"]=rng.choice([0.5,1,"2",-1.0,0])
        if rng.random()<0.9: s["instances"]=[{"transforms":_odd_transforms(rng)} if rng.random()<0.8 else {} for _ in range(rng.randrange(0,3))]
        r=rng.random()
        if r<0.3: s["material"]=rng.choice([{"type":"diffuse"},{"type":"mix"},{"type":"mix","A":{"type":"diffuse","color":[1,0,0]}},{"type":"add","A":{"type":"metal"},"B":{"type":"metal"}},
                                            {"type":"unknown"},{"no":"type"},{"type":"emissive","color":{"type":"checkerboard","size":3},"strength":{"type":"checkerboard","size":2}},
                                            {"type":"glass","color":[1,1,1],"roughness":{"path":images[0]},"IOR":{"r":1,"g":1,"b":1}},
                                            {"type":"plastic"},{"type":"transparent"},{"type":"metal","color":"t.png"},{"type":"diffuse","color":{"path":"nonexistent.png"}},
                                            {"type":"diffuse","color":{"type":"image","path":images[0],"transform":False,"lerp":True}}])
        else:
            if rng.random()<0.8: s["bsdf"]=rng.choice(["lambertian","metal","glass","plastic","emissive","EMISSIVE",5])
            if rng.random()<0.8: s["color"]=rng.choice([[1,0.5],[0.1,0.2,0.3,0.4],{"r":0.5},{"blackbody":2500},{"blackbody":"x","g":0.5},[]])
            if rng.random()<0.5: s["intensity"]=rng.choice([2,"3",0])
            if rng.random()<0.5: s["roughness"]=rng.choice([0.25,"0.5",-1])
            if rng.random()<0.5: s["IOR"]=rng.choice([1.5,"1.5"])
        prims.append(s)
    prims.append({"type":"cube"}) if rng.random()<0.3 else None
    cam={}
    if rng.random()<0.8: cam[rng.choice(["FOV","fov","Fov"])]=rng.choice([-5,0,45,181,90.5])
    if rng.random()<0.6: cam["focalDistance"]=rng.choice([-1,0,3.5])
    if rng.random()<0.6: cam["fstops"]=rng.choice([-1,0,2.8])
    if rng.random()<0.7: cam["transforms"]=_odd_transforms(rng)
    ren={}
    for k,vals in (("samples",[0,-1,3,2.7]),("bounces",[-2,0,7]),("width",[17,0.0,64]),("height",[9,33]),("tileWidth",[0,5]),("tileHeight",[-3,7]),("threads",[0,-1,3]),("tileOrder",["random","normal","xyz",3])):
        if rng.random()<0.7: ren[rng.choice([k,k.upper(),k.capitalize()])]=rng.choice(vals)
    amb=rng.choice([{}, {"offset":90}, {"down":[0,0,0]}, {"down":[1,1,1],"up":[0,0,1],"offset":"5"}, {"hdr":5,"up":[1,1,1],"down":{"blackbody":6000}}])
    sc={"camera":cam,"scene":{"ambientColor":amb,"primitives":prims}}
    if rng.random()<0.9: sc["renderer"]=ren
    return sc


def test_odd_inputs_against_live_reference(tmp_path, monkeypatch):
    """Defaults, clamps and fallbacks of the JSON dialect (sceneloader.c): 60 scenes made of values the loader has to
    tolerate — strings where numbers belong, missing radius/color/bsdf, lower-case keys, transforms without arguments,
    mix/add nodes with missing inputs, unknown node and primitive types, textures that do not exist."""
    if not os.path.exists(REF):
        pytest.skip("oracle/_ref/cray_ref_strict is only built where /root/reference exists")
    compared = 0
    for seed in range(60):
        rng = random.Random(777 + seed)
        d = str(tmp_path / ("odd%d" % seed))
        os.makedirs(d)
        sc = _odd_scene(rng, d)
        if any(k.lower() in ("width", "height") and v == 0 for k, v in sc.get("renderer", {}).items()):
            continue                                         # zero-sized image: the reference divides by zero, the loader reports it
        open(os.path.join(d, "s.json"), "w").write(json.dumps(sc))
        r = subprocess.run([REF, "export", "s.json", "0", "0", "0", "0", "ref.crscene"], cwd=d, stdout=subprocess.PIPE,
                           stderr=subprocess.STDOUT, text=True, errors="replace", timeout=60)
        assert r.returncode == 0, (seed, r.stdout[-500:])
        monkeypatch.chdir(d)
        mine = crscene.load_json("s.json")
        assert_same_scene(mine, load_crscene(os.path.join(d, "ref.crscene")))
        crscene.free(mine)
        compared += 1
    assert compared >= 40


# ------------------------------------------------------------------------------------------------ GPU end to end
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["g_nodes", "g_meshmat", "g_single"])
def test_json_scene_renders_like_reference(name, monkeypatch):
    """JSON -> loader -> GPU gives the reference's framebuffer (same bar as the .crscene parity tests)."""
    monkeypatch.chdir(GOLDEN)
    g = crgpu.GpuScene(name + ".json")
    g.render_frame()
    got = g.read()
    ref = np.fromfile(os.path.join(GOLDEN, name + ".f32"), dtype=np.float32).reshape(got.shape)
    rmse = float(np.sqrt(np.mean((got.astype(np.float64) - ref) ** 2)))
    g.close()
    assert rmse <= 1e-4, rmse
