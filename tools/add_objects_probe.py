"""Cost of adding meshes and spheres to a resident scene against reloading it (crgpu_scene_add_objects, include/crgpu.h).

Cases (tests/test_gpu_add_objects.py builds the same kind of scenes):
  hdr +venus     hdr.json at 1920x1080 with a second Venus mesh (274k triangles) and one more sphere
  spheres +pots  200 sphere instances of 8 objects, grown by the refraction scene's teapot meshes (9 load)
  hdr +1M        hdr.json with a generated 1,002,528-triangle mesh
  +64 meshes     the sphere scene grown by 64 teapot meshes in one call
For each case:
  first    crgpu_scene_add_objects on a freshly uploaded scene, the first add of the process for that case
  later    the same add, each on another freshly uploaded scene (medians of --reps)
  reload   crloader_load_json_buf of the grown JSON text + crgpu_prepare + crgpu_scene_create_prepared (medians of 3)
Each add is also checked bit for bit against a fresh upload of the grown scene at 160x90 (frame, ray records, P/T/S/I).  Times are
host wall clock around calls that end in a device synchronise; the split of an add's time into its steps is not measured.

    python tools/add_objects_probe.py [--reps 5] [--out profiles/r10_add_objects_probe.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "c-ray_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

import crgpu  # noqa: E402
import crscene  # noqa: E402
import test_gpu_add_objects as A  # noqa: E402
import test_gpu_mesh_edit as ME  # noqa: E402
import test_gpu_scene_edit as T  # noqa: E402
from edit_probe import wall  # noqa: E402


def reload_ms(doc, cfg, assets):
    L = crgpu.lib()
    L.crgpu_prepare.argtypes = [C.POINTER(crgpu.FlatScene), C.POINTER(C.c_void_p)]
    L.crgpu_prepared_free.argtypes = [C.c_void_p]
    t = time.perf_counter()
    flat = T.load(doc, T.REFDIR, assets)
    L.crscene_set_config(C.byref(flat), *cfg)
    p, h = C.c_void_p(), C.c_void_p()
    crgpu._check(L.crgpu_prepare(C.byref(flat), C.byref(p)), "crgpu_prepare")
    crgpu._check(L.crgpu_scene_create_prepared(p, 0, C.byref(h)), "crgpu_scene_create_prepared")
    ms = (time.perf_counter() - t) * 1e3
    L.crgpu_scene_destroy(h)
    L.crgpu_prepared_free(p)
    crscene.free(flat)
    return ms


def cases(assets):
    hdr = T.scene_json("hdr")
    big = (1920, 1080, 1000, 32)
    gen = (1920, 1080, 1000, 8)
    yield "hdr +venus", big, hdr, A.grown("hdr", hdr)
    spheres = T.sphere_scene(T.spread(200, 31), groups=8)
    yield "spheres +pots", gen, spheres, T.sphere_scene(T.spread(200, 31), groups=8, meshes=T.teapots())
    k = 708
    xs = np.arange(k + 1) / k
    X, Y = np.meshgrid(xs, xs, indexing="ij")
    assets.write("grid.obj", ME.grid_obj(k, 0.3 * np.sin(6.0 * X) * np.cos(5.0 * Y)))
    yield "hdr +1M", big, hdr, A.with_mesh(hdr, {"fileName": "grid.obj", "bsdf": "lambertian", "instances": [
        {"transforms": [{"type": "scaleUniform", "scale": 0.002}, {"type": "translate", "x": -0.2, "y": 0.0, "z": 0.0}]}]})
    pots = A.bundled_pots()
    many = spheres
    for i in range(64):
        many = A.with_mesh(many, pots[i % len(pots)], (25.0 * (i % 8), 0.0, 25.0 * (i // 8)))
    yield "+64 meshes", gen, spheres, many


def probe(label, cfg, doc_a, doc_b, reps, assets):
    a, b = T.Loaded(doc_a, *cfg, asset_path=assets), T.Loaded(doc_b, *cfg, asset_path=assets)
    added = dict(meshes=b.flat.mesh_count - a.flat.mesh_count, spheres=b.flat.sphere_count - a.flat.sphere_count,
                 polys=b.flat.poly_count - a.flat.poly_count)
    times = []
    for _ in range(reps + 1):
        g = a.upload()
        times.append(wall(lambda: g.add_objects(b.flat)))
        g.close()
    a.free()
    b.free()
    reload = [reload_ms(doc_b, cfg, assets) for _ in range(3)]
    sa, sb = T.Loaded(doc_a, 160, 90, 2, 8, asset_path=assets), T.Loaded(doc_b, 160, 90, 2, 8, asset_path=assets)
    g = sa.upload()
    g.add_objects(sb.flat)
    T.assert_same_as_fresh(g, sb, T.ray_set(sb.camera, n=4096))
    g.close()
    sa.free()
    sb.free()
    return dict(case=label, size=cfg[:2], added=added, add_objects_first_ms=times[0], add_objects_ms=float(np.median(times[1:])),
                reload_prepare_create_ms=float(np.median(reload)), checked=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the results to this JSON file")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True).stdout.strip()
    print("gpu:", gpu)
    out = dict(gpu=gpu, reps=args.reps, cases=[])
    assets = ME.Assets()
    try:
        for c in cases(assets):
            r = probe(*c, args.reps, assets.dir)
            out["cases"].append(r)
            print(json.dumps(r), flush=True)
    finally:
        assets.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
