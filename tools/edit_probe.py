"""Cost of editing a resident scene against reloading it (crgpu_scene_set_camera / crgpu_scene_set_instances, include/crgpu.h).

For hdr, venus, refraction and a generated scene of 20,009 instances (tests/test_gpu_scene_edit.py), at bench.py's frame size:
  reload   crloader_load_json_buf of the edited JSON text + crgpu_prepare + crgpu_scene_create_prepared (what an edit costs without
           the edit calls)
  camera   crgpu_scene_set_camera
  first    the first crgpu_scene_set_instances (it also copies the scene's BVH pair nodes into the scene's own block)
  later    later crgpu_scene_set_instances calls
Each edit is checked against a fresh upload of the edited scene (one small frame, bit for bit).  Then bench.py runs once on the
unedited default workload and its frame CRC is printed.  Times are host wall clock around calls that end in a device synchronise;
medians of --reps.

    python tools/edit_probe.py [--reps 20] [--out results.json]
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
sys.path[:0] = [os.path.join(ROOT, "c-ray_b200"), os.path.join(ROOT, "tests")]

import crgpu  # noqa: E402
import crscene  # noqa: E402
import test_gpu_scene_edit as T  # noqa: E402

SIZES = {"hdr": (1920, 1080, 1000, 32), "venus": (2560, 1600, 1000, 25), "refraction": (1920, 1080, 2500, 512), "many": (1920, 1080, 1000, 8)}


def docs(name):
    if name == "many":
        pos = T.spread(20000, 1)
        moved = pos + np.round(np.random.default_rng(2).normal(0.0, 15.0, pos.shape), 3)
        return (T.sphere_scene(pos, groups=40, meshes=T.teapots(), radius=2.0),
                T.sphere_scene(moved, groups=40, meshes=T.teapots(60.0), radius=2.0))
    doc = T.scene_json(name)
    return doc, T.edited(doc, T.STEP[name])


def wall(fn):
    t = time.perf_counter()
    fn()
    return (time.perf_counter() - t) * 1e3


def reload_ms(doc_b, cfg):
    L = crgpu.lib()
    L.crgpu_prepare.argtypes = [C.POINTER(crgpu.FlatScene), C.POINTER(C.c_void_p)]
    L.crgpu_prepared_free.argtypes = [C.c_void_p]
    t = time.perf_counter()
    flat = T.load(doc_b)
    L.crscene_set_config(C.byref(flat), *cfg)
    p, h = C.c_void_p(), C.c_void_p()
    crgpu._check(L.crgpu_prepare(C.byref(flat), C.byref(p)), "crgpu_prepare")
    crgpu._check(L.crgpu_scene_create_prepared(p, 0, C.byref(h)), "crgpu_scene_create_prepared")
    ms = (time.perf_counter() - t) * 1e3
    L.crgpu_scene_destroy(h)
    L.crgpu_prepared_free(p)
    crscene.free(flat)
    return ms


def probe(name, reps):
    doc_a, doc_b = docs(name)
    cfg = SIZES[name]
    a, b = T.Loaded(doc_a, *cfg), T.Loaded(doc_b, *cfg)
    n = len(b.instances)
    g = a.upload()
    first = wall(lambda: g.set_instances(b.instances))
    cam = [wall(lambda: g.set_camera(b.camera)) for _ in range(reps)]
    later = [wall(lambda: g.set_instances(b.instances)) for _ in range(reps)]
    g.close()
    reload = [reload_ms(doc_b, cfg) for _ in range(max(3, reps // 5))]
    a.free()
    b.free()
    # the same edit at a small size, against a fresh upload
    sa, sb = T.Loaded(doc_a, 160, 90, 2, 8), T.Loaded(doc_b, 160, 90, 2, 8)
    g = sa.upload()
    T.edit(g, sb)
    T.assert_same_as_fresh(g, sb, T.ray_set(sb.camera, n=4096))
    g.close()
    sa.free()
    sb.free()
    return dict(scene=name, instances=n, size=cfg[:2], set_camera_ms=float(np.median(cam)),
                set_instances_first_ms=first, set_instances_ms=float(np.median(later)), reload_prepare_create_ms=float(np.median(reload)),
                checked=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--no-bench", action="store_true")
    ap.add_argument("--out", default=None, help="also write the results to this JSON file")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True).stdout.strip()
    print("gpu:", gpu)
    out = dict(gpu=gpu, scenes=[])
    for name in ("hdr", "venus", "refraction", "many"):
        r = probe(name, args.reps)
        out["scenes"].append(r)
        print(json.dumps(r))
    if not args.no_bench:
        r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", "1", "--warmup", "1"],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, cwd=ROOT)
        line = [x for x in r.stdout.splitlines() if x.startswith("{")][-1]
        out["bench_frame_crc32"] = json.loads(line).get("frame_crc32")
        print("bench frame_crc32 (unedited hdr):", out["bench_frame_crc32"])
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
