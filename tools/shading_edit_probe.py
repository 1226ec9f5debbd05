"""Cost of editing the materials and the background of a resident scene against reloading it (crgpu_scene_set_shading,
include/crgpu.h).

Cases (tests/test_gpu_shading_edit.py recolour_doc builds the same variants):
  hdr         hdr.json with its environment swapped from HDRs/roof_garden_1k.hdr to HDRs/rooitou_park_1k.hdr at another offset, and
              its spheres recoloured and re-bsdf'd, at bench.py's frame size
  venus       venus.json with other mesh bsdfs and a sphere recoloured
  refraction  refraction.json, the same kind of edit
  reload      crloader_load_json_buf of the edited scene + crgpu_prepare + crgpu_scene_create_prepared (what the edit costs without
              set_shading)
  first       the first set_shading of the scene (it allocates the scene's shading block)
  later       later set_shading calls, alternating the edited and the original shading
Every call uploads the node graph, the texture table and all texel data (texel_bytes), whatever changed.  Each edit is also checked
against a fresh upload of the edited scene at a small size (frame, trace_kat records, shade_rays results and the shading queries, bit
for bit).  Then bench.py runs once on the unedited default workload and its frame CRC is printed.  Times are host wall clock around
calls that end in a device synchronise; medians of --reps.

    python tools/shading_edit_probe.py [--reps 10] [--out results.json]
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
import test_gpu_scene_edit as T  # noqa: E402
import test_gpu_shading_edit as S  # noqa: E402

CASES = {"hdr": (1920, 1080, 1000, 32), "venus": (2560, 1600, 32, 25), "refraction": (1920, 1080, 64, 512)}


def wall(fn):
    t = time.perf_counter()
    fn()
    return (time.perf_counter() - t) * 1e3


def reload_ms(doc, cfg):
    L = crgpu.lib()
    L.crgpu_prepare.argtypes = [C.POINTER(crgpu.FlatScene), C.POINTER(C.c_void_p)]
    L.crgpu_prepared_free.argtypes = [C.c_void_p]
    t = time.perf_counter()
    b = T.Loaded(doc, *cfg)
    p, h = C.c_void_p(), C.c_void_p()
    crgpu._check(L.crgpu_prepare(C.byref(b.flat), C.byref(p)), "crgpu_prepare")
    crgpu._check(L.crgpu_scene_create_prepared(p, 0, C.byref(h)), "crgpu_scene_create_prepared")
    ms = (time.perf_counter() - t) * 1e3
    L.crgpu_scene_destroy(h)
    L.crgpu_prepared_free(p)
    b.free()
    return ms


def probe(case, reps):
    cfg = CASES[case]
    doc, doc_b = T.scene_json(case), S.recolour_doc(case)
    a, b = S.bundled_pair(case, *cfg, doc_b=doc_b)
    g = a.upload()
    first = wall(lambda: g.set_shading(b.flat))
    later = [wall(lambda k=k: g.set_shading((a if k % 2 == 0 else b).flat)) for k in range(reps)]
    g.close()
    reload = [reload_ms(doc_b, cfg) for _ in range(max(3, reps // 3))]
    out = dict(case=case, size=cfg[:2], materials=int(a.flat.material_count), nodes=[int(a.flat.node_count), int(b.flat.node_count)],
               textures=[int(a.flat.texture_count), int(b.flat.texture_count)],
               texel_bytes=[int(a.flat.texdata_bytes), int(b.flat.texdata_bytes)],
               set_shading_first_ms=first, set_shading_ms=float(np.median(later)), reload_prepare_create_ms=float(np.median(reload)))
    a.free()
    b.free()
    a, b = S.bundled_pair(case, 160, 90, 2, 8, doc_b=doc_b)      # the same edit at a small size, against a fresh upload
    g = a.upload()
    g.set_shading(b.flat)
    S.assert_same_as_fresh(g, b.flat)
    g.close()
    a.free()
    b.free()
    out["checked"] = True
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--no-bench", action="store_true")
    ap.add_argument("--out", default=None, help="also write the results to this JSON file")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True).stdout.strip()
    print("gpu:", gpu)
    out = dict(gpu=gpu, cases=[])
    for case in CASES:
        r = probe(case, args.reps)
        out["cases"].append(r)
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
