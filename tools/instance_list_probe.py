"""Cost of adding and removing instances of a resident scene against reloading it (crgpu_scene_set_instance_list, include/crgpu.h).

Cases (tests/test_gpu_instance_list.py builds the same kind of scenes):
  hdr +venus    hdr.json at 1920x1080 with a second Venus instance (13 -> 14 instances)
  hdr -light    hdr.json at 1920x1080 without one of its light spheres (13 -> 12)
  grow 40,009   the 20,009-instance generated scene (20,000 spheres of 40 objects and 9 teapots) grown to 40,009
  scatter 1M    one sphere instance scattered to 1,000,000
For each case:
  first    the first crgpu_scene_set_instance_list to the new list (it also gives the scene its instance block, and a top region
           and pairs block when they have to grow)
  later    later calls to the new list, each after a call back to the original list (medians of --reps)
  back     those calls back to the original list
  reload   crloader_load_json_buf of the edited JSON text + crgpu_prepare + crgpu_scene_create_prepared (medians of 3)
Each edit is also checked bit for bit against a fresh upload of the edited scene at 160x90 (frame, ray records, P/T/S/I).  Times
are host wall clock around calls that end in a device synchronise.

    python tools/instance_list_probe.py [--reps 10] [--out profiles/r07_instance_list_probe.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "c-ray_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

import test_gpu_instance_list as I  # noqa: E402
import test_gpu_scene_edit as T  # noqa: E402
from edit_probe import reload_ms, wall  # noqa: E402


def cases():
    hdr = T.scene_json("hdr")
    big = (1920, 1080, 1000, 32)
    gen = (1920, 1080, 1000, 8)
    yield "hdr +venus", big, hdr, I.duplicated(hdr, "hdr")
    yield "hdr -light", big, hdr, I.removed(hdr)
    yield "grow 40,009", gen, I.objects(I.scattered(20000, 1), mesh_on=I.ALL), I.objects(I.scattered(40000, 2), mesh_on=I.ALL)
    yield "scatter 1M", gen, T.sphere_scene(T.spread(1, 3), radius=0.5), T.sphere_scene(T.spread(1000000, 4), radius=0.5)


def probe(label, cfg, doc_a, doc_b, reps):
    a, b = T.Loaded(doc_a, *cfg), T.Loaded(doc_b, *cfg)
    na, nb = len(a.instances), len(b.instances)
    g = a.upload()
    first = wall(lambda: g.set_instance_list(b.instances))
    later, back = [], []
    for _ in range(reps):
        back.append(wall(lambda: g.set_instance_list(a.instances)))
        later.append(wall(lambda: g.set_instance_list(b.instances)))
    g.close()
    a.free()
    b.free()
    reload = [reload_ms(doc_b, cfg) for _ in range(3)]
    sa, sb = T.Loaded(doc_a, 160, 90, 2, 8), T.Loaded(doc_b, 160, 90, 2, 8)
    g = sa.upload()
    g.set_instance_list(sb.instances)
    T.assert_same_as_fresh(g, sb, T.ray_set(sb.camera, n=4096))
    g.close()
    sa.free()
    sb.free()
    return dict(case=label, size=cfg[:2], instances_before=na, instances_after=nb, set_instance_list_first_ms=first,
                set_instance_list_ms=float(np.median(later)), set_instance_list_back_ms=float(np.median(back)),
                reload_prepare_create_ms=float(np.median(reload)), checked=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the results to this JSON file")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True).stdout.strip()
    print("gpu:", gpu)
    out = dict(gpu=gpu, reps=args.reps, cases=[])
    for c in cases():
        r = probe(*c, args.reps)
        out["cases"].append(r)
        print(json.dumps(r), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
