"""Cost of changing the render settings of a resident scene against re-creating it (crgpu_scene_set_render, include/crgpu.h).

Cases, on hdr.json uploaded at 1920x1080, 1000 spp, 32 bounces:
  1080p -> 540p      image size 960x540
  540p -> 2160p      then 3840x2160 on the same scene
  16 views -> 2160p  a 16-view list, all of them to 3840x2160
  spp/bounces        1920x1080 kept, 64 spp and 8 bounces, cameras kept
For each case:
  set_render       crgpu_scene_set_render: the first call of the process for the case, and the median of --reps calls, each on
                   another freshly uploaded scene
  update+create    crgpu_prepared_update_config + crgpu_scene_create_prepared from a prepared scene (loses every edit), and
                   crgpu_scene_set_views for the views case (medians of --reps)
  reload           crloader_load_json_buf of the JSON text + crscene_set_config + crgpu_prepare + crgpu_scene_create_prepared,
                   and crgpu_scene_set_views for the views case (medians of 3)
Each case is also checked bit for bit at a small size against a fresh upload at the new settings (every view's frame).  Times are
host wall clock around calls that end in a synchronise of the scene's stream, which holds all of their device work.

    python tools/render_settings_probe.py [--reps 5] [--out profiles/r11_render_settings_probe.json]
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
import test_gpu_scene_edit as T  # noqa: E402
from edit_probe import wall  # noqa: E402
from test_gpu_render_settings import Src, _At  # noqa: E402
from test_gpu_views import cameras  # noqa: E402

BIG = (1920, 1080, 1000, 32)
# label -> (settings before, settings after, views, cameras given); the small-size check uses the same change at a 1/12 scale
CASES = [("1080p -> 540p", BIG, (960, 540, 1000, 32), 1, True),
         ("540p -> 2160p", (960, 540, 1000, 32), (3840, 2160, 1000, 32), 1, True),
         ("16 views -> 2160p", BIG, (3840, 2160, 1000, 32), 16, True),
         ("spp/bounces", BIG, (1920, 1080, 64, 8), 1, False)]


def small(cfg):
    return (max(1, cfg[0] // 12), max(1, cfg[1] // 12), cfg[2] % 7 + 1, cfg[3])


def cams_at(src, cfg, n):
    return cameras("hdr", _At(src, cfg), n)


def lib():
    L = crgpu.lib()
    L.crgpu_prepare.argtypes = [C.POINTER(crgpu.FlatScene), C.POINTER(C.c_void_p)]
    L.crgpu_prepared_free.argtypes = [C.c_void_p]
    L.crgpu_prepared_update_config.argtypes = [C.c_void_p, C.POINTER(crgpu.FlatScene)]
    return L


def adopt(h, cfg):
    g = crgpu.GpuScene.__new__(crgpu.GpuScene)
    g.handle = h
    g.W, g.H, g.samples, g.bounces = cfg
    return g


def set_render_ms(src, before, after, views, with_cams):
    g = src.upload(before)
    if views > 1:
        g.set_views(cams_at(src, before, views))
    cams = cams_at(src, after, views) if with_cams else None
    ms = wall(lambda: g.set_render(*after, cams))
    g.close()
    return ms


def update_create_ms(src, before, after, views):
    """from a prepared scene: update its config and create the device scene again (and give it its views)"""
    L = lib()
    src.camera(before)
    p = C.c_void_p()
    crgpu._check(L.crgpu_prepare(C.byref(src.flat), C.byref(p)), "crgpu_prepare")
    cams = cams_at(src, after, views) if views > 1 else None
    src.camera(after)
    t = time.perf_counter()
    crgpu._check(L.crgpu_prepared_update_config(p, C.byref(src.flat)), "crgpu_prepared_update_config")
    h = C.c_void_p()
    crgpu._check(L.crgpu_scene_create_prepared(p, 0, C.byref(h)), "crgpu_scene_create_prepared")
    g = adopt(h, after)
    if cams:
        g.set_views(cams)
    ms = (time.perf_counter() - t) * 1e3
    g.close()
    L.crgpu_prepared_free(p)
    return ms


def reload_ms(src, doc, after, views):
    L = lib()
    cams = cams_at(src, after, views) if views > 1 else None
    t = time.perf_counter()
    flat = T.load(doc)
    L.crscene_set_config(C.byref(flat), *after)
    p, h = C.c_void_p(), C.c_void_p()
    crgpu._check(L.crgpu_prepare(C.byref(flat), C.byref(p)), "crgpu_prepare")
    crgpu._check(L.crgpu_scene_create_prepared(p, 0, C.byref(h)), "crgpu_scene_create_prepared")
    g = adopt(h, after)
    if cams:
        g.set_views(cams)
    ms = (time.perf_counter() - t) * 1e3
    g.close()
    L.crgpu_prepared_free(p)
    crscene.free(flat)
    return ms


def check(src, before, after, views, with_cams):
    """the change at a small size renders every view as a fresh upload at the new settings"""
    before, after = small(before), small(after)
    g = src.upload(before)
    h = src.upload(after)
    try:
        old = cams_at(src, before, views)
        if views > 1:
            g.set_views(old)
        new = cams_at(src, after, views) if with_cams else old
        g.set_render(*after, new if with_cams else None)
        full = [(0, 0, after[0], after[1])]
        for v in range(views):
            g.view_clear(v)
        g.render_views(full)
        for v in range(views):
            h.set_camera(new[v])
            h.clear()
            h.render_tiles(full)
            assert g.view_read(v).tobytes() == h.read().tobytes(), v
    finally:
        g.close()
        h.close()
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the results to this JSON file")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True).stdout.strip()
    print("gpu:", gpu)
    out = dict(gpu=gpu, reps=args.reps, cases=[])
    doc = T.scene_json("hdr")
    src = Src.doc(doc)
    try:
        for label, before, after, views, with_cams in CASES:
            sr = [set_render_ms(src, before, after, views, with_cams) for _ in range(args.reps + 1)]
            uc = [update_create_ms(src, before, after, views) for _ in range(args.reps)]
            rl = [reload_ms(src, doc, after, views) for _ in range(3)]
            r = dict(case=label, before=before, after=after, views=views, set_render_first_ms=sr[0],
                     set_render_ms=float(np.median(sr[1:])), update_config_create_ms=float(np.median(uc)),
                     reload_prepare_create_ms=float(np.median(rl)), checked=check(src, before, after, views, with_cams))
            out["cases"].append(r)
            print(json.dumps(r), flush=True)
    finally:
        src.free()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
