"""Cost of rendering V views of a resident scene in one call against V single-camera calls (crgpu_render_views, include/crgpu.h).

Cases: hdr.json and venus.json at 512x512 and 1920x1080, 16 and 64 spp, at the scenes' frame bounce limits (32, 25), with
V = 1, 4, 16, 64 cameras on an orbit around the scene camera's target.  Per case, in one process and alternated, three runs of:
  views   one crgpu_render_views over the whole image of all V views
  single  V x (crgpu_scene_set_camera, crgpu_render_tiles over the whole image)
each from zeroed framebuffers, timed by the host clock around work that ends in a device synchronise.  The per-view CRC32s of the
two ways must agree (the script fails otherwise), and both ways' kernel launch counts are recorded, with the GPU's name, power limit
and SM clock.

    python tools/views_probe.py [--out profiles/r09_views_probe.json] [--runs 3] [--scenes hdr,venus]
"""
import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "c-ray_b200"), os.path.join(ROOT, "tests")]

import crgpu  # noqa: E402
import crscene  # noqa: E402
import oracle_lib as O  # noqa: E402

SCENES = {"hdr": 32, "venus": 25}
SIZES = [(512, 512), (1920, 1080)]
SPPS = [16, 64]
VIEWS = [1, 4, 16, 64]


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return dict(zip(q.split(","), [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")])) if r.returncode == 0 else {}


def orbit(doc, W, H, n):
    """n cameras: the scene camera's position turned about the vertical axis through the point it looks at (its focal distance
    ahead), in steps of 360 / n degrees; camera 0 is the scene camera's transform chain as written."""
    flat = crscene.load_json_buf(json.dumps(dict(doc, scene={"meshes": [], "primitives": []})))
    crgpu.lib().crscene_set_config(C.byref(flat), W, H, 0, 0)
    cam0 = crgpu.Camera.from_buffer_copy(flat.camera)
    crscene.free(flat)
    out = [cam0]
    A = np.array(cam0.A, dtype=np.float64).reshape(4, 4)
    pos, fwd = A[:3, 3], np.array(cam0.forward, dtype=np.float64)
    target = pos + fwd * max(1e-3, float(cam0.focal_distance))
    for k in range(1, n):
        a = 2.0 * math.pi * k / n
        c, s = math.cos(a), math.sin(a)
        R = np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])
        cam = crgpu.Camera.from_buffer_copy(cam0)
        M = np.eye(4)
        M[:3, :3] = R @ A[:3, :3]
        M[:3, 3] = target + R @ (pos - target)
        cam.A[:] = [float(x) for x in M.reshape(-1)]
        for f in ("forward", "right", "up"):
            getattr(cam, f)[:] = [float(x) for x in R @ np.array(getattr(cam0, f), dtype=np.float64)]
        out.append(cam)
    return out


def crcs(imgs):
    return ["%08x" % zlib.crc32(x.tobytes()) for x in imgs]


def run_views(g, V, rects):
    for v in range(V):
        g.view_clear(v)
    t = time.perf_counter()
    st = g.render_views(rects)
    ms = (time.perf_counter() - t) * 1e3
    return ms, st["kernel_launches"], [g.view_read(v) for v in range(V)]


def run_single(g, cams, rects):
    imgs, launches, ms = [], 0, 0.0
    for cam in cams:
        g.set_camera(cam)
        g.clear()
        t = time.perf_counter()
        st = g.render_tiles(rects)
        ms += (time.perf_counter() - t) * 1e3
        launches += st["kernel_launches"]
        imgs.append(g.read().copy())
    g.set_camera(cams[0])
    return ms, launches, imgs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r09_views_probe.json"))
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--scenes", default=",".join(SCENES), help="comma-separated subset of " + ", ".join(SCENES))
    args = ap.parse_args()
    info = gpu_info()
    print(json.dumps(info), flush=True)
    tmp = os.path.join(os.environ.get("TMPDIR", "/tmp"), "views_probe")
    os.makedirs(tmp, exist_ok=True)
    cases = []
    for name in args.scenes.split(","):
        bounces = SCENES[name]
        doc = json.load(open(os.path.join(ROOT, "oracle", "_ref", "input", name + ".json")))
        path = O.bundled_scene(name, tmp)
        for W, H in SIZES:
            for spp in SPPS:
                g = crgpu.GpuScene(path, W, H, spp, bounces)
                rects = [(0, 0, W, H)]
                cams_all = orbit(doc, W, H, max(VIEWS))
                for V in VIEWS:
                    cams = cams_all[:: max(VIEWS) // V][:V]
                    g.set_views(cams)
                    run_views(g, V, rects)                  # warm: the wave buffers, the pixel list, the kernels
                    tv, ts = [], []
                    for _ in range(args.runs):
                        ms, lv, iv = run_views(g, V, rects)
                        tv.append(ms)
                        ms, ls, isg = run_single(g, cams, rects)
                        ts.append(ms)
                        cv, cs = crcs(iv), crcs(isg)
                        assert cv == cs, (name, W, H, spp, V, cv, cs)
                    rec = {"scene": name, "W": W, "H": H, "spp": spp, "bounces": bounces, "views": V,
                           "views_ms": [round(x, 2) for x in tv], "single_ms": [round(x, 2) for x in ts],
                           "speedup_median": round(float(np.median(ts)) / float(np.median(tv)), 3),
                           "views_launches": lv, "single_launches": ls, "view_crc32": cv}
                    print(json.dumps({k: rec[k] for k in rec if k != "view_crc32"}), flush=True)
                    cases.append(rec)
                    write(args.out, info, args.runs, cases)
                g.close()
    print("wrote", args.out)


def write(out, info, runs, cases):
    res = {"gpu": info, "runs": runs, "timing": "host clock around calls that end in a device synchronise (ms)", "cases": cases}
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    with open(out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
