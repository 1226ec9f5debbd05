"""What adaptive sampling saves (crgpu_adaptive_round, include/crgpu.h), against the fixed frame and a uniform frame of the same paths.

Workloads: hdr.json at 1920x1080, 1000 spp, 32 bounces (bench.py's default) and venus.json at 2560x1600, 1000 spp, 25 bounces (its
BASELINE configuration), each one resident scene with the default paths-in-flight budget and the whole image as one tile.
For each workload and repetition (the repetitions alternate the order of the runs):
  fixed        render_tiles(0, spp) from a cleared framebuffer: the wall time, and the frame every RMSE below is taken against
  adaptive T   for T = 0.1, 0.05, 0.02, 0.01 (min_passes 16, round_passes 16, floor 0.01: the CLI's defaults): reset, then rounds
               until no pixel is active; wall time, paths, mean passes per pixel, rounds, and the RMSE of the frame
  uniform T    render_tiles(0, P) with P = the adaptive run's paths / pixels, rounded: the same budget spread evenly, and its RMSE
  select       the wall time of one round that finds no active pixel (a select over the whole tile set and its readback: the fixed
               cost every round pays before it renders), median of 5, after each adaptive run
RMSE is over every channel of every pixel.  The adaptive and uniform frames are prefixes of the fixed frame's sample sequence (a
pixel's passes are seeded by pixel, pass and sample count only), so both RMSEs understate the error against an independent
reference by the same token.  Wall times are host clocks around synchronous calls.

    python tools/adaptive_probe.py [--reps 2] [--out profiles/r12_adaptive_probe.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "c-ray_b200"), os.path.join(ROOT, "tests")]

import crgpu  # noqa: E402
import oracle_lib as O  # noqa: E402

WORKLOADS = [("hdr", 1920, 1080, 1000, 32), ("venus", 2560, 1600, 1000, 25)]
THRESHOLDS = [0.1, 0.05, 0.02, 0.01]
MIN_PASSES, ROUND_PASSES, FLOOR = 16, 16, 0.01


def rmse(a, b):
    d = a.astype(np.float64) - b.astype(np.float64)
    return float(np.sqrt(np.mean(d * d)))


def timed(fn):
    t = time.perf_counter()
    r = fn()
    return time.perf_counter() - t, r


def fixed(g, rects, passes):
    g.clear()
    t, st = timed(lambda: g.render_tiles(rects, 0, passes))
    return t, st, g.read().copy()


def adaptive(g, rects, thr):
    def run():
        g.clear()
        g.adaptive_reset()
        return g.render_adaptive(rects, MIN_PASSES, ROUND_PASSES, thr, FLOOR)
    t, st = timed(run)
    img = g.read().copy()
    n, _ = g.adaptive_read()
    empty = []
    for _ in range(5):
        te, d = timed(lambda: g.adaptive_round(rects, MIN_PASSES, ROUND_PASSES, thr, FLOOR))
        assert d["active"] == 0
        empty.append(te)
    return t, st, img, n, float(np.median(empty))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r12_adaptive_probe.json"))
    ap.add_argument("--small", action="store_true", help="tiny sizes: a rehearsal of the script, not a measurement")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
    out = {"gpu": gpu[0] if gpu else "unknown", "rule": dict(min_passes=MIN_PASSES, round_passes=ROUND_PASSES, floor=FLOOR),
           "workloads": []}
    tmp = tempfile.mkdtemp()
    for name, W, H, spp, b in WORKLOADS:
        if args.small:
            W, H, spp = W // 16, H // 16, 64
        g = crgpu.GpuScene(O.bundled_scene(name, tmp), W, H, spp, b)
        rects = [(0, 0, W, H)]
        fixed(g, rects, min(spp, 16))                                  # warm-up: modules, wave buffers, pixel list
        reps = []
        ref = None
        for rep in range(args.reps):
            runs = {"fixed": None, "adaptive": []}
            order = [None] + THRESHOLDS if rep % 2 == 0 else THRESHOLDS[::-1] + [None]
            results = {}
            for thr in order:
                if thr is None:
                    t, st, img = fixed(g, rects, spp)
                    ref = img if ref is None else ref
                    assert img.tobytes() == ref.tobytes()
                    runs["fixed"] = {"wall_s": t, "paths": st["paths"]}
                else:
                    results[thr] = adaptive(g, rects, thr)
            for thr in THRESHOLDS:
                t, st, img, n, empty = results[thr]
                mean_passes = float(n.mean())
                P = max(1, int(round(st["paths"] / (W * H))))
                tu, _, uimg = fixed(g, rects, P)
                runs["adaptive"].append({
                    "threshold": thr, "wall_s": t, "paths": st["paths"], "mean_passes": mean_passes, "rounds": st["rounds"],
                    "pixels_at_min_passes": int((n == MIN_PASSES).sum()), "pixels_at_spp": int((n == spp).sum()),
                    "select_readback_ms_per_round": 1e3 * empty, "rmse": rmse(img, ref),
                    "uniform": {"passes": P, "paths": P * W * H, "wall_s": tu, "rmse": rmse(uimg, ref)}})
            reps.append(runs)
            print(json.dumps({"workload": name, "rep": rep, **runs}, indent=1), flush=True)
        out["workloads"].append({"scene": name, "width": W, "height": H, "spp": spp, "bounces": b, "reps": reps})
        g.close()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()
