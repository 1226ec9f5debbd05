"""What stopping costs and how fast it is (crgpu_stop_enable, include/crgpu.h), on one GPU.

1. Overhead: bench.py's frame (hdr.json 1920x1080, 1000 spp, 32 bounces) rendered unarmed and armed, alternated, with the frame
   CRC of each run (they must be equal: an armed frame that is never stopped is bit-identical).
2. Stop latency: from crgpu_request_stop (another thread) to the return of the call, at several points of the hdr, venus and
   refraction frames, with the passes committed at that point.
3. The card, its power limit and the SM clock (nvidia-smi queries, read only).

    python tools/stop_probe.py [--runs 3] [--out profiles/r03_stop_probe.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import threading
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "c-ray_b200"), os.path.join(ROOT, "tests")]

import crgpu  # noqa: E402
import oracle_lib as O  # noqa: E402

# name -> (W, H, spp, bounces)
FRAMES = {"hdr": (1920, 1080, 1000, 32), "venus": (2560, 1600, 1000, 25), "refraction": (1280, 720, 500, 512)}


def smi(fields):
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader"], stdout=subprocess.PIPE, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unavailable: {e}"


def timed(g):
    g.clear()
    t0 = time.perf_counter()
    st = g.render_tile(0, 0, g.W, g.H)
    ms = 1e3 * (time.perf_counter() - t0)
    return ms, zlib.crc32(g.read().tobytes()), st["kernel_launches"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    tmp = tempfile.mkdtemp()
    out = {"card": smi("name,power.limit,clocks.sm,clocks.max.sm"), "overhead": [], "latency": []}

    path = O.bundled_scene("hdr", tmp)
    g = crgpu.GpuScene(path, *FRAMES["hdr"])
    timed(g)                                                   # warm-up: allocation, first launches
    for i in range(args.runs):
        for armed in (False, True):
            g.enable_stop(armed)
            ms, crc, launches = timed(g)
            out["overhead"].append({"run": i, "armed": armed, "ms": round(ms, 2), "crc32": f"{crc:08x}", "launches": launches})
            print(out["overhead"][-1], flush=True)
    g.close()

    for name, cfg in FRAMES.items():
        path = O.bundled_scene(name, tmp)
        if not path:
            continue
        g = crgpu.GpuScene(path, *cfg)
        g.enable_stop()
        T, _, _ = timed(g)
        for frac in (0.1, 0.5, 0.9):
            g.clear_stop()
            g.clear()
            req = {}

            def stop():
                req["t"] = time.perf_counter()
                g.request_stop()

            t = threading.Timer(frac * T / 1e3, stop)
            t.start()
            st = g.render_tile(0, 0, g.W, g.H)
            t_end = time.perf_counter()
            t.join()
            done = g.progress()[0]
            rec = {"scene": name, "config": "%dx%d %d spp %d bounces" % cfg, "frame_ms": round(T, 1), "at": frac,
                   "latency_ms": round(1e3 * (t_end - req["t"]), 2) if "t" in req else None, "passes_done": done, "stopped": st["stopped"]}
            out["latency"].append(rec)
            print(rec, flush=True)
        g.close()
    out["card_after"] = smi("name,power.limit,clocks.sm")
    text = json.dumps(out, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
