#!/usr/bin/env python3
"""Split the benchmark frame's time by kernel launch, bounce by bounce: K1, K2, K4 and each of K3's three launches.

One run renders the frame bench.py measures (hdr.json through this repository's loader, 1920x1080, 1000 spp, 32 bounces,
the dispatcher's 64-pixel tile grid, one GPU) from one build, in a process of its own, and reports:
  frame_ms        the untimed frame path (two wave sets, no per-kernel events): host clock around a synchronous render,
                  best of --frames after one warm-up frame
  crc             CRC-32 of the untimed frame: every build must render the same bits
  k1_ms           K1 (k_generate), summed over the batches of one frame rendered with CRGPU_FLAG_TIME_KERNELS and CRGPU_DUMP_TIMES=2
  per bounce      from the same frame, summed over its batches: trace (K2), shade (K4 + K3 + the K4b sort when one is on) and
                  shade's parts: k4, miss, flat and generic (K3's three launches) and sort
A build is a repository root whose c-ray_b200/ holds a built libcrgpu.so (this tree by default), optionally followed by
:NAME=VALUE,... environment settings for that run.  Builds are alternated (run 1 of every build, then run 2, ...), so that a
drift of the card's clock shows as spread inside a build and not as a difference between builds.

  python tools/shade_split.py --out split.json --reps 2 /path/to/parent_build .
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time
import zlib

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
from k2_order_sweep import Clocks  # noqa: E402

BOUNCE = re.compile(r"crgpu: batch (\d+) depth (\d+) trace ([0-9.]+) ms shade ([0-9.]+) ms k4 ([0-9.]+) miss ([0-9.]+) flat ([0-9.]+) "
                    r"generic ([0-9.]+) sort ([0-9.]+)")
K1 = re.compile(r"crgpu: batch (\d+) k1 ([0-9.]+) ms")
PARTS = ("trace", "shade", "k4", "miss", "flat", "generic", "sort")


def one(args):
    """child: render the frame with the build at args.root; print one JSON line"""
    sys.path.insert(0, os.path.join(args.root, "c-ray_b200"))
    import crgpu
    import crhost
    assert os.path.dirname(os.path.abspath(crgpu.__file__)) == os.path.join(os.path.abspath(args.root), "c-ray_b200")
    refdir = os.path.join(ROOT, "oracle", "_ref")
    cwd = os.getcwd()
    os.chdir(refdir)                       # texture paths inside the scene resolve against the reference's input directory
    try:
        R = crhost.Renderer(os.path.join("input", args.scene + ".json"), args.width, args.height, args.spp, args.bounces, gpus=1, tile=64, quiet=True)
    finally:
        os.chdir(cwd)
    R.join(None, 0, 1, 0)
    R.prepare()
    rects, _, _ = R.rank_tiles(0, 1)
    g = crgpu.GpuScene(None, samples=args.spp, bounces=args.bounces, device=0, prepared=R.prepared())
    times = []
    st = None
    for i in range(1 + args.frames):
        g.clear()
        t0 = time.perf_counter()
        st = g.render_tiles(rects)           # synchronous: returns after the device finished the frame
        if i:
            times.append(1e3 * (time.perf_counter() - t0))
    crc = zlib.crc32(g.read().tobytes())
    g.clear()
    sys.stderr.flush()
    prof = g.render_tiles(rects, flags=crgpu.FLAG_TIME_KERNELS)
    g.close()
    R.close()
    print(json.dumps({"frame_ms": min(times), "frame_ms_all": [round(t, 1) for t in times], "rays": st["rays"], "crc": f"{crc:08x}",
                      "trace_ms": prof["trace_ms"], "shade_ms": prof["shade_ms"], "timed_total_ms": prof["total_ms"]}))


def parse(build):
    root, _, env = build.partition(":")
    e = dict(os.environ)
    e["CRGPU_DUMP_TIMES"] = "2"
    for kv in filter(None, env.split(",")):
        k, v = kv.split("=")
        e[k] = v
    return os.path.abspath(root), e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("builds", nargs="*", default=["."])
    ap.add_argument("--out", required=True, help="JSON file to write")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--frames", type=int, default=2, help="untimed frames per run after the warm-up frame")
    ap.add_argument("--scene", default="hdr")
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--spp", type=int, default=1000)
    ap.add_argument("--bounces", type=int, default=32)
    ap.add_argument("--root", default=ROOT, help=argparse.SUPPRESS)
    ap.add_argument("--one", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.one:
        one(args)
        return
    clocks = Clocks()
    clocks.start()
    runs = []
    for rep in range(args.reps):
        for b in args.builds:
            root, env = parse(b)
            child = [sys.executable, os.path.abspath(__file__), "--one", "--out", "-", "--root", root, "--frames", str(args.frames),
                     "--scene", args.scene, "--width", str(args.width), "--height", str(args.height), "--spp", str(args.spp),
                     "--bounces", str(args.bounces)]
            clocks.take()
            r = subprocess.run(child, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=900)
            rec = {"build": b, "rep": rep, "clocks": clocks.take()}
            if r.returncode != 0 or not r.stdout.strip():
                rec["error"] = f"rc={r.returncode} " + r.stderr[-600:]
            else:
                rec.update(json.loads(r.stdout.strip().splitlines()[-1]))
                rec["k1_ms"] = round(sum(float(m.group(2)) for m in K1.finditer(r.stderr)), 2)
                per = {}
                for m in BOUNCE.finditer(r.stderr):
                    d = per.setdefault(int(m.group(2)), [0.0] * len(PARTS))
                    for k in range(len(PARTS)):
                        d[k] += float(m.group(3 + k))
                rec["per_bounce"] = {str(d): [round(x, 2) for x in v] for d, v in sorted(per.items())}
            runs.append(rec)
            print(json.dumps({k: rec.get(k) for k in ("build", "rep", "frame_ms", "k1_ms", "trace_ms", "shade_ms", "crc", "error")}), flush=True)
    clocks.stop = True
    summary = {}
    for b in args.builds:
        ok = [r for r in runs if r["build"] == b and "error" not in r]
        if not ok:
            continue
        pb = {}
        for r in ok:
            for d, v in r["per_bounce"].items():
                pb.setdefault(d, []).append(v)
        mean = {d: [round(sum(x[k] for x in l) / len(l), 2) for k in range(len(PARTS))] for d, l in sorted(pb.items(), key=lambda t: int(t[0]))}
        total = [round(sum(v[k] for v in mean.values()), 1) for k in range(len(PARTS))]
        fm = sorted(r["frame_ms"] for r in ok)
        summary[b] = {"frame_ms_min": round(fm[0], 1), "frame_ms_max": round(fm[-1], 1), "crcs": sorted({r["crc"] for r in ok}),
                      "k1_ms": [r["k1_ms"] for r in ok], "columns": list(PARTS), "total_ms_mean": total, "per_bounce_ms_mean": mean}
    out = {"card": clocks.info, "workload": f"{args.scene} {args.width}x{args.height} {args.spp} spp {args.bounces} bounces",
           "reps": args.reps, "frames_per_run": args.frames, "summary": summary, "runs": runs}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(clocks.info))
    for b, s in summary.items():
        print(f"{b}: frame {s['frame_ms_min']:.1f}..{s['frame_ms_max']:.1f} ms  k1 {s['k1_ms']}  crc {s['crcs']}")
        print("  depth " + " ".join(f"{c:>8s}" for c in PARTS))
        for d, v in s["per_bounce_ms_mean"].items():
            print(f"  {d:>5s} " + " ".join(f"{x:8.2f}" for x in v))
        print("  total " + " ".join(f"{x:8.1f}" for x in s["total_ms_mean"]))


if __name__ == "__main__":
    main()
