#!/usr/bin/env python3
"""Time the traversal kernel's (K2) launch variants and ray orders on the benchmark frame, bounce by bounce.

Every variant is a set of CRGPU_TRACE_* environment values.  The library reads them once per process, so each run is a
process of its own.  Variants are alternated (run 1 of every variant, then run 2 of every variant, ...), so that a drift of
the card's clock shows as spread inside a variant and not as a difference between variants.

One run renders the frame bench.py measures (hdr.json through this repository's loader, 1920x1080, 1000 spp, 32 bounces,
the dispatcher's 64-pixel tile grid, one GPU) and reports:
  frame_ms        the untimed frame path (two wave sets, no per-kernel events): host clock around a synchronous render,
                  best of --frames after one warm-up frame
  trace_ms/shade_ms per bounce, summed over the batches of one frame rendered with CRGPU_FLAG_TIME_KERNELS and
                  CRGPU_DUMP_TIMES=2: trace = K2; shade = K4 + K3 + (when a sort is on) the K4b sort of the next bounce
  crc             CRC-32 of the untimed frame: every variant must render the same bits

  python tools/k2_order_sweep.py --out k2_sweep.json --reps 2 default SORT=1 SORT=4,MINB=2
A variant is "default" or comma-separated NAME=VALUE pairs; NAME is the part after CRGPU_TRACE_ (SORT, MINB, DEFER, ...).
"""
import argparse
import json
import os
import re
import subprocess
import sys
import threading
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DUMP = re.compile(r"crgpu: batch (\d+) depth (\d+) trace ([0-9.]+) ms shade ([0-9.]+) ms")


def one(args):
    """child: render the frame under the environment it was started with; print one JSON line"""
    sys.path.insert(0, os.path.join(ROOT, "c-ray_b200"))
    import crgpu
    import crhost
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
    rays = st["rays"]
    g.clear()
    sys.stderr.flush()
    prof = g.render_tiles(rects, flags=crgpu.FLAG_TIME_KERNELS)
    g.close()
    R.close()
    print(json.dumps({"frame_ms": min(times), "frame_ms_all": [round(t, 1) for t in times], "rays": rays, "crc": f"{crc:08x}",
                      "trace_ms": prof["trace_ms"], "shade_ms": prof["shade_ms"], "timed_total_ms": prof["total_ms"]}))


def env_of(variant):
    env = dict(os.environ)
    env["CRGPU_DUMP_TIMES"] = "2"
    if variant != "default":
        for kv in variant.split(","):
            k, v = kv.split("=")
            env["CRGPU_TRACE_" + k] = v
    return env


class Clocks(threading.Thread):
    """SM clock while the runs go on, through NVML (no nvidia-smi process per sample)"""

    def __init__(self):
        super().__init__(daemon=True)
        self.sm, self.stop, self.nv, self.info = [], False, None, {}
        try:
            import pynvml
            pynvml.nvmlInit()
            self.nv = pynvml
            vis = os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]
            self.h = pynvml.nvmlDeviceGetHandleByIndex(int(vis) if vis.strip().isdigit() else 0)
            name = pynvml.nvmlDeviceGetName(self.h)
            self.info = {"name": name.decode() if isinstance(name, bytes) else name,
                         "power_limit_w": pynvml.nvmlDeviceGetEnforcedPowerLimit(self.h) / 1000.0,
                         "sm_max_mhz": pynvml.nvmlDeviceGetMaxClockInfo(self.h, pynvml.NVML_CLOCK_SM)}
        except Exception as e:   # noqa: BLE001
            self.info = {"nvml_error": str(e)[:200]}

    def run(self):
        while self.nv and not self.stop:
            try:
                self.sm.append(self.nv.nvmlDeviceGetClockInfo(self.h, self.nv.NVML_CLOCK_SM))
            except Exception:   # noqa: BLE001
                pass
            time.sleep(0.2)

    def take(self):
        s, self.sm = sorted(self.sm), []
        return {"sm_mhz_median": s[len(s) // 2], "sm_mhz_min": s[0], "sm_mhz_max": s[-1]} if s else {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("variants", nargs="*", default=["default"])
    ap.add_argument("--out", required=True, help="JSON file to write")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--frames", type=int, default=2, help="untimed frames per run after the warm-up frame")
    ap.add_argument("--scene", default="hdr")
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--spp", type=int, default=1000)
    ap.add_argument("--bounces", type=int, default=32)
    ap.add_argument("--one", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.one:
        one(args)
        return
    clocks = Clocks()
    clocks.start()
    runs = []
    child = [sys.executable, os.path.abspath(__file__), "--one", "--out", "-", "--frames", str(args.frames), "--scene", args.scene,
             "--width", str(args.width), "--height", str(args.height), "--spp", str(args.spp), "--bounces", str(args.bounces)]
    for rep in range(args.reps):
        for v in args.variants:
            clocks.take()
            r = subprocess.run(child, env=env_of(v), stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=900)
            rec = {"variant": v, "rep": rep, "clocks": clocks.take()}
            if r.returncode != 0 or not r.stdout.strip():
                rec["error"] = f"rc={r.returncode} " + r.stderr[-600:]
            else:
                rec.update(json.loads(r.stdout.strip().splitlines()[-1]))
                per = {}
                for m in DUMP.finditer(r.stderr):
                    d = per.setdefault(int(m.group(2)), [0.0, 0.0])
                    d[0] += float(m.group(3))
                    d[1] += float(m.group(4))
                rec["per_bounce"] = {str(d): [round(a, 2), round(b, 2)] for d, (a, b) in sorted(per.items())}
            runs.append(rec)
            print(json.dumps({k: rec.get(k) for k in ("variant", "rep", "frame_ms", "trace_ms", "shade_ms", "crc", "error")}), flush=True)
    clocks.stop = True
    summary = {}
    for v in args.variants:
        ok = [r for r in runs if r["variant"] == v and "error" not in r]
        if not ok:
            continue
        fm = sorted(r["frame_ms"] for r in ok)
        pb = {}
        for r in ok:
            for d, (a, b) in r["per_bounce"].items():
                pb.setdefault(d, []).append((a, b))
        summary[v] = {"frame_ms_min": round(fm[0], 1), "frame_ms_max": round(fm[-1], 1), "crcs": sorted({r["crc"] for r in ok}),
                      "trace_ms": [round(r["trace_ms"], 1) for r in ok], "shade_ms": [round(r["shade_ms"], 1) for r in ok],
                      "per_bounce_trace_shade_ms_mean": {d: [round(sum(x[0] for x in l) / len(l), 2), round(sum(x[1] for x in l) / len(l), 2)]
                                                         for d, l in sorted(pb.items(), key=lambda t: int(t[0]))}}
    out = {"card": clocks.info, "workload": f"{args.scene} {args.width}x{args.height} {args.spp} spp {args.bounces} bounces",
           "reps": args.reps, "frames_per_run": args.frames, "summary": summary, "runs": runs}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    for v, s in summary.items():
        print(f"{v:40s} frame {s['frame_ms_min']:8.1f}..{s['frame_ms_max']:8.1f} ms  trace {s['trace_ms']}  shade {s['shade_ms']}  crc {s['crcs']}")


if __name__ == "__main__":
    main()
