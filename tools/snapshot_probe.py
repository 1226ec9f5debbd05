"""What reading the image of a running render costs and how fast it arrives (crgpu_request_snapshot / crgpu_take_snapshot,
include/crgpu.h), on one GPU.

1. Overhead: bench.py's frame (hdr.json 1920x1080, 1000 spp, 32 bounces) and the same scene at 8K (7680x4320, each snapshot
   about 100 MB; 100 spp so that a frame takes seconds, not minutes), rendered armed without snapshots and armed with a snapshot
   taken at every commit (another thread requests the next one as soon as it has taken the last), alternated.  Each run reports
   the frame time, the frame CRC (equal in both modes), the kernel launches (equal in both modes) and the snapshots taken.
2. Latency: from crgpu_request_snapshot to the image in host memory, requested at 10%, 50% and 90% of each frame.
3. With --parent LIB: the armed bench frame without snapshots through this build and through another build of libcrgpu.so (the
   one whose publish step is a one-thread kernel), each in its own child process, alternated.
4. The card, its power limit and the SM clock, in the same run (nvidia-smi queries, read only).

    python tools/snapshot_probe.py [--runs 3] [--parent LIB] [--out profiles/r05_snapshot_probe.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import threading
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "c-ray_b200"), os.path.join(ROOT, "tests")]

import crgpu  # noqa: E402
import oracle_lib as O  # noqa: E402

# name -> (W, H, spp, bounces)
FRAMES = {"hdr": (1920, 1080, 1000, 32), "hdr8k": (7680, 4320, 100, 32)}


def smi(fields):
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader"], stdout=subprocess.PIPE, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unavailable: {e}"


class Snapper:
    """takes snapshots of g's calls on its own thread into one preallocated buffer: at every commit, or once at a given time"""

    def __init__(self, g):
        self.g = g
        self.buf = np.empty((g.H, g.W, 3), dtype=np.uint8)
        self.L = crgpu.lib()

    def take(self, stop=None):
        """request, then poll until the image is in host memory; returns its pass index, or None when stopped first"""
        self.g.request_snapshot()
        k = C.c_int(0)
        while stop is None or not stop.is_set():
            rc = self.L.crgpu_take_snapshot(self.g.handle, self.buf.ctypes.data, C.byref(k))
            if rc == 0:
                return k.value
            if rc != crgpu.PENDING:
                raise crgpu.CrgpuError(f"crgpu_take_snapshot failed ({rc})")
            time.sleep(0.0001)
        return None


def frame(g, snap):
    """one armed frame, synchronous; with snap, snapshots at every commit.  (ms, crc, launches, snapshots taken)"""
    g.clear()
    stop, taken = threading.Event(), []
    s = Snapper(g)

    def loop():
        while not stop.is_set():
            k = s.take(stop)
            if k is not None:
                taken.append(k)

    th = threading.Thread(target=loop) if snap else None
    if th:
        th.start()
    t0 = time.perf_counter()
    st = g.render_tile(0, 0, g.W, g.H)
    ms = 1e3 * (time.perf_counter() - t0)
    stop.set()
    if th:
        th.join()
        s.take()            # a request the loop left behind: answered from the framebuffer, so no image stays staged
    return ms, zlib.crc32(g.read().tobytes()), st["kernel_launches"], len(taken)


def child(lib):
    """one armed bench frame without snapshots through the library at `lib`, after a warm-up frame; prints one JSON line"""
    crgpu.LIB_PATH = lib
    g = crgpu.GpuScene(O.bundled_scene("hdr", tempfile.mkdtemp()), *FRAMES["hdr"])
    g.enable_stop()
    frame(g, False)
    ms, crc, launches, _ = frame(g, False)
    print(json.dumps({"ms": round(ms, 1), "crc32": f"{crc:08x}", "launches": launches}), flush=True)


def armed_vs_parent(parent, runs):
    env = {k: v for k, v in os.environ.items() if not k.startswith("CRGPU_")}
    recs = []
    for i in range(runs):
        for name, lib in (("parent", os.path.abspath(parent)), ("this", crgpu.LIB_PATH)):
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", lib], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                               text=True, env=env, timeout=600)
            line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
            if r.returncode != 0 or not line:
                raise RuntimeError(r.stdout[-3000:])
            rec = dict(json.loads(line[-1]), build=name, run=i)
            recs.append(rec)
            print(rec, flush=True)
    return recs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--parent", default=None, help="another build of libcrgpu.so to compare the armed frame with")
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if args.child:
        child(args.child)
        return
    tmp = tempfile.mkdtemp()
    out = {"card": smi("name,power.limit,clocks.sm,clocks.max.sm"), "frames": {n: "%dx%d %d spp %d bounces" % c for n, c in FRAMES.items()},
           "overhead": [], "latency": []}
    if args.parent:
        out["armed_vs_parent"] = armed_vs_parent(args.parent, args.runs)
    path = O.bundled_scene("hdr", tmp)
    for name, cfg in FRAMES.items():
        g = crgpu.GpuScene(path, *cfg)
        g.enable_stop()
        frame(g, False)                                            # warm-up: allocation, first launches
        frame(g, True)
        T = []
        for i in range(args.runs):
            for snap in (False, True):
                ms, crc, launches, n = frame(g, snap)
                T.append(ms)
                rec = {"frame": name, "run": i, "snapshots": snap, "ms": round(ms, 1), "crc32": f"{crc:08x}", "launches": launches, "taken": n}
                out["overhead"].append(rec)
                print(rec, flush=True)
        Tm = sum(T) / len(T)
        s = Snapper(g)
        for frac in (0.1, 0.5, 0.9):
            g.clear()
            # the render on a thread of its own: enqueueing thousands of launches blocks once the launch queue is full
            th = threading.Thread(target=g.render_tile, args=(0, 0, g.W, g.H))
            t0 = time.perf_counter()
            th.start()
            while time.perf_counter() - t0 < frac * Tm / 1e3:
                time.sleep(0.0005)
            t_req = time.perf_counter()
            k = s.take()
            lat = 1e3 * (time.perf_counter() - t_req)
            busy_after = g.progress()[1]
            th.join()
            rec = {"frame": name, "at": frac, "latency_ms": round(lat, 2), "passes_shown": k, "call_still_running": bool(busy_after)}
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
