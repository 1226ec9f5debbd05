"""The kernels a render call enqueues, counted by stats.kernel_launches, against the schedule of DESIGN.md section 4.

Per batch: K1 and K5.  Per bounce: K2, K4 and K3's three launches, and the tail kernel from bounce 6 on (not with FLAG_COUNT).
An armed call adds one stop gate per bounce (one after K1 when bounces == 0), one publish step per pass batch, and the begin and
end steps of the call.  A call's batches are max_paths / pixels passes each, in equal shares, halved over two wave sets when they
overlap (two or more batches, without FLAG_COUNT or FLAG_TIME_KERNELS); a pixel set larger than max_paths is cut into pieces of
rows (a rectangle) or of list ranges (a tile set), walked piece by piece unarmed and pass batch by pass batch armed.

The knobs are read once per process, so the calls run in a child process with no CRGPU_* variable set, on the library this
process loaded (crgpu.LIB_PATH).  Run as a script (`python tests/test_gpu_launch_schedule.py LIB`) the module prints one JSON line
per call shape: launches, paths, rays and the framebuffer's CRC32 (tools/driver_check.py compares two libraries with it).
"""
import json
import os
import subprocess
import sys
import zlib

import pytest

W, H, SPP, BOUNCES = 64, 36, 8, 8
TAIL_FROM = 6
K3_LAUNCHES = 3
HALVES = [(0, 0, 40, H), (40, 0, W, H)]
# name -> (pixel set, max paths in flight, flags, armed, bounces, stop requested before the call)
SHAPES = {
    "fits": ("rect", 1 << 20, 0, False, BOUNCES, False),
    "overlap": ("rect", 4 * W * H, 0, False, BOUNCES, False),
    "rect_pieces": ("rect", 1024, 0, False, BOUNCES, False),
    "tiles_pieces": ("tiles", 1024, 0, False, BOUNCES, False),
    "armed_fits": ("rect", 1 << 20, 0, True, BOUNCES, False),
    "armed_overlap": ("rect", 4 * W * H, 0, True, BOUNCES, False),
    "armed_rect_pieces": ("rect", 1024, 0, True, BOUNCES, False),
    "armed_tiles_pieces": ("tiles", 1024, 0, True, BOUNCES, False),
    "no_bounces": ("rect", 4 * W * H, 0, False, 0, False),
    "armed_no_bounces": ("rect", 4 * W * H, 0, True, 0, False),
    "count": ("rect", 4 * W * H, 0x1, False, BOUNCES, False),        # FLAG_COUNT
    "time_kernels": ("rect", 4 * W * H, 0x2, False, BOUNCES, False), # FLAG_TIME_KERNELS
    "armed_stopped": ("rect", 4 * W * H, 0, True, BOUNCES, True),
    "armed_stopped_pieces": ("tiles", 1024, 0, True, BOUNCES, True),
}


def _ceil(a, b):
    return -(-a // b)


def batches(pixels, max_paths, passes, overlap):
    """the batch loop's plan: the number of batches of `passes` passes over `pixels` pixels"""
    b = max(1, max_paths // pixels)
    if overlap and 2 <= b < passes:
        b //= 2
    b = min(b, passes)
    b = _ceil(passes, _ceil(passes, b))
    return _ceil(passes, b)


def pieces(kind, max_paths):
    if kind == "rect" and W * H > max_paths:
        rows = max_paths // W
        return [W * min(rows, H - y) for y in range(0, H, rows)]
    return [min(max_paths, W * H - p) for p in range(0, W * H, max_paths)]


def per_batch(bounces, count, armed):
    n = 2 + (1 if armed and bounces == 0 else 0)
    for d in range(bounces):
        n += 2 + K3_LAUNCHES + (1 if d >= TAIL_FROM and not count else 0) + (1 if armed else 0)
    return n


def expected_launches(shape):
    kind, mp, flags, armed, bounces, stopped = SHAPES[shape]
    count, overlap = bool(flags & 0x1), not flags
    parts = pieces(kind, mp)
    if not armed:
        return sum(batches(p, mp, SPP, overlap) * per_batch(bounces, count, False) for p in parts)
    if stopped:
        return 2
    if len(parts) == 1:
        return batches(parts[0], mp, SPP, overlap) * (per_batch(bounces, count, True) + 1) + 2
    step = max(1, mp // max(parts))
    total = 2
    for pb in range(0, SPP, step):
        n = min(step, SPP - pb)
        total += sum(batches(p, mp, n, overlap) * per_batch(bounces, count, True) for p in parts) + 1
    return total


def measure(lib_path):
    """every shape on a fresh scene: one asynchronous render call, then a synchronous crgpu_get_stats"""
    import crgpu
    crgpu.LIB_PATH = lib_path
    scene = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "g_legacy.crscene")
    for name, (kind, mp, flags, armed, bounces, stopped) in SHAPES.items():
        g = crgpu.GpuScene(scene, W, H, SPP, bounces, force_bounces=bounces, max_paths=mp)
        g.get_stats()
        if armed:
            g.enable_stop()
        if stopped:
            g.request_stop()
        if kind == "rect":
            g.render_tile(0, 0, W, H, 0, SPP, flags | crgpu.FLAG_ASYNC)
        else:
            g.render_tiles(HALVES, 0, SPP, flags | crgpu.FLAG_ASYNC)
        st = g.get_stats()
        rec = {"shape": name, "kernel_launches": st["kernel_launches"], "paths": st["paths"], "rays": st["rays"],
               "crc32": "%08x" % zlib.crc32(g.read().tobytes())}
        print(json.dumps(rec), flush=True)
        g.close()


def run_child(lib_path):
    """measure(lib_path) in a child process without CRGPU_* variables; returns {shape: record}"""
    here = os.path.dirname(os.path.abspath(__file__))
    env = {k: v for k, v in os.environ.items() if not k.startswith("CRGPU_")}
    env["PYTHONPATH"] = os.pathsep.join([os.path.join(os.path.dirname(here), "c-ray_b200"), here])
    r = subprocess.run([sys.executable, os.path.abspath(__file__), lib_path], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:]
    out = {}
    for line in r.stdout.splitlines():
        if line.startswith("{"):
            rec = json.loads(line)
            out[rec["shape"]] = rec
    return out


@pytest.mark.gpu
def test_launch_counts_follow_the_schedule():
    import crgpu
    # the shapes engage what they are named for: one batch, four overlapped batches (two without overlap), three pieces
    assert batches(W * H, 1 << 20, SPP, True) == 1 and pieces("rect", 1 << 20) == [W * H]
    assert batches(W * H, 4 * W * H, SPP, True) == 4 and batches(W * H, 4 * W * H, SPP, False) == 2
    assert pieces("rect", 1024) == [1024, 1024, 256] and pieces("tiles", 1024) == [1024, 1024, 256]
    got = run_child(crgpu.LIB_PATH)
    assert sorted(got) == sorted(SHAPES)
    for name, (kind, mp, flags, armed, bounces, stopped) in SHAPES.items():
        rec = got[name]
        assert rec["kernel_launches"] == expected_launches(name), (name, rec)
        assert rec["paths"] == (0 if stopped else W * H * SPP), (name, rec)


if __name__ == "__main__":
    measure(sys.argv[1])
