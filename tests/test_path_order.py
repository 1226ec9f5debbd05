"""The path order of a batch (CRGPU_PATH_ORDER, c-ray_b200/csrc/crgpu_wave.cuh): which (pass, pixel) pair every path id renders.

CPU: the map and its inverse, through the host entry point crgpu_path_order_map, exhaustively over a grid of batch shapes (one
pixel or pass, primes, shapes that are not multiples of the pass group or the pixel block, the benchmark's edge tiles), and the
blocked pixel order of rectangles.  GPU: frames rendered under every order must be the default order's bits, for a rectangle,
a tile list, several pieces, an armed call that is stopped and resumed at a pass boundary, and a snapshot.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import crgpu
import oracle_lib as O
from conftest import GOLDEN, ROOT

ORDERS = range(8)
# (P passes per group, Q pixels per block, blocked pixels) of each CRGPU_PATH_ORDER value
SHAPE = {0: (1, 32, False), 1: (1, 32, True), 2: (8, 4, True), 3: (4, 8, True), 4: (2, 16, True), 5: (8, 4, False),
         6: (16, 2, True), 7: (32, 1, True)}
NPIX = [1, 2, 3, 4, 5, 7, 8, 13, 31, 32, 33, 37, 63, 64, 97, 3584, 4096, 4099]
PASSES = [1, 2, 3, 4, 5, 7, 8, 9, 13, 16, 17]


def path_map(order, npix, passes):
    n = npix * passes
    pl, px, inv = (np.full(n, 0xffffffff, dtype=np.uint32) for _ in range(3))
    rc = crgpu.lib().crgpu_path_order_map(order, npix, passes, pl.ctypes.data, px.ctypes.data, inv.ctypes.data, 0, 0, None)
    assert rc == 0
    return pl, px, inv


def pixel_order(order, w, h):
    xy = np.full(w * h, 0xffffffff, dtype=np.uint32)
    assert crgpu.lib().crgpu_path_order_map(order, 1, 1, None, None, None, w, h, xy.ctypes.data) == 0
    return (xy & 0xffff).astype(np.int64), (xy >> 16).astype(np.int64)


@pytest.mark.parametrize("order", ORDERS)
def test_path_map_is_a_bijection_with_its_inverse(order):
    for npix in NPIX:
        for passes in PASSES:
            pl, px, inv = path_map(order, npix, passes)
            assert (pl < passes).all() and (px < npix).all(), (npix, passes)
            key = pl.astype(np.int64) * npix + px
            assert np.array_equal(np.sort(key), np.arange(npix * passes)), (npix, passes)
            assert np.array_equal(inv[key], np.arange(npix * passes, dtype=np.uint32)), (npix, passes)


def test_order_zero_is_pass_major():
    for npix in NPIX:
        for passes in PASSES:
            pl, px, inv = path_map(0, npix, passes)
            ids = np.arange(npix * passes)
            assert np.array_equal(pl, ids // npix) and np.array_equal(px, ids % npix)
            assert np.array_equal(inv, ids)


@pytest.mark.parametrize("order", [2, 3, 4, 5, 6, 7])
def test_a_warp_of_paths_covers_p_passes_of_q_pixels(order):
    """Where the batch holds whole pass groups and pixel blocks, every aligned run of 32 path ids is P passes of Q consecutive
    pixels, and the pixels' passes stay in the group of their pass."""
    P, Q, _ = SHAPE[order]
    npix, passes = 4096, 3 * P
    pl, px, _ = path_map(order, npix, passes)
    for w in range(0, npix * passes, 32 * 37):
        run_p, run_x = pl[w:w + 32], px[w:w + 32]
        assert len(set(run_p.tolist())) == P and len(set(run_x.tolist())) == Q
        assert run_x.min() % Q == 0 and run_x.max() == run_x.min() + Q - 1
        assert run_p.min() % P == 0 and run_p.max() == run_p.min() + P - 1


@pytest.mark.parametrize("order", ORDERS)
def test_pixel_order_is_a_bijection_of_the_rectangle(order):
    for w in (1, 2, 3, 7, 8, 9, 17, 56, 64, 65):
        for h in (1, 3, 4, 5, 8, 13, 56, 64):
            x, y = pixel_order(order, w, h)
            assert (x < w).all() and (y < h).all()
            assert np.array_equal(np.sort(y * w + x), np.arange(w * h)), (w, h)
            if not SHAPE[order][2]:
                assert np.array_equal(y * w + x, np.arange(w * h))


def test_blocked_pixel_order_walks_squares():
    """In the blocked order 4, 8, 16 and 32 aligned consecutive pixels of a 64x56 tile are 2x2, 4x2, 4x4 and 8x4 squares."""
    x, y = pixel_order(1, 64, 56)
    for run, (bw, bh) in ((4, (2, 2)), (8, (4, 2)), (16, (4, 4)), (32, (8, 4))):
        for s in range(0, 64 * 56, run):
            rx, ry = x[s:s + run], y[s:s + run]
            assert rx.max() - rx.min() == bw - 1 and ry.max() - ry.min() == bh - 1
            assert rx.min() % bw == 0 and ry.min() % bh == 0


def test_path_order_map_rejects_bad_arguments():
    L = crgpu.lib()
    assert L.crgpu_path_order_map(-1, 4, 4, None, None, None, 0, 0, None) == -3
    assert L.crgpu_path_order_map(8, 4, 4, None, None, None, 0, 0, None) == -3
    assert L.crgpu_path_order_map(0, 1 << 20, 1 << 13, None, None, None, 0, 0, None) == -3
    assert L.crgpu_path_order_map(0, 4, 4, None, None, None, 70000, 1, None) == -3


# ---- GPU -----------------------------------------------------------------------------------------------------------------------

_FRAME_CODE = r"""
import hashlib, json, sys
sys.path[:0] = sys.argv[1:3]
import numpy as np, crgpu
def h(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
out = {}
for name, path, W, H, spp, b in json.loads(sys.argv[3]):
    g = crgpu.GpuScene(path, W, H, spp, b)
    W, H, spp = g.W, g.H, g.samples
    g.set_max_paths(max(1024, W * H * 3))             # batches of 3 passes: pass groups cut short, two wave sets
    g.render_tile(0, 0, W, H)
    out[name + "/frame"] = h(g.read())
    g.clear()
    g.render_tile(3, 1, W - 2, H - 6)                 # a rectangle of odd width and height
    out[name + "/rect"] = h(g.read())
    g.clear()
    rects = [(x, y, min(x + 37, W), min(y + 29, H)) for y in range(0, H, 29) for x in range(0, W, 37)]
    g.render_tiles(rects)                             # a tile list with edge tiles
    out[name + "/tiles"] = h(g.read())
    g.set_max_paths(5000)                             # pieces: rows of the rectangle, ranges of the list
    g.clear()
    g.render_tile(0, 0, W, H, pass_count=min(5, spp))
    out[name + "/pieces"] = h(g.read())
    g.clear()
    g.render_tiles(rects, pass_count=min(5, spp))
    out[name + "/pieces_tiles"] = h(g.read())
    g.set_max_paths(max(1024, W * H * 3))
    g.enable_stop()                                   # armed: a call stopped at its first boundary, resumed in two calls
    g.clear()
    g.request_stop()
    st = g.render_tile(0, 0, W, H)
    assert st["stopped"] and g.progress() == (0, False)
    g.clear_stop()
    g.render_tile(0, 0, W, H, pass_begin=0, pass_count=spp // 2)
    g.render_tile(0, 0, W, H, pass_begin=spp // 2)
    assert g.progress() == (spp, False)
    out[name + "/resumed"] = h(g.read())
    g.clear()
    g.request_snapshot()                              # staged by the first publish step: passes [0, 3)
    g.render_tiles(rects)
    img, done = g.take_snapshot()
    out[name + "/snapshot"] = h(img) + " %d" % done
    out[name + "/armed_tiles"] = h(g.read())
    g.close()
print("FRAMES " + json.dumps(out))
"""


def _frames(env, jobs):
    e = {k: v for k, v in os.environ.items() if not k.startswith("CRGPU_")}
    e.update(env)
    r = subprocess.run([sys.executable, "-c", _FRAME_CODE, os.path.join(ROOT, "c-ray_b200"), os.path.join(ROOT, "tests"), json.dumps(jobs)],
                       env=e, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("FRAMES ")]
    assert r.returncode == 0 and lines, r.stdout[-2000:]
    return json.loads(lines[-1][7:])


@pytest.mark.gpu
def test_every_path_order_renders_the_default_frame(tmp_path):
    """Every CRGPU_PATH_ORDER renders the default order's bits: g_nodes and g_f4 (the complete interpreter) at their own sizes, and
    hdr at 240x135, 16 spp, 32 bounces, for a whole rectangle, an odd rectangle, a tile list, pieces of both, an armed call
    stopped and resumed at a pass boundary, and a snapshot."""
    jobs = [["g_nodes", os.path.join(GOLDEN, "g_nodes.crscene"), 0, 0, 0, 0], ["g_f4", os.path.join(GOLDEN, "g_f4.crscene"), 0, 0, 0, 0]]
    hdr = O.bundled_scene("hdr", str(tmp_path))
    if hdr:
        jobs.append(["hdr", hdr, 240, 135, 16, 32])
    base = _frames({}, jobs)
    assert len(base) == 8 * len(jobs)
    bad = []
    for order in ORDERS:
        got = _frames({"CRGPU_PATH_ORDER": str(order)}, jobs)
        bad += [(order, k) for k in base if got[k] != base[k]]
    assert not bad, bad
