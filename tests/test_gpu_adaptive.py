"""Rendering adaptively on the GPU (crgpu_adaptive_reset / _round / _read, include/crgpu.h; DESIGN §4 "Rendering adaptively").

The target is exact: a pixel that an adaptive render left at n passes holds, bit for bit, what crgpu_render_tiles(rects, 0, n) gives it
on a cleared framebuffer of a second upload, whatever the round length, the path budget, the pieces, the tile split across scenes, a
stop in between or the asynchronous flag.  Its count and error are those of the rule replayed in numpy float32 on the oracle's
per-sample radiance.

CPU: argument checks of the new entry points and of the CLI.  GPU: everything else.
"""
import ctypes as C
import hashlib
import json
import math
import os
import subprocess
import threading
import time

import numpy as np
import pytest

import crgpu
import oracle_lib as O
from conftest import GOLDEN, ROOT

DIGESTS = os.path.join(GOLDEN, "shade_frames.sha256.json")
REFDIR = os.path.join(ROOT, "oracle", "_ref")
EXE = os.path.join(ROOT, "c-ray_b200", "cray_b200")
CFG = (240, 135, 64, 0)        # W, H, spp, bounces (0: the scene's) of the exactness runs
FLOOR = 0.01


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


# ---- CPU -----------------------------------------------------------------------------------------------------------------------

def test_entry_points_reject_null_arguments():
    L = crgpu.lib()
    rect = np.array([0, 0, 1, 1], dtype=np.int32)
    a = crgpu.Adaptive(2, 1, 1, 0.1, 0.01)
    n, pb, pe = C.c_uint32(0), C.c_int(0), C.c_int(0)
    passes = np.zeros(4, dtype=np.uint32)
    assert L.crgpu_adaptive_reset(None) == -3
    assert L.crgpu_adaptive_round(None, rect.ctypes.data, 1, C.byref(a), 0, None, C.byref(n), C.byref(pb), C.byref(pe)) == -3
    assert L.crgpu_adaptive_round(None, rect.ctypes.data, 1, None, 0, None, None, None, None) == -3
    assert L.crgpu_adaptive_read(None, passes.ctypes.data, None) == -3
    assert L.crgpu_adaptive_read(None, None, None) == -3


def test_no_scene_to_adapt_without_a_device():
    """Without a GPU no scene exists to adapt: creating one fails loudly (CRGPU_ERR_NO_DEVICE), never on the CPU."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    with pytest.raises(crgpu.CrgpuError):
        crgpu.GpuScene(os.path.join(GOLDEN, "g_single.crscene")).adaptive_reset()


@pytest.mark.parametrize("value", ["-0.05", "abc", "nan", "inf", "0.1x", ""])
def test_cli_refuses_a_bad_threshold(value, tmp_path):
    """--adaptive takes a finite threshold >= 0; anything else ends the CLI with an error before it loads the scene or touches a
    device (the scene named here does not exist, so a later failure would name the scene instead)."""
    if not os.path.exists(EXE):
        pytest.skip("cray_b200 not built")
    r = subprocess.run([EXE, str(tmp_path / "missing.json"), "--adaptive", value], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=60)
    assert r.returncode == 1, r.stdout
    assert "Invalid --adaptive parameter" in r.stdout


# ---- helpers ---------------------------------------------------------------------------------------------------------------------

def scene_path(name, tmp):
    if name.startswith("g_"):
        return os.path.join(GOLDEN, name + ".crscene")
    p = O.bundled_scene(name, str(tmp))
    if not p:
        pytest.skip(f"{name} not available")
    return p


def upload(name, tmp, cfg=CFG, max_paths=None):
    return crgpu.GpuScene(scene_path(name, tmp), *cfg, max_paths=max_paths)


def grid(W, H, tw=37, th=29):
    """a tile list with edge tiles, not aligned to the 8x4 pixel blocks"""
    return [(x, y, min(x + tw, W), min(y + th, H)) for y in range(0, H, th) for x in range(0, W, tw)]


def adaptive(g, rects, rule, clear=True):
    """reset, then rounds until none is active; returns (framebuffer, counts, err, summed stats)"""
    if clear:
        g.clear()
    g.adaptive_reset()
    st = g.render_adaptive(rects, *rule)
    n, err = g.adaptive_read()
    return g.read().copy(), n, err, st


def calibrate(g, rects, min_passes, pass_end):
    """a threshold that stops about half the pixels at their first test: the median error at min_passes"""
    g.clear()
    g.adaptive_reset()
    g.adaptive_round(rects, min_passes, 16, 0.0, FLOOR, pass_end)
    g.adaptive_round(rects, min_passes, 16, 0.0, FLOOR, pass_end)     # tests every pixel at min_passes, stops none
    _, err = g.adaptive_read()
    e = err[np.isfinite(err)]
    return float(np.median(e))


def check_counts_exact(h, rects, img, n, what):
    """each pixel with count k equals render_tiles(rects, 0, k) on a cleared framebuffer of the second upload h"""
    for k in np.unique(n):
        h.clear()
        if k:
            h.render_tiles(rects, 0, int(k))
        ref = h.read()
        sel = n == k
        assert ref[sel].tobytes() == img[sel].tobytes(), f"{what}: pixels at {k} passes differ from render_tiles(0, {k})"


# ---- GPU: exactness ----------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", ["g_nodes", "hdr"])
def test_each_pixel_is_its_fixed_render(name, tmp_path):
    """Thresholds that give several counts, some pixels at min_passes and some at pass_end: each count's pixels equal the fixed
    render of that many passes, with round lengths 1, 7 and 16, and with a path budget that cuts every round into pieces.  The counts
    and errors do not depend on the round length's pieces or the budget."""
    g, h = upload(name, tmp_path), upload(name, tmp_path)
    try:
        W, H, spp = g.W, g.H, g.samples
        rects = grid(W, H)
        thr = calibrate(g, rects, 16, spp)
        results = {}
        for rp, budget in ((16, None), (7, None), (1, None), (16, 8192)):
            if budget:
                g.set_max_paths(budget)
            img, n, err, st = adaptive(g, rects, (16, rp, thr, FLOOR, spp))
            what = f"{name} round {rp} budget {budget}"
            counts = set(np.unique(n).tolist())
            assert len(counts) >= 3 and 16 in counts and spp in counts, (what, sorted(counts))
            assert st["paths"] == int(n.sum()), what
            check_counts_exact(h, rects, img, n, what)
            results[(rp, budget)] = (img, n, err)
        # the same rule with another round length tests at other pass counts; the same round length with pieces is the same frame
        a, b = results[(16, None)], results[(16, 8192)]
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
    finally:
        g.close()
        h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["g_nodes", "hdr"])
def test_threshold_zero_is_the_fixed_render(name, tmp_path):
    """Threshold 0 stops no pixel early: every count is pass_end and the frame is render_tiles(0, pass_end), also the committed
    digest of tests/golden/shade_frames.sha256.json at that configuration."""
    want = json.load(open(DIGESTS))
    cfg, budget = ((0, 0, 0, 0), None) if name == "g_nodes" else ((240, 135, 16, 32), 240 * 135 * 4)
    g, h = upload(name, tmp_path, cfg, budget), upload(name, tmp_path, cfg, budget)
    try:
        rects = grid(g.W, g.H)
        img, n, err, _ = adaptive(g, rects, (2, 3, 0.0, FLOOR, g.samples))
        assert (n == g.samples).all()
        h.clear()
        h.render_tiles(rects, 0, g.samples)
        assert img.tobytes() == h.read().tobytes()
        assert digest(img) == want[name]
    finally:
        g.close()
        h.close()


def replay(L, min_passes, round_passes, pass_end, threshold, floor):
    """the rule in numpy float32 on per-sample radiance L [pixels, passes, 3]: (counts, err)"""
    f = np.float32
    npx = L.shape[0]
    n = np.zeros(npx, np.uint32)
    mean = np.zeros(npx, f)
    m2 = np.zeros(npx, f)
    err = np.full(npx, np.inf, f)
    done = np.zeros(npx, bool)
    with np.errstate(divide="ignore", invalid="ignore"):
        return _replay(L, n, mean, m2, err, done, min_passes, round_passes, pass_end, threshold, floor)


def _replay(L, n, mean, m2, err, done, min_passes, round_passes, pass_end, threshold, floor):
    f = np.float32
    for k in range(pass_end + 1):
        if k >= min_passes and k < pass_end and (k - min_passes) % round_passes == 0:
            t = ~done
            kf = f(k)
            e = np.sqrt((m2 / f(k - 1)) / kf) / np.where(mean > f(floor), mean, f(floor))
            err[t] = e[t]
            done |= t & (e < f(threshold))
        if k == pass_end:
            break
        live = ~done
        s = L[:, k]
        y = (f(0.2126) * s[:, 0] + f(0.7152) * s[:, 1]) + f(0.0722) * s[:, 2]
        nn = n + live
        d = y - mean
        new_mean = mean + d / nn.astype(f)
        new_m2 = m2 + d * (y - new_mean)
        mean = np.where(live, new_mean, mean)
        m2 = np.where(live, new_m2, m2)
        n = nn.astype(np.uint32)
    return n, err


@pytest.mark.gpu
def test_counts_and_errors_against_the_oracle(tmp_path):
    """A 16x16 region of g_nodes at 32 passes: per-sample radiance from the oracle's camera states run to the end of their paths
    (semantics 1), the K5 update and the test-point rule replayed in numpy float32, give every pixel's count and error bit for bit,
    except pixels with a flagged sample (under 1e-5 of the samples)."""
    path = os.path.join(GOLDEN, "g_nodes.crscene")
    spp = 32
    x0, y0, x1, y1 = 8, 4, 24, 20
    o = O.OracleScene(path, 0, 0, spp, 0)
    try:
        st = o.camera_states(x0, y0, x1, y1, passes=(0, spp))
        res = o.path_step(st, 0, bounces=1 << 30)
        W, H = o.W, o.H
    finally:
        o.close()
    npx = (x1 - x0) * (y1 - y0)
    L = res["next"]["L"].reshape(npx, spp, 3).astype(np.float32)
    flag = ((res["flag"] != 0) | (st["pad"] != 0)).reshape(npx, spp).any(axis=1)
    assert flag.sum() <= max(1, npx * spp * 1e-5), f"{flag.sum()} of {npx} pixels have a flagged sample"
    _, err0 = replay(L, 8, 4, spp, 0.0, FLOOR)
    g = crgpu.GpuScene(path, 0, 0, spp, 0)
    try:
        assert (g.W, g.H) == (W, H)
        for thr in (float(np.median(err0[np.isfinite(err0)])), 0.05):
            want_n, want_err = replay(L, 8, 4, spp, thr, FLOOR)
            _, n, err, _ = adaptive(g, [(x0, y0, x1, y1)], (8, 4, thr, FLOOR, spp))
            # framebuffer rows are H-1-y; the oracle's region is row-major with y up
            got_n = n[H - y1:H - y0, x0:x1][::-1].reshape(-1)
            got_err = err[H - y1:H - y0, x0:x1][::-1].reshape(-1)
            ok = ~flag
            assert np.array_equal(got_n[ok], want_n[ok]), thr
            assert got_err[ok].tobytes() == want_err[ok].astype(np.float32).tobytes(), thr
            assert len(np.unique(want_n)) >= 2, thr
    finally:
        g.close()


# ---- GPU: stop, resume, snapshots, split ------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_stop_and_resume_mid_round(tmp_path):
    """On an armed scene, asynchronous rounds with a stop requested from a thread once the progress has moved, then resumed, leave the
    framebuffer, counts and errors of an uninterrupted synchronous run; a snapshot taken during a round shows the frame at the pass it
    reports (the run with pass_end at that pass)."""
    cfg = (480, 270, 64, 0)
    rule = lambda thr, end=64: (16, 16, thr, FLOOR, end)
    g = upload("hdr", tmp_path, cfg, 480 * 270 * 2)
    h = upload("hdr", tmp_path, cfg, 480 * 270 * 2)
    try:
        rects = grid(g.W, g.H, 64, 64)
        thr = calibrate(h, rects, 16, 64)
        want = adaptive(h, rects, rule(thr))
        g.enable_stop(True)
        g.clear()
        g.adaptive_reset()
        stops, snap = 0, None
        while True:
            d = g.adaptive_round(rects, *rule(thr), flags=crgpu.FLAG_ASYNC)
            if d["active"] == 0:
                break
            pb = d["pass_begin"]
            stopper = None
            if stops < 2 and d["pass_end"] - pb > 2:
                def stop_when_moved(pb=pb):
                    while True:
                        done, busy = g.progress()
                        if done > pb or not busy:
                            g.request_stop()
                            return
                        time.sleep(0.0005)
                stopper = threading.Thread(target=stop_when_moved)
                stopper.start()
            elif snap is None:
                g.request_snapshot()
            while True:
                if snap is None and stopper is None:
                    s = g.take_snapshot()
                    if s is not None and pb < s[1]:
                        snap = s
                if not g.progress()[1]:
                    break
                time.sleep(0.001)
            if stopper:
                stopper.join()
                stops += 1
                g.clear_stop()
            g.get_stats()
        got_n, got_err = g.adaptive_read()
        assert stops == 2
        assert g.read().tobytes() == want[0].tobytes()
        assert got_n.tobytes() == want[1].tobytes() and got_err.tobytes() == want[2].tobytes()
        if snap is not None:
            img, k = snap
            adaptive(h, rects, rule(thr, k))
            assert img.tobytes() == h.srgb8().tobytes(), k
    finally:
        g.close()
        h.close()


def split(rects, parts):
    """the interleave of the host renderer's workers (cr_renderer.c tile_rank) over a 37x29 grid"""
    return [[r for r in rects if ((r[0] // 37) + 5 * (r[1] // 29)) % parts == p] for p in range(parts)]


@pytest.mark.gpu
def test_independent_of_the_tile_split(tmp_path):
    """One scene rendering the whole tile set and two scenes each rendering an interleaved half of it (as -j 2 does) give the same
    counts, errors and pixels."""
    a, b, c = (upload("hdr", tmp_path) for _ in range(3))
    try:
        rects = grid(a.W, a.H)
        thr = calibrate(a, rects, 16, 64)
        img, n, err, _ = adaptive(a, rects, (16, 16, thr, FLOOR, 64))
        halves = split(rects, 2)
        parts = [adaptive(s, part, (16, 16, thr, FLOOR, 64)) for s, part in zip((b, c), halves)]
        for part, (pimg, pn, perr, _) in zip(halves, parts):
            for x0, y0, x1, y1 in part:
                rows = slice(a.H - y1, a.H - y0)
                assert pimg[rows, x0:x1].tobytes() == img[rows, x0:x1].tobytes()
                assert pn[rows, x0:x1].tobytes() == n[rows, x0:x1].tobytes()
                assert perr[rows, x0:x1].tobytes() == err[rows, x0:x1].tobytes()
    finally:
        for s in (a, b, c):
            s.close()


# ---- GPU: edits and refusals -----------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_edits(tmp_path):
    """After set_camera, a clear and a reset, rounds give what a fresh upload of the edited scene gives; after set_render to a new
    size a round without a reset is refused, and after one it works at the new size."""
    from test_gpu_scene_edit import Loaded, scene_json
    doc = scene_json("hdr")
    W, H, spp, b = 240, 135, 64, 32
    base = Loaded(doc, W, H, spp, b)
    moved = json.loads(json.dumps(doc))
    for tr in moved["camera"]["transforms"]:
        if tr["type"] == "translate":
            tr["x"] = tr.get("x", 0) + 0.05
    edited = Loaded(moved, W, H, spp, b)
    g, h = base.upload(), edited.upload()
    try:
        rects = grid(W, H)
        rule = (16, 16, 0.05, FLOOR, spp)
        adaptive(g, rects, rule)
        g.set_camera(edited.camera)
        got = adaptive(g, rects, rule)
        want = adaptive(h, rects, rule)
        for x, y in zip(got[:3], want[:3]):
            assert x.tobytes() == y.tobytes()
        small = Loaded(moved, 160, 90, spp, b)
        g.set_render(160, 90, spp, b, [small.camera])
        fb = g.read().copy()
        with pytest.raises(crgpu.CrgpuError):
            g.adaptive_round(grid(160, 90), *rule)
        assert g.read().tobytes() == fb.tobytes()
        h2 = small.upload()
        try:
            got = adaptive(g, grid(160, 90), rule)
            want = adaptive(h2, grid(160, 90), rule)
            for x, y in zip(got[:3], want[:3]):
                assert x.tobytes() == y.tobytes()
        finally:
            h2.close()
            small.free()
    finally:
        g.close()
        h.close()
        base.free()
        edited.free()


@pytest.mark.gpu
def test_refusals_change_nothing(tmp_path):
    """Each bad field, overlapping tiles, two tile sets left at different counts and a missing reset are refused, and leave the
    framebuffer, counts and errors byte-identical."""
    g = upload("hdr", tmp_path)
    try:
        rects = grid(g.W, g.H)
        with pytest.raises(crgpu.CrgpuError):                        # no reset yet
            g.adaptive_round(rects, 16, 16, 0.05, FLOOR)
        with pytest.raises(crgpu.CrgpuError):
            g.adaptive_read()
        g.clear()
        g.adaptive_reset()
        left = [r for r in rects if r[0] < g.W // 2]
        g.adaptive_round(left, 16, 16, 0.05, FLOOR)                  # the left half at 16 passes, the rest at 0
        before = (g.read().tobytes(),) + tuple(x.tobytes() for x in g.adaptive_read())
        good = dict(min_passes=16, round_passes=16, threshold=0.05, floor=FLOOR, pass_end=64)
        bad = [dict(min_passes=1), dict(min_passes=0), dict(round_passes=0), dict(pass_end=0), dict(pass_end=65),
               dict(threshold=-0.01), dict(threshold=math.nan), dict(threshold=math.inf), dict(floor=0.0), dict(floor=-1.0),
               dict(floor=math.nan), dict(floor=math.inf)]
        for change in bad:
            with pytest.raises(crgpu.CrgpuError):
                g.adaptive_round(rects, **dict(good, **change))
        overlapping = rects + [(5, 5, 9, 9)]
        with pytest.raises(crgpu.CrgpuError, match="overlaps"):
            g.adaptive_round(overlapping, **good)
        with pytest.raises(crgpu.CrgpuError, match="passes"):        # the whole set: pixels at 0 and at 16 are active
            g.adaptive_round(rects, **good)
        after = (g.read().tobytes(),) + tuple(x.tobytes() for x in g.adaptive_read())
        assert after == before
        d = g.adaptive_round(left, **good)                            # the left half goes on from 16
        assert d["pass_begin"] == 16 and d["active"] > 0
    finally:
        g.close()


# ---- GPU: the CLI ------------------------------------------------------------------------------------------------------------------

def decode_png(path):
    from test_host import decode_png as dec
    return dec(path)


@pytest.mark.gpu
def test_cli_adaptive(tmp_path):
    """cray_b200 --adaptive writes the sRGB8 of the Python path's adaptive frame and --dump-passes its counts; with two GPUs -j 2
    gives the same bits."""
    src = os.path.join(REFDIR, "input", "hdr.json")
    if not os.path.exists(EXE) or not os.path.exists(src):
        pytest.skip("cray_b200 or input/hdr.json not available")
    outs = {}
    for j in ([1, 2] if crgpu.device_count() >= 2 else [1]):
        png, passes = str(tmp_path / f"o{j}.png"), str(tmp_path / f"p{j}.u32")
        r = subprocess.run([EXE, os.path.join("input", "hdr.json"), "-d", "240x135", "-s", "64", "--adaptive", "0.05", "--dump-passes",
                            passes, "-o", png, "-j", str(j), "-q"], cwd=REFDIR, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                           text=True, timeout=300)
        assert r.returncode == 0, r.stdout[-2000:]
        outs[j] = (decode_png(png), np.fromfile(passes, dtype=np.uint32).reshape(135, 240))
    here = os.getcwd()
    os.chdir(REFDIR)                             # the CLI's scene: the same JSON, assets resolved from the same directory
    try:
        g = crgpu.GpuScene(os.path.join("input", "hdr.json"), 240, 135, 64, 0)
    finally:
        os.chdir(here)
    try:
        _, n, _, _ = adaptive(g, [(0, 0, 240, 135)], (16, 16, 0.05, FLOOR, 64))
        assert np.array_equal(outs[1][0], g.srgb8())
        assert np.array_equal(outs[1][1], n)
    finally:
        g.close()
    if 2 in outs:
        assert np.array_equal(outs[1][0], outs[2][0]) and np.array_equal(outs[1][1], outs[2][1])
