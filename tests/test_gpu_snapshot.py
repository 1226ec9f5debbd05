"""Reading the image of an armed render while it runs (crgpu_request_snapshot / crgpu_take_snapshot, include/crgpu.h), and the host
renderer's live preview built on it (crhostCurrentImage).

After each publish step of an armed call the framebuffer holds exactly the passes [pass_begin, k), so every snapshot is checked
byte for byte against the sRGB8 image of a fresh render of the passes it claims to show.  When a snapshot lands is up to the thread
timing; every outcome is checked deterministically.

CPU: argument checks of the new entry points.  GPU: everything else.
"""
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

import crgpu
from conftest import GOLDEN, ROOT

DIGESTS = os.path.join(GOLDEN, "shade_frames.sha256.json")
# (W, H, spp, bounces, max paths in flight), the frames of the stop tests: hdr runs 4 overlapped batches of 4 passes, refraction
# (the tail kernel) 4 of 2
FRAMES = {"hdr": (240, 135, 16, 32, 240 * 135 * 4), "refraction": (240, 135, 8, 512, 240 * 135 * 2)}
# hdr at 960x540, 32 spp, 2 bounces: whole calls run 32 overlapped batches of one pass, the pieces walks 4 pieces of about 131k
# pixels per pass
BIG = (960, 540, 32, 2)
BIG_PATHS = {"tile": 960 * 540 * 2, "tiles": 960 * 540 * 2, "pieces": 131072, "pieces_tiles": 131072}


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


# ---- CPU -----------------------------------------------------------------------------------------------------------------------

def test_snapshot_entry_points_reject_a_null_scene():
    L = crgpu.lib()
    buf = (C.c_uint8 * 12)()
    k = C.c_int(0)
    assert L.crgpu_request_snapshot(None) == -3
    assert L.crgpu_take_snapshot(None, buf, C.byref(k)) == -3
    assert L.crgpu_take_snapshot(None, None, None) == -3
    assert crgpu.PENDING == 2


def test_no_scene_without_a_device():
    """Without a GPU the scene a snapshot needs cannot be created: the product path fails loudly (CRGPU_ERR_NO_DEVICE) at scene
    creation, never on the CPU.  (The calls on a NULL or unarmed scene are checked above and in the GPU tests.)"""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    L = crgpu.lib()
    h = C.c_void_p()
    flat = crgpu.FlatScene()
    assert L.crscene_load(C.byref(flat), os.path.join(GOLDEN, "g_single.crscene").encode()) == 0
    assert L.crgpu_scene_create(C.byref(flat), 0, C.byref(h)) == -1
    L.crscene_free(C.byref(flat))
    with pytest.raises(crgpu.CrgpuError):
        crgpu.GpuScene(os.path.join(GOLDEN, "g_single.crscene"))


def test_host_preview_without_a_frame():
    """crhostCurrentImage before any frame: a blank image of the scene's size, and no frame rendering"""
    import crhost
    R = crhost.Renderer(os.path.join(GOLDEN, "g_single.crscene"), 32, 16, 4, 2)
    busy, img, passes = R.current_image(workers=1)
    assert busy is False and img.shape == (16, 32, 3) and not img.any() and passes == [0]
    R.close()


def _current_image_exact(R, w, h):
    """crhostCurrentImage into a buffer of exactly w*h*3 bytes followed by a guard: (busy, image bytes); fails if it wrote past"""
    import crhost
    n = w * h * 3
    buf = np.full(n + 4096, 0xAB, dtype=np.uint8)
    busy = crhost.lib().crhostCurrentImage(R.r, buf.ctypes.data)
    assert (buf[n:] == 0xAB).all(), "crhostCurrentImage wrote past the image"
    assert not (buf[:n] == 0xAB).all(), "crhostCurrentImage did not write the image"
    return busy, buf[:n]


def test_host_preview_follows_the_image_size():
    """after a size change between frames the preview has the new size: it writes exactly W*H*3 bytes (blank until the next
    frame), smaller or larger than before"""
    import crhost
    R = crhost.Renderer(os.path.join(GOLDEN, "g_single.crscene"), 64, 32, 4, 2)
    L = crhost.lib()
    for w, h in ((16, 8), (96, 48), (64, 32)):
        assert L.applySceneConfig(R.r, w, h, 0, 0) == 0
        busy, img = _current_image_exact(R, w, h)
        assert busy == 0 and not img.any()
    R.close()


# ---- GPU -----------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def scenes(tmp_path_factory):
    import oracle_lib as O
    d = str(tmp_path_factory.mktemp("snapshot_scenes"))
    out = {}
    for n in FRAMES:
        p = O.bundled_scene(n, d)
        if p:
            out[n] = p
    return out


def _need(scenes, name):
    if name not in scenes:
        pytest.skip(f"{name} not available")
    return scenes[name]


def _render(g, how, begin, count, flags=0, rects=None):
    if rects is not None:
        return g.render_tiles(rects, begin, count, flags)
    if how.endswith("tiles"):
        return g.render_tiles([(0, 0, g.W // 2, g.H), (g.W // 2, 0, g.W, g.H)], begin, count, flags)
    return g.render_tile(0, 0, g.W, g.H, begin, count, flags)


class Fresh:
    """sRGB8 images of fresh renders of [0, k) on top of a starting framebuffer, cached by k"""

    def __init__(self, g, how="tile", start=None, rects=None):
        self.g, self.how, self.start, self.rects, self.cache = g, how, start, rects, {}

    def __call__(self, k):
        if k not in self.cache:
            g = self.g
            if self.start is None:
                g.clear()
            else:
                g.write(self.start)
            if k:
                _render(g, self.how, 0, k, rects=self.rects)
            self.cache[k] = g.srgb8()
        return self.cache[k]


def _wait_taken(g, timeout=60):
    t0 = time.perf_counter()
    while time.perf_counter() - t0 < timeout:
        r = g.take_snapshot()
        if r is not None:
            return r
        time.sleep(0.0001)
    raise AssertionError("no snapshot within the timeout")


@pytest.mark.gpu
def test_unarmed_scene_rejects_snapshots():
    g = crgpu.GpuScene(os.path.join(GOLDEN, "g_single.crscene"))
    L = crgpu.lib()
    buf = np.zeros((g.H, g.W, 3), dtype=np.uint8)
    k = C.c_int(0)
    assert L.crgpu_request_snapshot(g.handle) == -3
    assert L.crgpu_take_snapshot(g.handle, buf.ctypes.data, C.byref(k)) == -3
    g.enable_stop()
    assert L.crgpu_take_snapshot(g.handle, None, C.byref(k)) == -3
    g.enable_stop(False)
    assert L.crgpu_request_snapshot(g.handle) == -3
    g.close()


@pytest.mark.gpu
def test_snapshot_is_staged_by_the_device_mid_call(scenes):
    """The request is made before an asynchronous call of 32 batches is enqueued, so only a publish step can answer it: the first
    image taken shows 0 < k < 32 passes, and equals a fresh render of [0, k)."""
    g = crgpu.GpuScene(_need(scenes, "hdr"), *BIG, max_paths=BIG_PATHS["tile"])
    g.enable_stop()
    g.clear()
    g.request_snapshot()
    g.render_tile(0, 0, g.W, g.H, 0, g.samples, crgpu.FLAG_ASYNC)
    img, k = _wait_taken(g)
    g.get_stats()
    assert g.progress() == (g.samples, False)
    assert 0 < k < g.samples, k
    assert img.tobytes() == Fresh(g)(k).tobytes(), k
    g.close()


# Every walk, through one call each, with repeated request / take cycles; run in a subprocess because CRGPU_OVERLAP is read once
# per process.  Prints one line per walk: the passes shown and whether every image and the final frame matched.
WALK_CODE = r"""
import sys, json, hashlib, time, tempfile
import numpy as np, crgpu, oracle_lib as O
BIG, PATHS = %r, %r
p = O.bundled_scene('hdr', tempfile.mkdtemp())
if not p: print('SKIP'); sys.exit(0)
def render(g, how, b, n, flags=0):
    if how.endswith('tiles'): return g.render_tiles([(0, 0, g.W // 2, g.H), (g.W // 2, 0, g.W, g.H)], b, n, flags)
    return g.render_tile(0, 0, g.W, g.H, b, n, flags)
for how in sorted(PATHS):
    g = crgpu.GpuScene(p, *BIG, max_paths=PATHS[how])
    g.enable_stop(); g.clear()
    render(g, how, 0, g.samples, crgpu.FLAG_ASYNC)
    shots, bad = [], []
    while True:
        busy = g.progress()[1]
        g.request_snapshot()
        r = None
        while r is None:
            r = g.take_snapshot()
        done = g.progress()[0]
        if r[1] > done: bad.append(('ahead of progress', r[1], done))
        shots.append(r)
        if not busy: break
    g.get_stats()
    final = hashlib.sha256(g.read().tobytes()).hexdigest()
    ks = [k for _, k in shots]
    if any(a > b for a, b in zip(ks, ks[1:])): bad.append(('went backwards', ks))
    fresh = {}
    for img, k in shots:
        if k not in fresh:
            g.clear()
            if k: render(g, how, 0, k)
            fresh[k] = g.srgb8().tobytes()
        if img.tobytes() != fresh[k]: bad.append(('image differs', k))
    print('WALK', json.dumps({'how': how, 'passes': sorted(set(ks)), 'mid': sum(0 < k < g.samples for k in ks), 'final': final, 'bad': bad}))
    g.close()
"""


@pytest.mark.gpu
@pytest.mark.parametrize("overlap", ["0", "1"])
def test_every_walk_bit_for_bit(scenes, overlap):
    """tile, tile union, pieces by rows, pieces by pixel list: each image equals a fresh render of its k, k never decreases and
    never passes crgpu_progress, and the frame still ends on the digest of an uninterrupted render"""
    p = _need(scenes, "hdr")
    g = crgpu.GpuScene(p, *BIG)
    g.clear()
    g.render_tile(0, 0, g.W, g.H)
    want = digest(g.read())
    g.close()
    env = dict(os.environ, CRGPU_OVERLAP=overlap, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "c-ray_b200"), os.path.join(ROOT, "tests")]))
    r = subprocess.run([sys.executable, "-c", WALK_CODE % (BIG, BIG_PATHS)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       env=env, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:]
    walks = [json.loads(line[5:]) for line in r.stdout.splitlines() if line.startswith("WALK ")]
    assert sorted(w["how"] for w in walks) == sorted(BIG_PATHS), r.stdout[-3000:]
    for w in walks:
        print(overlap, w["how"], "passes shown:", w["passes"])
        assert not w["bad"], w
        assert w["final"] == want, w["how"]
    assert any(w["mid"] for w in walks), "no snapshot landed inside a call"


@pytest.mark.gpu
def test_pixels_outside_the_tiles(scenes):
    """a tile-union call over a poisoned framebuffer: the snapshot is a fresh render of [0, k) of those tiles over the poison, and
    every pixel outside the tiles is srgb8(poison)"""
    g = crgpu.GpuScene(_need(scenes, "hdr"), *BIG, max_paths=BIG_PATHS["tile"])
    g.enable_stop()
    poison = np.random.default_rng(11).standard_normal((g.H, g.W, 3)).astype(np.float32)
    rects = [(0, 0, 96, 64), (300, 200, 701, 333), (900, 500, 960, 540)]
    g.write(poison)
    want_out = g.srgb8()
    g.request_snapshot()
    g.render_tiles(rects, 0, g.samples, crgpu.FLAG_ASYNC)
    img, k = _wait_taken(g)
    g.get_stats()
    inside = np.zeros((g.H, g.W), dtype=bool)
    for x0, y0, x1, y1 in rects:
        inside[g.H - y1:g.H - y0, x0:x1] = True            # rows of the framebuffer layout: row H-1-y
    assert 0 < k <= g.samples
    assert img[~inside].tobytes() == want_out[~inside].tobytes()
    assert img.tobytes() == Fresh(g, start=poison, rects=rects)(k).tobytes(), k
    g.close()


@pytest.mark.gpu
def test_snapshot_and_stop(scenes):
    """after an in-flight stop the image shows exactly the committed passes; with the stop set before the call it shows the
    untouched framebuffer; with no call in flight it equals crgpu_framebuffer_to_srgb8"""
    g = crgpu.GpuScene(_need(scenes, "hdr"), *BIG, max_paths=BIG_PATHS["tile"])
    g.enable_stop()
    fresh = Fresh(g)
    g.clear()
    g.render_tile(0, 0, g.W, g.H, 0, g.samples, crgpu.FLAG_ASYNC)
    t0 = time.perf_counter()
    while g.progress()[0] < 4 and g.progress()[1] and time.perf_counter() - t0 < 60:
        time.sleep(0.0001)
    g.request_snapshot()
    g.request_stop()
    g.get_stats()
    done, busy = g.progress()
    assert not busy and done < g.samples, done
    img, k = _wait_taken(g)                               # staged by a publish step, or the framebuffer after the call
    assert k <= done
    committed = g.srgb8()
    g.request_snapshot()
    img2, k2 = _wait_taken(g)
    assert k2 == done and img2.tobytes() == committed.tobytes()
    g.clear_stop()                                        # (the fresh renders must not stop)
    assert img.tobytes() == fresh(k).tobytes(), (k, done)
    assert committed.tobytes() == fresh(done).tobytes(), done

    g.request_stop()
    poison = np.random.default_rng(5).standard_normal((g.H, g.W, 3)).astype(np.float32)
    g.write(poison)
    want = g.srgb8()
    for begin in (0, 5):
        g.request_snapshot()
        st = g.render_tile(0, 0, g.W, g.H, begin, g.samples - begin)
        assert st["stopped"] is True
        img, k = _wait_taken(g)
        assert k == begin and img.tobytes() == want.tobytes()
    g.clear_stop()

    g.clear()
    g.render_tile(0, 0, g.W, g.H)
    g.request_snapshot()
    img, k = _wait_taken(g)
    assert k == g.samples and img.tobytes() == g.srgb8().tobytes()
    img, k = _wait_taken(g)                               # no call in flight: the framebuffer, also without a request
    assert k == g.samples and img.tobytes() == g.srgb8().tobytes()
    g.close()


def _snap_through(g, how, flags=0):
    """render [0, spp) asynchronously while this thread requests and takes snapshots throughout; returns the passes shown"""
    ks = []
    _render(g, how, 0, g.samples, crgpu.FLAG_ASYNC | flags)
    while True:
        busy = g.progress()[1]
        g.request_snapshot()
        r = None
        while r is None:
            r = g.take_snapshot()
        ks.append(r[1])
        if not busy:                 # the call was over before this request: the last image is the finished frame
            break
    return ks


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(FRAMES))
def test_snapshots_leave_the_frame_alone(scenes, name):
    """frames rendered while snapshots are taken throughout end on the committed digests, with the kernel launches of a call
    that took none"""
    W, H, spp, b, mp = FRAMES[name]
    want = json.load(open(DIGESTS))[name]
    g = crgpu.GpuScene(_need(scenes, name), W, H, spp, b, max_paths=mp)
    g.enable_stop()
    for how in ("tile", "tiles"):
        g.clear()
        plain = _render(g, how, 0, g.samples)
        assert digest(g.read()) == want
        g.clear()
        ks = _snap_through(g, how)
        st = g.get_stats()
        assert digest(g.read()) == want, (how, ks)
        assert st["kernel_launches"] == plain["kernel_launches"], how
        assert st["paths"] == plain["paths"]
        assert ks == sorted(ks) and ks[-1] == g.samples, ks
    g.close()


# ---- the host renderer (libcrhost.so) ------------------------------------------------------------------------------------------
HOST = (480, 270, 4000, 32)       # hdr: 518 M paths, several batches at the default paths-in-flight budget


def _gpus(n):
    try:
        return crgpu.device_count() >= n
    except crgpu.CrgpuError:
        return False


@pytest.mark.gpu
@pytest.mark.parametrize("gpus", [1, 2])
def test_host_preview(scenes, gpus):
    """crhostCurrentImage polled from another thread through a frame: each worker's tiles in every image equal a fresh render
    of the passes that worker had committed at its snapshot, and the frame's image and framebuffer are those of a frame nobody
    watched"""
    import crhost
    if not _gpus(gpus):
        pytest.skip(f"needs {gpus} GPUs")
    p = _need(scenes, "hdr")
    W, H, spp, b = HOST
    R = crhost.Renderer(p, W, H, spp, b, gpus=gpus, tile=32)
    R.prepare()
    _, _, every = R.rank_tiles(0, 1)
    owners = np.zeros(len(every), dtype=np.int32)
    crhost.lib().crhostTileOwners(R.r, gpus, owners.ctypes.data)

    assert R.render() is not None
    quiet_fb = R.framebuffer().copy()
    busy, quiet_img, passes = R.current_image(gpus)
    assert not busy and passes == [spp] * gpus

    seen, out = [], {}
    th = threading.Thread(target=lambda: out.setdefault("r", R.render()))
    th.start()
    while th.is_alive():
        busy, img, passes = R.current_image(gpus)
        committed = [R.worker_passes(t) for t in range(gpus)]
        if busy:
            assert all(p <= c for p, c in zip(passes, committed)), (passes, committed)
            if not seen or seen[-1][0] != passes:
                seen.append((passes, img))
        time.sleep(0.01)
    th.join()
    assert out["r"] is not None
    busy, img, passes = R.current_image(gpus)
    assert not busy and passes == [spp] * gpus
    assert img.tobytes() == quiet_img.tobytes()
    assert R.framebuffer().tobytes() == quiet_fb.tobytes()
    shown = sorted({k for ps, _ in seen for k in ps})
    print(f"{gpus} GPU(s): {len(seen)} distinct previews, passes shown {shown}")
    assert any(0 < k < spp for k in shown), "no preview landed inside the frame"
    # a size change after the frame: the preview follows it (blank, exactly W*H*3 bytes), never the last frame's bytes
    assert crhost.lib().applySceneConfig(R.r, W // 2, H // 2, 0, 0) == 0
    busy, small = _current_image_exact(R, W // 2, H // 2)
    assert busy == 0 and not small.any()
    assert crhost.lib().applySceneConfig(R.r, W, H, 0, 0) == 0

    g = crgpu.GpuScene(p, W, H, spp, b)
    fresh = {}
    for ps, im in seen:
        for t, k in enumerate(ps):
            rects = [tuple(every[i]) for i in range(len(every)) if owners[i] == t]
            if (t, k) not in fresh:
                g.clear()
                if k:
                    g.render_tiles(rects, 0, k)
                fresh[(t, k)] = g.srgb8()
            mask = np.zeros((H, W), dtype=bool)
            for x0, y0, x1, y1 in rects:
                mask[H - y1:H - y0, x0:x1] = True
            assert im[mask].tobytes() == fresh[(t, k)][mask].tobytes(), (t, k)
    g.close()
    R.close()
