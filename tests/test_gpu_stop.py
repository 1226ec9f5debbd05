"""Stopping, pausing and resuming a render at a pass boundary (crgpu_stop_enable / crgpu_request_stop, include/crgpu.h), and the
host renderer's abort / pause controls built on it (crhostAbort / crhostSetPaused / crhostProgress).

An armed call adds each batch of passes only in pass order and only if no stop was seen during it, so after any call the
framebuffer holds exactly the passes [0, passes_done) and a call for [passes_done, spp) finishes the frame bit for bit.  When a
stop lands is up to the thread timing; every outcome is checked deterministically against fresh renders and against the committed
digests of tests/golden/shade_frames.sha256.json.  Stops are requested through the API only.

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
# (name, W, H, spp, bounces, max paths in flight): hdr runs 4 overlapped batches of 4 passes, refraction (the tail kernel) 4 of 2
FRAMES = {"hdr": (240, 135, 16, 32, 240 * 135 * 4), "refraction": (240, 135, 8, 512, 240 * 135 * 2)}


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


# ---- CPU -----------------------------------------------------------------------------------------------------------------------

def test_entry_points_reject_a_null_scene():
    L = crgpu.lib()
    n, b = C.c_int(0), C.c_int(0)
    assert L.crgpu_stop_enable(None, 1) == -3
    assert L.crgpu_stop_enable(None, 0) == -3
    assert L.crgpu_request_stop(None) == -3
    assert L.crgpu_clear_stop(None) == -3
    assert L.crgpu_progress(None, C.byref(n), C.byref(b)) == -3
    assert crgpu.STOPPED == 1


def test_no_scene_to_arm_without_a_device():
    """Without a GPU no scene exists to arm: the product path fails loudly (CRGPU_ERR_NO_DEVICE), never on the CPU."""
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
        crgpu.GpuScene(os.path.join(GOLDEN, "g_single.crscene")).enable_stop()


# ---- GPU -----------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def scenes(tmp_path_factory):
    import oracle_lib as O
    d = str(tmp_path_factory.mktemp("stop_scenes"))
    out = {}
    for n in FRAMES:
        p = O.bundled_scene(n, d)
        if p:
            out[n] = p
    return out


def _scene(scenes, name, max_paths=None):
    if name not in scenes:
        pytest.skip(f"{name} not available")
    W, H, spp, b, mp = FRAMES[name]
    return crgpu.GpuScene(scenes[name], W, H, spp, b, max_paths=max_paths or mp)


def _full(g):
    g.clear()
    g.render_tile(0, 0, g.W, g.H)
    return g.read().copy()


@pytest.mark.gpu
def test_unarmed_scene_rejects_stop_and_progress():
    g = crgpu.GpuScene(os.path.join(GOLDEN, "g_single.crscene"))
    L = crgpu.lib()
    assert L.crgpu_request_stop(g.handle) == -3
    assert L.crgpu_clear_stop(g.handle) == -3
    assert L.crgpu_progress(g.handle, None, None) == -3
    g.enable_stop(False)                          # disarming an idle, unarmed scene is a no-op
    g.enable_stop(True)
    assert g.progress() == (0, False)
    g.enable_stop(False)
    assert L.crgpu_request_stop(g.handle) == -3
    g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(FRAMES))
def test_armed_frame_is_bit_identical(scenes, name):
    want = json.load(open(DIGESTS))[name]
    g = _scene(scenes, name)
    plain = _full(g)
    u = g.render_tile(0, 0, g.W, g.H, 0, 0)       # an empty call
    g.enable_stop()
    g.clear()
    st = g.render_tile(0, 0, g.W, g.H)
    armed = g.read().copy()
    assert st["stopped"] is False and st["paths"] == g.W * g.H * g.samples
    assert g.progress() == (g.samples, False)
    assert digest(plain) == want and digest(armed) == want
    g.clear()
    g.render_tiles([(0, 0, g.W // 2, g.H), (g.W // 2, 0, g.W, g.H)])
    assert digest(g.read()) == want
    g.close()
    assert u["paths"] == 0


@pytest.mark.gpu
def test_armed_frame_without_overlap():
    """CRGPU_OVERLAP=0 (one wave set, read once per process): the armed hdr frame still reproduces its digest"""
    code = ("import sys, json, hashlib, crgpu, oracle_lib as O, tempfile\n"
            "p = O.bundled_scene('hdr', tempfile.mkdtemp())\n"
            "if not p: print('SKIP'); sys.exit(0)\n"
            "g = crgpu.GpuScene(p, 240, 135, 16, 32, max_paths=240 * 135 * 2)\n"
            "g.enable_stop(); g.render_tile(0, 0, 240, 135)\n"
            "print('DIGEST', hashlib.sha256(g.read().tobytes()).hexdigest())\n")
    env = dict(os.environ, CRGPU_OVERLAP="0", PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "c-ray_b200"), os.path.join(ROOT, "tests")]))
    r = subprocess.run([sys.executable, "-c", code], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env, timeout=600)
    if "SKIP" in r.stdout:
        pytest.skip("hdr not available")
    assert "DIGEST " + json.load(open(DIGESTS))["hdr"] in r.stdout, r.stdout[-2000:]


@pytest.mark.gpu
def test_stop_before_the_call_commits_nothing(scenes):
    g = _scene(scenes, "hdr")
    g.enable_stop()
    poison = np.random.default_rng(7).standard_normal((g.H, g.W, 3)).astype(np.float32)
    g.write(poison)
    g.request_stop()
    for begin in (0, 5):
        st = g.render_tile(0, 0, g.W, g.H, begin, g.samples - begin)
        assert st["stopped"] is True and st["paths"] == 0
        assert g.progress() == (begin, False)
        st = g.render_tiles([(0, 0, 16, 16), (100, 50, 140, 90)], begin, g.samples - begin)
        assert st["stopped"] is True and g.progress() == (begin, False)
    assert g.read().tobytes() == poison.tobytes()
    g.clear_stop()
    g.close()


def _render(g, how, begin, count, flags=0):
    if how.endswith("tiles"):
        return g.render_tiles([(0, 0, g.W // 2, g.H), (g.W // 2, 0, g.W, g.H)], begin, count, flags)
    return g.render_tile(0, 0, g.W, g.H, begin, count, flags)


def _stopped_run(g, how, delay, begin=0):
    """render [begin, spp) while another thread requests a stop after `delay` seconds; returns passes_done"""
    t = threading.Timer(delay, g.request_stop)
    t.start()
    st = _render(g, how, begin, g.samples - begin)
    t.join()
    done, busy = g.progress()
    assert not busy and begin <= done <= g.samples
    assert st["stopped"] == (done < g.samples)
    assert st["paths"] == g.W * g.H * (done - begin)
    return done


def _stop_in_flight(g, how, begin, at):
    """Enqueue [begin, spp) asynchronously, so that every batch is queued before the stop and only the device's gates can
    act on it; wait until `at` passes are committed, request the stop, and return the committed pass index."""
    _render(g, how, begin, g.samples - begin, crgpu.FLAG_ASYNC)
    t0 = time.perf_counter()
    while True:
        done, busy = g.progress()
        if done >= at or not busy or time.perf_counter() - t0 > 60:
            break
        time.sleep(0.0001)
    g.request_stop()
    st = g.get_stats()
    done, busy = g.progress()
    assert not busy and begin <= done <= g.samples
    assert st["paths"] == g.W * g.H * (done - begin)
    return done


def _check_prefix_and_resume(g, how, done, want):
    """the framebuffer is a fresh render of [0, done), and resuming from it ends on `want` (a digest)"""
    stopped = g.read().copy()
    g.clear_stop()
    g.clear()
    if done:
        _render(g, how, 0, done)
    assert g.read().tobytes() == stopped.tobytes(), done
    g.write(stopped)
    if done < g.samples:
        st = _render(g, how, done, g.samples - done)
        assert st["stopped"] is False
    assert digest(g.read()) == want, done


@pytest.mark.gpu
@pytest.mark.parametrize("name,how", [("hdr", "tile"), ("hdr", "tiles"), ("hdr", "pieces"), ("hdr", "pieces_tiles"),
                                      ("refraction", "tile"), ("refraction", "pieces")])
def test_stop_from_another_thread(scenes, name, how):
    """stops at several delays over the frame (early bounces, the tail kernel's bounces, the last batch): the framebuffer is
    a fresh render of [0, passes_done), and resuming from there ends on the committed digest"""
    want = json.load(open(DIGESTS))[name]
    g = _scene(scenes, name, max_paths=8192 if how.startswith("pieces") else None)
    g.enable_stop()
    g.clear()
    t0 = time.perf_counter()
    _render(g, how, 0, g.samples)
    T = time.perf_counter() - t0
    assert digest(g.read()) == want
    seen = set()
    for frac in (0.0, 0.05, 0.2, 0.4, 0.6, 0.8, 0.95):
        g.clear_stop()
        g.clear()
        done = _stopped_run(g, how, frac * T)
        seen.add(done)
        _check_prefix_and_resume(g, how, done, want)
    print(f"{name}/{how}: frame {1e3 * T:.1f} ms, passes done at the stops: {sorted(seen)}")
    g.close()


# A frame of many short batches that takes tens of ms on an H100 and is enqueued in a few ms: hdr at 960x540, 32 spp, 2 bounces.
# Whole calls run 32 overlapped batches of one pass; the pieces walks run 4 pieces of about 131k pixels per pass.
BIG = (960, 540, 32, 2)
BIG_PATHS = {"tile": 960 * 540 * 2, "tiles": 960 * 540 * 2, "pieces": 131072, "pieces_tiles": 131072}


@pytest.fixture(scope="module")
def big_frame(scenes):
    if "hdr" not in scenes:
        pytest.skip("hdr not available")
    g = crgpu.GpuScene(scenes["hdr"], *BIG)
    full = digest(_full(g))
    g.close()
    return full


@pytest.mark.gpu
@pytest.mark.parametrize("how", sorted(BIG_PATHS))
def test_stop_takes_effect_in_flight(scenes, big_frame, how):
    """Every batch is queued before the stop is requested, so the host never sees it: a call that still commits fewer passes
    than asked proves that the device's gates read the stop and the commit step honoured it."""
    g = crgpu.GpuScene(scenes["hdr"], *BIG, max_paths=BIG_PATHS[how])
    g.enable_stop()
    spp = g.samples
    g.clear()
    done = _stop_in_flight(g, how, 0, 0)                # right after the enqueue
    assert done < spp, "the stop requested while the batches ran did not take effect"
    _check_prefix_and_resume(g, how, done, big_frame)
    g.clear_stop()
    g.clear()
    done = _stop_in_flight(g, how, 0, spp // 4)         # after a quarter of the passes is committed
    assert spp // 4 <= done < spp, done
    _check_prefix_and_resume(g, how, done, big_frame)
    g.close()


@pytest.mark.gpu
def test_repeated_pause_and_resume(scenes, big_frame):
    """several stop / resume cycles in one frame, each stopped while its batches run; the frame ends bit-identical"""
    g = crgpu.GpuScene(scenes["hdr"], *BIG, max_paths=BIG_PATHS["tile"])
    g.enable_stop()
    g.clear()
    begin, cycles = 0, 0
    while begin + 12 < g.samples:
        g.clear_stop()
        done = _stop_in_flight(g, "tile", begin, begin + 4)
        assert begin + 4 <= done < g.samples, (begin, done)
        begin, cycles = done, cycles + 1
    assert cycles >= 2
    g.clear_stop()
    st = g.render_tile(0, 0, g.W, g.H, begin, g.samples - begin)
    assert st["stopped"] is False
    assert digest(g.read()) == big_frame
    g.close()


@pytest.mark.gpu
def test_stop_without_bounces(scenes):
    """bounces = 0: the batch has no bounce, only the gate that follows K1"""
    if "hdr" not in scenes:
        pytest.skip("hdr not available")
    g = crgpu.GpuScene(scenes["hdr"], 960, 540, 256, 0, force_bounces=0, max_paths=960 * 540)   # 256 batches of one pass
    plain = _full(g)
    g.enable_stop()
    g.write(np.ones_like(plain))
    g.request_stop()
    st = g.render_tile(0, 0, g.W, g.H)
    assert st["stopped"] is True and g.progress() == (0, False)
    assert (g.read() == 1).all()
    g.clear_stop()
    g.clear()
    done = _stop_in_flight(g, "tile", 0, 0)
    assert done < g.samples, "the stop requested while the batches ran did not take effect"
    assert g.read().tobytes() == plain.tobytes()          # black, whatever the pass count
    g.clear_stop()
    g.render_tile(0, 0, g.W, g.H, done, g.samples - done)
    assert g.read().tobytes() == plain.tobytes()
    g.close()


# ---- the host renderer (libcrhost.so) ------------------------------------------------------------------------------------------
HOST = (480, 270, 4000, 32)       # hdr: 518 M paths, several batches at the default paths-in-flight budget


def _host_frame(R, gpus, drive):
    """one renderFrame of R in a thread while this thread runs drive(R, total tile-passes) and then polls the progress"""
    seen, out = [], {}

    def run():
        out["r"] = R.render()

    th = threading.Thread(target=run)
    th.start()
    while not R.progress()[0] and th.is_alive():
        time.sleep(0.0005)
    drive(R, R.samples * int(crhost_lib().crhostTileCount(R.r)))
    while th.is_alive():
        seen.append(R.progress()[1])
        time.sleep(0.002)
    th.join()
    seen.append(R.progress()[1])
    assert all(a <= c for a, c in zip(seen, seen[1:])), "progress went backwards"
    fb = R.framebuffer().copy() if out["r"] is not None else None
    return out["r"], fb, [R.worker_passes(t) for t in range(gpus)]


def crhost_lib():
    import crhost
    return crhost.lib()


def _wait_committed(R, at_least=1):
    """until the workers have committed some passes (their first batch), or the frame ended"""
    t0 = time.perf_counter()
    while R.progress()[0] and R.progress()[1] < at_least and time.perf_counter() - t0 < 60:
        time.sleep(0.0005)


def _host_reference(scenes, passes_of_tile, every):
    """fresh single-GPU renders: each tile with its worker's committed passes"""
    W, H, spp, b = HOST
    g = crgpu.GpuScene(scenes["hdr"], W, H, spp, b)
    g.clear()
    for p in sorted(set(passes_of_tile)):
        rects = [tuple(every[i]) for i in range(len(every)) if passes_of_tile[i] == p]
        if p:
            g.render_tiles(rects, 0, p)
    fb = g.read().copy()
    g.close()
    return fb


def _gpus(n):
    try:
        return crgpu.device_count() >= n
    except crgpu.CrgpuError:
        return False


@pytest.mark.gpu
@pytest.mark.parametrize("gpus", [1, 2])
def test_host_renderer_pause_resume_and_abort(scenes, gpus):
    """One Renderer, four frames, polled from this thread throughout: uninterrupted, paused and resumed, aborted with and
    without saving.  Each control acts after the workers' first commit, while later batches are still queued."""
    import crhost
    if not _gpus(gpus):
        pytest.skip(f"needs {gpus} GPUs")
    if "hdr" not in scenes:
        pytest.skip("hdr not available")
    W, H, spp, b = HOST
    R = crhost.Renderer(scenes["hdr"], W, H, spp, b, gpus=gpus, tile=32)
    R.prepare()
    _, _, every = R.rank_tiles(0, 1)
    owners = np.zeros(len(every), dtype=np.int32)
    crhost.lib().crhostTileOwners(R.r, gpus, owners.ctypes.data)

    r, full, passes = _host_frame(R, gpus, lambda R, total: None)
    assert r is not None and passes == [spp] * gpus

    paused = []

    def pause_cycles(R, total):
        for _ in range(3):
            _wait_committed(R, (paused[-1][1] if paused else 0) + 1)
            if not R.progress()[0]:
                break
            R.set_paused(True)
            time.sleep(0.2)                   # the stop drains
            p1 = R.progress()[1]
            time.sleep(0.1)
            paused.append((p1, R.progress()[1], total))
            R.set_paused(False)

    r, fb, passes = _host_frame(R, gpus, pause_cycles)
    assert r is not None and passes == [spp] * gpus
    held = [(p1, p2) for p1, p2, total in paused if p1 < total]      # pauses that landed before the last batch's end
    assert held and all(p1 == p2 for p1, p2 in held), paused                      # the pause held the workers
    assert fb.tobytes() == full.tobytes()

    def abort(save):
        def drive(R, total):
            _wait_committed(R)
            R.abort(save=save)
        return drive

    r, fb, passes = _host_frame(R, gpus, abort(True))
    assert r is not None
    assert all(p < spp for p in passes), passes                                  # the abort stopped every worker
    ref = _host_reference(scenes, [passes[o] for o in owners], every)
    assert fb.tobytes() == ref.tobytes(), passes

    r, _, passes = _host_frame(R, gpus, abort(False))
    assert r is None and all(p < spp for p in passes), passes
    R.close()
