"""The kernels of adaptive rendering, each on its own, against a numpy float32 replay (DESIGN §4 "Rendering adaptively").

K5 (k_accumulate, all eight path orders, plain and <ADAPTIVE>) runs on given radiance through crgpu_accumulate_samples; the select,
the scan and the compaction of a round run on given records through crgpu_adaptive_write and crgpu_adaptive_select.  The library is
built with -fmad=false and IEEE division and square root, so numpy float32 gives the same bits: NaN equals any NaN, -0 and +0 differ.
The sizes reach the paths that only large tile sets take: K5's second grid-stride pass (more pixels than its 132 x 8 x 256 threads),
the select and compaction's second grid-stride pass and the scan's third level (more than 1,048,576 pixels), up to a whole 3840x2160
frame.  Last, a 1920x1080 adaptive render is checked against fixed renders and against the oracle's per-sample radiance.

CPU: argument refusals of the entry points, and the numpy references against a float64 restatement.  GPU: everything else.
"""
import ctypes as C
import os

import numpy as np
import pytest

import crgpu
import oracle_lib as O
from conftest import GOLDEN
from test_gpu_adaptive import FLOOR, calibrate, check_counts_exact, grid, replay

f32 = np.float32
DONE = crgpu.ADAPTIVE_DONE
NODES = os.path.join(GOLDEN, "g_nodes.crscene")
BIG_PASS = 2 ** 24 - 3            # (float)completed rounds from here on
SPECIALS = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 1e-45, 1e-40, -1e-40, 3e19, -3e19, 1e30, 3.4e38], dtype=f32)


# ---- the numpy references --------------------------------------------------------------------------------------------------------

@np.errstate(all="ignore")
def ref_accumulate(fb, s, pass_begin):
    """K5's running average (renderer.c:283-300): fb [n, 3] after passes pass_begin.. of the samples s [n, passes, 3]"""
    r = np.array(fb, dtype=f32)
    for j in range(s.shape[1]):
        completed = pass_begin + j + 1
        k, t = f32(completed - 1), f32(1) / f32(completed)
        r = (r * k + s[:, j]) * t
    return r


@np.errstate(all="ignore")
def luminance(s):
    return (f32(0.2126) * s[..., 0] + f32(0.7152) * s[..., 1]) + f32(0.0722) * s[..., 2]


@np.errstate(all="ignore")
def ref_welford(n, mean, m2, s):
    """K5 <ADAPTIVE>'s record update for each pass of s [n, passes, 3]: (n, mean, M2), the done bit kept"""
    n, mean, m2 = np.array(n, np.uint32), np.array(mean, f32), np.array(m2, f32)
    for j in range(s.shape[1]):
        y = luminance(s[:, j])
        n = n + np.uint32(1)
        d = y - mean
        mean = mean + d / (n & np.uint32(~DONE & 0xffffffff)).astype(f32)
        m2 = m2 + d * (y - mean)
    return n, mean, m2


@np.errstate(all="ignore")
def ref_test(recs, min_passes, round_passes, pass_end, threshold, floor):
    """the select's test (crg_adapt_test) on records (ADAPT_RECORD_DTYPE): (records after it, active mask)"""
    out = np.array(recs, dtype=crgpu.ADAPT_RECORD_DTYPE)
    done = (out["n"] & DONE) != 0
    n = (out["n"] & ~np.uint32(DONE)).astype(np.int64)
    point = (n >= min_passes) & (n < pass_end) & ((n - min_passes) % round_passes == 0)
    t = point & ~done
    nn = np.maximum(n, 2)
    e = np.sqrt((out["m2"] / (nn - 1).astype(f32)) / nn.astype(f32)) / np.where(out["mean"] > f32(floor), out["mean"], f32(floor))
    out["err"] = np.where(t, e, out["err"])
    stop = t & (e < f32(threshold))
    out["n"] = np.where(stop, out["n"] | np.uint32(DONE), out["n"])
    active = ~(done | stop) & (n < pass_end)
    return out, active


def nan_equal(a, b):
    """elementwise: the same bits, or both NaN"""
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def assert_bits(got, want, what):
    eq = nan_equal(got, want)
    if not eq.all():
        i = np.argwhere(~eq)[0]
        raise AssertionError(f"{what}: {(~eq).sum()} of {eq.size} values differ; first at {i.tolist()}: got "
                             f"{np.asarray(got)[tuple(i)]!r}, want {np.asarray(want)[tuple(i)]!r}")


# ---- CPU ------------------------------------------------------------------------------------------------------------------------

def test_entry_points_reject_null_arguments():
    L = crgpu.lib()
    rect = np.array([0, 0, 1, 1], dtype=np.int32)
    a = crgpu.Adaptive(2, 1, 1, 0.1, 0.01)
    samples = np.zeros(4, dtype=np.float32)
    recs = np.zeros(1, dtype=crgpu.ADAPT_RECORD_DTYPE)
    out = np.zeros(4, dtype=np.uint32)
    n, lo, hi = C.c_uint32(0), C.c_uint32(0), C.c_uint32(0)
    assert L.crgpu_accumulate_samples(None, rect.ctypes.data, 1, 0, 1, -1, 0, samples.ctypes.data, None) == -3
    assert L.crgpu_accumulate_samples(None, rect.ctypes.data, 1, 0, 1, -1, 1, None, out.ctypes.data) == -3
    assert L.crgpu_adaptive_write(None, recs.ctypes.data) == -3
    assert L.crgpu_adaptive_write(None, None) == -3
    assert L.crgpu_adaptive_records(None, recs.ctypes.data) == -3
    assert L.crgpu_adaptive_records(None, None) == -3
    assert L.crgpu_adaptive_select(None, rect.ctypes.data, 1, C.byref(a), out.ctypes.data, C.byref(n), C.byref(lo), C.byref(hi)) == -3
    assert L.crgpu_adaptive_select(None, rect.ctypes.data, 1, None, None, None, None, None) == -3


def test_no_scene_for_the_kernels_without_a_device():
    """Without a GPU there is no scene to run the kernels on: creating one fails loudly (CRGPU_ERR_NO_DEVICE), never on the CPU."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    with pytest.raises(crgpu.CrgpuError):
        crgpu.GpuScene(NODES).accumulate_samples([(0, 0, 1, 1)], 0, np.zeros((1, 1, 4), np.float32))


def test_running_average_reference_against_float64():
    """ref_accumulate, from a cleared and from a seeded framebuffer, is the float64 mean of what it was given to 1e-5 relative."""
    rng = np.random.default_rng(1)
    for pass_begin, passes in ((0, 1), (0, 64), (7, 33), (999, 17), (BIG_PASS, 17)):
        s = rng.random((500, passes, 3), dtype=f32) * 4
        fb = rng.random((500, 3), dtype=f32) * 2 if pass_begin else np.zeros((500, 3), f32)
        got = ref_accumulate(fb, s, pass_begin).astype(np.float64)
        want = (fb.astype(np.float64) * pass_begin + s.astype(np.float64).sum(axis=1)) / (pass_begin + passes)
        np.testing.assert_allclose(got, want, rtol=1e-5, atol=0, err_msg=f"{pass_begin} + {passes}")


def test_welford_reference_against_float64():
    """ref_welford from an empty record, and continuing a record, is the float64 mean and sum of squared deviations of the
    luminance, to 1e-5 relative (mean) and 1e-4 relative (M2); the count is n + passes and the done bit stays."""
    rng = np.random.default_rng(2)
    s = rng.random((400, 48, 3), dtype=f32) * 3
    y = luminance(s.astype(np.float64))
    n0 = np.where(np.arange(400) % 2 == 0, 0, DONE).astype(np.uint32)
    n, mean, m2 = ref_welford(n0, np.zeros(400, f32), np.zeros(400, f32), s)
    assert (n == n0 + 48).all()
    np.testing.assert_allclose(mean, y.mean(axis=1), rtol=1e-5)
    np.testing.assert_allclose(m2, ((y - y.mean(axis=1, keepdims=True)) ** 2).sum(axis=1), rtol=1e-4)
    n2, mean2, m22 = ref_welford(n, mean, m2, s)          # 48 more passes: the statistics of all 96
    y2 = np.concatenate([y, y], axis=1)
    assert (n2 == n0 + 96).all()
    np.testing.assert_allclose(mean2, y2.mean(axis=1), rtol=1e-5)
    np.testing.assert_allclose(m22, ((y2 - y2.mean(axis=1, keepdims=True)) ** 2).sum(axis=1), rtol=1e-4)


def test_convergence_test_reference_against_float64():
    """ref_test at a test point is the float64 relative standard error of the mean luminance (floor below dark means) to 1e-5;
    pixels well clear of the threshold stop exactly when the float64 error is below it; pixels not at a test point, done pixels
    and pixels at or past pass_end keep their records, and the active ones are those not done and below pass_end."""
    rng = np.random.default_rng(3)
    N = 2000
    y = rng.random((N, 32)) * np.where(rng.random(N) < 0.2, 0.001, 1.0)[:, None]
    recs = np.zeros(N, crgpu.ADAPT_RECORD_DTYPE)
    n = rng.choice([15, 16, 17, 24, 32, 40, 48, 63, 64, 70], N)
    recs["n"] = n
    recs["n"][rng.random(N) < 0.2] |= np.uint32(DONE)
    recs["mean"] = y.mean(axis=1)
    recs["m2"] = ((y - y.mean(axis=1, keepdims=True)) ** 2).sum(axis=1)
    recs["err"] = np.inf
    thr = 0.05
    out, active = ref_test(recs, 16, 16, 64, thr, FLOOR)
    done0 = (recs["n"] & DONE) != 0
    tested = ~done0 & np.isin(n, [16, 32, 48])
    e64 = np.sqrt(recs["m2"].astype(np.float64) / (n - 1) / n) / np.maximum(recs["mean"].astype(np.float64), FLOOR)
    np.testing.assert_allclose(out["err"][tested], e64[tested], rtol=1e-5)
    clear = tested & (np.abs(e64 - thr) > 1e-4 * thr)
    assert (((out["n"] & DONE) != 0)[clear] == (e64 < thr)[clear]).all()
    assert out[~tested].tobytes() == recs[~tested].tobytes()
    assert (active == (((out["n"] & DONE) == 0) & (n < 64))).all()
    assert tested.sum() > 100 and (tested & active).sum() > 10 and (tested & ~active).sum() > 10


# ---- tile sets -------------------------------------------------------------------------------------------------------------------

def tiles_of(npix, W, H, tw=37, th=29):
    """a disjoint tile list of exactly npix pixels: the clipped tiles of the grid's right column and bottom row first, then the
    whole tiles, then the remainder as the top rows of one more grid tile and a part of the row below them"""
    cells = [(x, y, min(x + tw, W), min(y + th, H)) for y in range(0, H, th) for x in range(0, W, tw)]
    edge = [c for c in cells if c[2] - c[0] < tw or c[3] - c[1] < th]
    inner = [c for c in cells if c not in edge]
    out, total = [], 0
    for c in edge + inner:
        size = (c[2] - c[0]) * (c[3] - c[1])
        if total + size <= npix:
            out.append(c)
            total += size
        elif total < npix:
            x0, y0, x1, _ = c
            w, r = x1 - x0, npix - total
            if r // w:
                out.append((x0, y0, x1, y0 + r // w))
            if r % w:
                out.append((x0, y0 + r // w, x0 + r % w, y0 + r // w + 1))
            total = npix
        if total == npix:
            break
    assert total == npix, (npix, total)
    return out


def fb_index(pixels, W, H):
    """framebuffer index (row H-1-y) of each list pixel x | y << 16"""
    x = (pixels & 0xffff).astype(np.int64)
    y = (pixels >> 16).astype(np.int64)
    return (H - 1 - y) * W + x


def upload_nodes(W, H, spp=64):
    return crgpu.GpuScene(NODES, W, H, spp, 0)


# ---- GPU: K5 ---------------------------------------------------------------------------------------------------------------------

K5_W, K5_H = 640, 480
K5_NPIX = [1, 31, 32, 33, 255, 256, 257, 4095, 132 * 8 * 256 + 77]
ORDERS = [(1, 32), (1, 32), (8, 4), (4, 8), (2, 16), (8, 4), (16, 2), (32, 1)]       # (P, Q) of CRGPU_PATH_ORDER 0..7


@pytest.fixture(scope="module")
def k5_scene():
    g = upload_nodes(K5_W, K5_H)
    try:
        g.set_render(K5_W, K5_H, 2 ** 24 + 64, g.bounces)                           # room for passes past 2^24
        g.adaptive_reset()
        yield g
    finally:
        g.close()


def samples(rng, npix, passes):
    """random distinct radiance per (pixel, pass), with special values in single samples and in every pass of whole pixels"""
    s = rng.random((npix, passes, 4), dtype=f32) * f32(4)
    hit = rng.random((npix, passes, 3)) < 0.04
    s[..., :3][hit] = rng.choice(SPECIALS, int(hit.sum()))
    whole = rng.random(npix) < 0.03
    s[whole, :, :3] = rng.choice(SPECIALS, (int(whole.sum()), 1, 3))
    return s


def seeded_fb(rng, kind, H, W):
    if kind == 0:
        return np.zeros((H, W, 3), f32)
    fb = rng.random((H, W, 3), dtype=f32) * f32(2)
    if kind == 2:
        m = rng.random((H, W, 3)) < 0.05
        fb[m] = rng.choice(SPECIALS, int(m.sum()))
    return fb


def seeded_records(rng, H, W):
    recs = np.zeros((H, W), crgpu.ADAPT_RECORD_DTYPE)
    recs["n"] = rng.choice([0, 1, 2, 15, 16, 1000, 2 ** 24 - 5, 2 ** 24 + 1], (H, W)).astype(np.uint32)
    recs["n"][rng.random((H, W)) < 0.1] |= np.uint32(DONE)
    recs["mean"] = rng.random((H, W), dtype=f32)
    recs["m2"] = rng.random((H, W), dtype=f32) * f32(3)
    for k in ("mean", "m2"):
        m = rng.random((H, W)) < 0.05
        recs[k][m] = rng.choice(SPECIALS, int(m.sum()))
    recs["err"] = rng.choice(SPECIALS, (H, W))
    return recs


def k5_cases(P):
    """every pixel count with every pass count (1, P - 1, P, P + 1, 17), the first passes cycling through 0, 1, 999 and 2^24 - 3"""
    counts = sorted({c for c in (1, P - 1, P, P + 1, 17) if c >= 1})
    cases = [(npix, c) for npix in K5_NPIX for c in counts]
    return [(npix, c, (0, 1, 999, BIG_PASS)[i % 4]) for i, (npix, c) in enumerate(cases)]


@pytest.mark.gpu
@pytest.mark.parametrize("adaptive", [False, True], ids=["plain", "adaptive"])
@pytest.mark.parametrize("order", range(8))
def test_accumulate_against_the_replay(k5_scene, order, adaptive):
    """K5 under path order `order` adds given samples bit for bit as the float32 running average does, at pixel counts around a
    warp, a block and K5's whole grid and at pass counts around the order's pass group P, from 0, 1, 999 and 2^24 - 3 passes on
    cleared, seeded and NaN-seeded framebuffers; <ADAPTIVE> also leaves each record's count, mean and M2 of the Welford replay.
    Pixels and records outside the tile set keep their bytes."""
    g = k5_scene
    W, H = g.W, g.H
    P, _ = ORDERS[order]
    rng = np.random.default_rng(100 + 2 * order + adaptive)
    for i, (npix, passes, pass_begin) in enumerate(k5_cases(P)):
        what = f"order {order} {'adaptive' if adaptive else 'plain'}: {npix} pixels x {passes} passes from {pass_begin}"
        rects = tiles_of(npix, W, H)
        fb0 = seeded_fb(rng, i % 3, H, W)
        g.write(fb0)
        if adaptive:
            rec0 = seeded_records(rng, H, W)
            g.adaptive_write(rec0)
        s = samples(rng, npix, passes)
        pixels = g.accumulate_samples(rects, pass_begin, s, order=order, adaptive=adaptive)
        assert len(pixels) == npix and len(np.unique(pixels)) == npix, what
        idx = fb_index(pixels, W, H)
        inside = np.zeros(H * W, bool)
        inside[idx] = True
        got = g.read().reshape(-1, 3)
        flat0 = fb0.reshape(-1, 3)
        assert got[~inside].tobytes() == flat0[~inside].tobytes(), what + ": pixels outside the tiles changed"
        assert_bits(got[idx], ref_accumulate(flat0[idx], s[..., :3], pass_begin), what)
        if adaptive:
            rec = g.adaptive_records().reshape(-1)
            r0 = rec0.reshape(-1)
            assert rec[~inside].tobytes() == r0[~inside].tobytes(), what + ": records outside the tiles changed"
            n, mean, m2 = ref_welford(r0["n"][idx], r0["mean"][idx], r0["m2"][idx], s[..., :3])
            assert (rec["n"][idx] == n).all(), what + ": counts"
            assert_bits(rec["mean"][idx], mean, what + ": mean")
            assert_bits(rec["m2"][idx], m2, what + ": M2")
            assert rec["err"][idx].tobytes() == r0["err"][idx].tobytes(), what + ": K5 changed an error"


@pytest.mark.gpu
def test_accumulate_refusals(k5_scene):
    """Bad orders and passes, a bad tile list, more paths than the budget and <ADAPTIVE> without records are refused."""
    g = k5_scene
    one = np.zeros((1, 1, 4), f32)
    with pytest.raises(crgpu.CrgpuError, match="path order"):
        g.accumulate_samples([(0, 0, 1, 1)], 0, one, order=8)
    with pytest.raises(crgpu.CrgpuError, match="path order"):
        g.accumulate_samples([(0, 0, 1, 1)], 0, one, order=-2)
    with pytest.raises(crgpu.CrgpuError, match="passes"):
        g.accumulate_samples([(0, 0, 1, 1)], 2 ** 24 + 64, one)
    with pytest.raises(crgpu.CrgpuError, match="outside"):
        g.accumulate_samples([(0, 0, K5_W + 1, 1)], 0, np.zeros((K5_W + 1, 1, 4), f32))
    h = upload_nodes(64, 32)
    try:
        with pytest.raises(crgpu.CrgpuError, match="adaptive"):
            h.accumulate_samples([(0, 0, 1, 1)], 0, one, adaptive=True)
        h.set_max_paths(1024)
        with pytest.raises(crgpu.CrgpuError, match="paths in flight"):
            h.accumulate_samples([(0, 0, 64, 32)], 0, np.zeros((2048, 1, 4), f32))
        h.accumulate_samples([(0, 0, 64, 16)], 0, np.zeros((1024, 1, 4), f32))
    finally:
        h.close()


# ---- GPU: select and compaction ------------------------------------------------------------------------------------------------------

RULE = dict(min_passes=16, round_passes=16, pass_end=64)


def select_records(rng, pixels, W, H, k, rule):
    """records for a tile set whose pixels that stay active all hold k passes: pixels at k (with adversarial means and M2), done
    pixels at any count, and pixels at or past pass_end; pixels outside the set hold anything"""
    recs = seeded_records(rng, H, W).reshape(-1)
    idx = fb_index(pixels, W, H)
    m = len(idx)
    cls = rng.choice(4, m, p=[0.5, 0.25, 0.15, 0.10])
    n = np.full(m, k, np.uint32)
    n[cls == 1] = rng.choice([0, k, rule["min_passes"], 40, 48, rule["pass_end"], 1000], int((cls == 1).sum())).astype(np.uint32) | np.uint32(DONE)
    n[cls == 2] = rule["pass_end"] + rng.choice([0, 1, 16, 1000], int((cls == 2).sum())).astype(np.uint32)
    mean = rng.random(m, dtype=f32) * f32(0.5)
    m2 = rng.random(m, dtype=f32) * f32(0.05) * f32(max(k, 2))
    a = cls == 3                                              # adversarial statistics at count k
    mean[a] = rng.choice(np.array([0.0, -0.0, 0.001, 0.01, -0.5, np.nan, np.inf, 1e-40, 3e19], f32), int(a.sum()))
    m2[a] = rng.choice(np.array([0.0, -0.0, -1.0, np.nan, np.inf, 1e-45, 3e38], f32), int(a.sum()))
    n[a] = k
    recs["n"][idx] = n
    recs["mean"][idx] = mean
    recs["m2"][idx] = m2
    recs["err"][idx] = rng.choice(SPECIALS, m)
    return recs.reshape(H, W)


def check_select(g, rects, pixels, recs, rule, thr, what):
    """one select on the records: the active list, its counts and every record after it, against ref_test"""
    W, H = g.W, g.H
    idx = fb_index(pixels, W, H)
    g.adaptive_write(recs)
    flat = recs.reshape(-1)
    want, act = ref_test(flat[idx], rule["min_passes"], rule["round_passes"], rule["pass_end"], thr, FLOOR)
    counts = want["n"][act] & ~np.uint32(DONE)
    lo, hi = (int(counts.min()), int(counts.max())) if act.any() else (0xffffffff, 0)
    if lo != hi and act.any():
        with pytest.raises(crgpu.CrgpuError, match=f"hold {lo} to {hi} passes"):
            g.adaptive_select(rects, threshold=thr, floor=FLOOR, **rule)
        assert g.adaptive_records().tobytes() == recs.tobytes(), what + ": a refused select changed a record"
        return None
    active, glo, ghi = g.adaptive_select(rects, threshold=thr, floor=FLOOR, **rule)
    assert (glo, ghi) == (lo, hi), what
    assert np.array_equal(active, pixels[act]), what + f": active list of {len(active)}, want {int(act.sum())}"
    got = g.adaptive_records().reshape(-1)
    outside = np.ones(H * W, bool)
    outside[idx] = False
    assert got[outside].tobytes() == flat[outside].tobytes(), what + ": records outside the tile set changed"
    assert (got["n"][idx] == want["n"]).all(), what + ": done bits"
    assert_bits(got["err"][idx], want["err"], what + ": errors")
    assert got["mean"][idx].tobytes() == want["mean"].tobytes() and got["m2"][idx].tobytes() == want["m2"].tobytes(), what
    return act


SELECT_SIZES = [1, 31, 32, 33, 1023, 1024, 1025, 1024 ** 2 - 1, 1024 ** 2, 1024 ** 2 + 1]


@pytest.fixture(scope="module")
def hd_scene():
    g = upload_nodes(1920, 1080)
    try:
        g.adaptive_reset()
        yield g
    finally:
        g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("npix", SELECT_SIZES + ["1920x1080", "3840x2160"])
def test_select_against_the_replay(hd_scene, npix):
    """Select, scan and compaction on records at a count between test points, at the first and a later test point and below
    min_passes, with done
    pixels, pixels at and past pass_end and adversarial means and M2 (below floor, NaN, negative, infinite, subnormal, overflowing)
    and a threshold equal to one pixel's error: every record, the active list in list order and the least and largest count
    are the replay's.  The same records with one active pixel at another count (first, last, or amid the list) are refused and
    left byte-identical.  Sizes around a warp, a block, the scan's block of 1024 and its third level at 1024^2, up to whole
    1920x1080 and 3840x2160 frames."""
    if isinstance(npix, str):
        W, H = map(int, npix.split("x"))
        g = hd_scene if (W, H) == (1920, 1080) else upload_nodes(W, H)
        rects = [(0, 0, W, H)]
    else:
        g, W, H = hd_scene, 1920, 1080
        rects = tiles_of(npix, W, H)
    try:
        if (W, H) != (1920, 1080):
            g.adaptive_reset()
        pixels = g.accumulate_samples(rects, 0, np.zeros((sum((r[2] - r[0]) * (r[3] - r[1]) for r in rects), 0, 4), f32))
        rng = np.random.default_rng(len(pixels))
        idx = fb_index(pixels, W, H)
        for k in (40, 32, 16, 0):                             # between test points, at test points, below min_passes
            what = f"{len(pixels)} pixels at {k} passes"
            recs = select_records(rng, pixels, W, H, k, RULE)
            flat = recs.reshape(-1)
            # at a test point, a threshold equal to the error of a tested pixel: that pixel is not done (err < threshold)
            probe, _ = ref_test(flat[idx], RULE["min_passes"], RULE["round_passes"], RULE["pass_end"], 0.0, FLOOR)
            e = np.sort(probe["err"][(flat["n"][idx] == k) & np.isfinite(probe["err"]) & (probe["err"] > 0)])
            thr = float(e[len(e) // 2]) if k in (16, 32) and len(e) else 0.05
            act = check_select(g, rects, pixels, recs, RULE, thr, what)
            assert act is not None, what + ": expected a select with one count"
            if k in (16, 32) and len(e):
                at = np.nonzero((probe["err"] == f32(thr)))[0]
                assert len(at) and act[at].all(), what + ": a pixel whose error equals the threshold stopped"
            if len(pixels) < 2 or not act.any():
                continue
            for where in ("first", "last", "middle"):
                odd = recs.copy().reshape(-1)
                cand = np.nonzero(act)[0]
                j = cand[{"first": 0, "last": -1, "middle": len(cand) // 2}[where]]
                odd["n"][idx[j]] = np.uint32(k + 1)            # not a test point: it stays active at another count
                assert check_select(g, rects, pixels, odd.reshape(H, W), RULE, thr, what + f", one at {k + 1} ({where})") is None
    finally:
        if g is not hd_scene:
            g.close()


@pytest.mark.gpu
def test_a_round_with_no_active_pixel(hd_scene):
    """With every pixel done or at pass_end, a select finds none (least count 0xffffffff, largest 0) and changes no record, and a
    round renders nothing and returns pass_end as both its first and its last pass."""
    g = hd_scene
    W, H = g.W, g.H
    rects = tiles_of(1024 ** 2 + 1, W, H)
    rng = np.random.default_rng(9)
    recs = seeded_records(rng, H, W)
    recs["n"] = np.where(rng.random((H, W)) < 0.5, recs["n"] | np.uint32(DONE), np.uint32(RULE["pass_end"]))
    g.adaptive_write(recs)
    active, lo, hi = g.adaptive_select(rects, threshold=0.05, floor=FLOOR, **RULE)
    assert (len(active), lo, hi) == (0, 0xffffffff, 0)
    assert g.adaptive_records().tobytes() == recs.tobytes()
    fb = g.read().copy()
    d = g.adaptive_round(rects, RULE["min_passes"], RULE["round_passes"], 0.05, FLOOR, RULE["pass_end"])
    assert (d["active"], d["pass_begin"], d["pass_end"], d["paths"]) == (0, RULE["pass_end"], RULE["pass_end"], 0)
    assert g.read().tobytes() == fb.tobytes() and g.adaptive_records().tobytes() == recs.tobytes()


# ---- GPU: end to end at 1080p ----------------------------------------------------------------------------------------------------------

E2E = (1920, 1080, 48, 0)


@pytest.mark.gpu
def test_adaptive_1080p_end_to_end(tmp_path):
    """hdr at 1920x1080 and 48 spp with the CLI's rule (16, 16, floor 0.01) and a threshold that leaves three counts: rendered as one
    tile set and as a 64x64 tile grid, the two agree; each count's pixels equal render_tiles(rects, 0, k) of a second upload; and
    16 scattered 8x8 regions have the counts and errors of the replay on the oracle's per-sample radiance."""
    path = O.bundled_scene("hdr", str(tmp_path)) or NODES
    g, h = crgpu.GpuScene(path, *E2E), crgpu.GpuScene(path, *E2E)
    try:
        W, H, spp = g.W, g.H, g.samples
        whole = [(0, 0, W, H)]
        tiled = grid(W, H, 64, 64)
        rule = (16, 16)
        thr = calibrate(g, whole, 16, spp)
        runs = []
        for rects in (whole, tiled):
            g.clear()
            g.adaptive_reset()
            g.render_adaptive(rects, *rule, thr, FLOOR, spp)
            n, err = g.adaptive_read()
            img = g.read().copy()
            counts = sorted(np.unique(n).tolist())
            assert len(counts) >= 3, counts
            check_counts_exact(h, rects, img, n, f"{len(rects)} tiles")
            runs.append((img, n, err))
        for a, b in zip(*runs):
            assert a.tobytes() == b.tobytes()
        _, n, err = runs[0]
    finally:
        g.close()
        h.close()
    rng = np.random.default_rng(5)
    regions = [(int(x), int(y)) for x, y in zip(rng.integers(0, W - 8, 16), rng.integers(0, H - 8, 16))]
    o = O.OracleScene(path, *E2E)
    try:
        Ls, flags = [], []
        for x0, y0 in regions:
            st = o.camera_states(x0, y0, x0 + 8, y0 + 8, passes=(0, spp))
            res = o.path_step(st, 0, bounces=1 << 30)
            Ls.append(res["next"]["L"].reshape(64, spp, 3).astype(f32))
            flags.append(((res["flag"] != 0) | (st["pad"] != 0)).reshape(64, spp).any(axis=1))
    finally:
        o.close()
    L, flag = np.concatenate(Ls), np.concatenate(flags)
    assert flag.sum() <= max(1, L.shape[0] * spp * 1e-5), f"{flag.sum()} of {L.shape[0]} pixels have a flagged sample"
    want_n, want_err = replay(L, 16, 16, spp, thr, FLOOR)
    assert len(np.unique(want_n)) >= 2
    got_n = np.concatenate([n[H - y0 - 8:H - y0, x0:x0 + 8][::-1].reshape(-1) for x0, y0 in regions])
    got_err = np.concatenate([err[H - y0 - 8:H - y0, x0:x0 + 8][::-1].reshape(-1) for x0, y0 in regions])
    ok = ~flag
    assert np.array_equal(got_n[ok], want_n[ok])
    assert got_err[ok].tobytes() == want_err[ok].astype(f32).tobytes()
