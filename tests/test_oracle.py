"""CPU tests: the oracle (oracle/cray_oracle.c) against the reference's own outputs.

The golden files were produced by the unmodified reference built with -ffp-contract=off
(tests/golden/make_golden.py).  The bar for the oracle is BIT-EXACT fp32.
"""
import os

import numpy as np
import pytest

import oracle_lib as O
from conftest import GOLDEN, GOLDEN_SCENES, GOLDEN_FLAT, BUILT


def test_sampler_kat_bit_exact():
    k = np.fromfile(os.path.join(GOLDEN, "kat.bin"), dtype=np.uint32).reshape(-1, 16)
    assert len(k) == 10
    for row in k:
        pix, p, mp = (int(v) for v in row[:3])
        mine = O.sampler_kat(pix, p, mp, 13)
        assert np.array_equal(row[3:], mine.view(np.uint32)), (pix, p, mp)


def test_sampler_seed_wraps_in_32_bits():
    # sampler.c:42: pixelIndex * maxPasses + pass is uint32 arithmetic
    a = O.sampler_kat(2073599, 2499, 2500, 4)
    wrapped = (2073599 * 2500 + 2499) & 0xFFFFFFFF
    b = O.sampler_kat(wrapped, 0, 1, 4)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_draw_range_inclusive_one():
    # random.c:17: 2^-32 * (float)u32 rounds up to exactly 1.0f for u32 >= 2^32-128
    v = O.sampler_kat(0, 0, 1, 4096)
    assert v.min() >= 0.0 and v.max() <= 1.0


@pytest.mark.parametrize("name", GOLDEN_FLAT)
def test_framebuffer_bit_exact(name):
    sc = O.OracleScene(os.path.join(GOLDEN, name + ".crscene"))
    ref = np.fromfile(os.path.join(GOLDEN, name + ".f32"), dtype=np.float32).reshape(sc.H, sc.W, 3)
    img = sc.render(threads=4)
    assert np.array_equal(img.view(np.uint32), ref.view(np.uint32))
    sc.close()


@pytest.mark.parametrize("name", GOLDEN_FLAT)
def test_hit_records_bit_exact(name):
    sc = O.OracleScene(os.path.join(GOLDEN, name + ".crscene"))
    h = np.fromfile(os.path.join(GOLDEN, name + ".hits.bin"), dtype=O.HIT_KAT_DTYPE)
    assert len(h) == 96
    for i, r in enumerate(h):
        m = sc.trace_kat(int(r["x"]), int(r["y"]), i % sc.s.prefs.sample_count)
        assert r.tobytes() == m.tobytes(), (name, i)
    sc.close()


@pytest.mark.parametrize("name", GOLDEN_FLAT)
def test_tiles_and_pass_ranges_compose(name):
    """Tile size, thread count and splitting the passes never change a pixel (renderer.c:271-320)."""
    sc = O.OracleScene(os.path.join(GOLDEN, name + ".crscene"))
    ref = np.fromfile(os.path.join(GOLDEN, name + ".f32"), dtype=np.float32).reshape(sc.H, sc.W, 3)
    img = np.zeros_like(ref)
    spp = sc.s.prefs.sample_count
    for (pb, pc) in ((0, 3), (3, spp - 3)):
        for y0 in range(0, sc.H, 16):
            for x0 in range(0, sc.W, 16):
                sc.render(threads=1, tile=(x0, y0, min(x0 + 16, sc.W), min(y0 + 16, sc.H)), passes=(pb, pc), rgb=img)
    assert np.array_equal(img.view(np.uint32), ref.view(np.uint32))
    sc.close()


def test_counters_consistent():
    sc = O.OracleScene(os.path.join(GOLDEN, "g_legacy.crscene"))
    _, c = sc.render(threads=2, count=True)
    assert c["paths"] == sc.W * sc.H * sc.s.prefs.sample_count
    assert c["paths"] <= c["rays"] <= c["paths"] * sc.s.prefs.bounces
    assert c["max_depth"] <= sc.s.prefs.bounces and c["max_stack"] <= 64
    assert c["node_pairs"] > 0 and c["tri_tests"] > 0 and c["sphere_tests"] > 0 and c["inst_visits"] > 0
    sc.close()


def test_srgb8_matches_reference_formula():
    rgb = np.array([0.0, 0.001, 0.0031308, 0.2, 0.5, 1.0, 1.5, 7.0, 0.99999], dtype=np.float32)
    rgb = np.resize(rgb, 9).astype(np.float32)
    out = np.zeros(9, dtype=np.uint8)
    O.lib().cro_to_srgb8(rgb.ctypes.data, out.ctypes.data, 3)
    exp = []
    for c in rgb:
        s = 12.92 * c if c <= 0.0031308 else 1.055 * c ** 0.4166666667 - 0.055
        exp.append(min(int(min(s * 255.0, 255.0)), 255))
    assert np.abs(out.astype(int) - np.array(exp)).max() <= 1


@pytest.mark.parametrize("name,W,H,spp,b", [("hdr", 96, 54, 4, 32), ("scene", 80, 50, 4, 4), ("refraction", 64, 36, 2, 512), ("venus", 40, 64, 4, 25),
                                            ("alphanode", 96, 60, 8, 0), ("fence", 96, 60, 8, 0), ("glowmetal", 96, 60, 8, 0),
                                            ("statues", 96, 60, 8, 0), ("uvsphere", 96, 60, 8, 0)])
def test_bundled_scenes_against_reference_framebuffers(name, W, H, spp, b, tmp_path):
    """Bundled input/*.json scenes: the oracle's frame is bit-exact to the one the strict reference rendered (its SHA-256 is
    stored in tests/golden/ref_frames.sha256.json; scenes/_built/ref_*.f32 holds the frame itself where build() made it)."""
    scene = O.bundled_scene(name, tmp_path)
    if not scene:
        pytest.skip("bundled scenes: neither scenes/_built nor oracle/_ref/input present")
    sc = O.OracleScene(scene, W, H, spp, b)
    img = sc.render(threads=os.cpu_count())
    assert O.frame_digest(img) == O.reference_digest(name, W, H, spp, b)
    ref_path = os.path.join(BUILT, f"ref_{name}_{W}x{H}x{spp}_b{b}.f32")
    if os.path.exists(ref_path):
        ref = np.fromfile(ref_path, dtype=np.float32).reshape(H, W, 3)
        assert np.array_equal(img.view(np.uint32), ref.view(np.uint32))
    sc.close()


@pytest.mark.parametrize("name,W,H,spp,b", [("hdr", 1920, 1080, 2, 32), ("venus", 2560, 1600, 1, 25), ("refraction", 1920, 1080, 1, 512)])
def test_full_size_frames_bit_exact_against_live_reference(name, W, H, spp, b, tmp_path):
    """BASELINE.json configs C2 / C4 / C3 at their full image sizes (few spp): the strict reference build, run here, and the
    oracle produce the same fp32 frame bit for bit.  (The GPU suite then checks bands of these frames against the oracle.)"""
    import subprocess
    from conftest import ROOT
    ref_exe = os.path.join(ROOT, "oracle", "_ref", "cray_ref_strict")
    scene = os.path.join(BUILT, name + ".crscene")
    if not (os.path.exists(ref_exe) and os.path.exists(scene)):
        pytest.skip("needs oracle/_ref (built where /root/reference exists)")
    out = str(tmp_path / "ref.f32")
    r = subprocess.run([ref_exe, "render", os.path.join("input", name + ".json"), str(W), str(H), str(spp), str(b), str(os.cpu_count() or 1), "0", "0", out],
                       cwd=os.path.join(ROOT, "oracle", "_ref"), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-1000:]
    ref = np.fromfile(out, dtype=np.float32).reshape(H, W, 3)
    sc = O.OracleScene(scene, W, H, spp, b)
    img = sc.render(threads=os.cpu_count())
    assert np.array_equal(img.view(np.uint32), ref.view(np.uint32))
    sc.close()


def test_glass_total_internal_reflection_with_draw_of_exactly_one(tmp_path):
    """glass.c:47 declares `refracted` uninitialised and reads it when refract() failed (total internal reflection) AND the
    reflect/refract draw is exactly 1.0f (129 of 2^32 draws): the compiled reference scatters along (0, 0, <stale stack word>).
    Known occurrence (round-1 judge): hdr.json 1920x1080x1000spp, pixel x=165 y(up)=768, pass 576, bounce 2.  The oracle and the
    device DEFINE that case as a reflection (DESIGN.md deviation #3), so (a) the sample is finite, (b) the pixel differs from the
    strict reference by at most that one sample's share, (c) every pixel around it stays bit-identical to the reference."""
    scene = O.bundled_scene("hdr", tmp_path)
    if not scene:
        pytest.skip("bundled scenes: neither scenes/_built nor oracle/_ref/input present")
    W, H, spp, b = 1920, 1080, 1000, 32
    sc = O.OracleScene(scene, W, H, spp, b)
    one = np.zeros((H, W, 3), np.float32)
    sc.render(threads=1, tile=(165, 768, 166, 769), passes=(576, 1), rgb=one)       # running average from zero: (0*575 + L)/576
    sample = one[H - 1 - 768, 165].astype(np.float64) * 577.0
    assert np.isfinite(sample).all(), sample
    img = np.zeros((H, W, 3), np.float32)
    sc.render(threads=os.cpu_count(), tile=(160, 764, 172, 772), rgb=img)
    blk = img[H - 772:H - 764, 160:172]
    assert np.isfinite(blk).all()
    ref_path = os.path.join(BUILT, f"ref_hdr_{W}x{H}x{spp}_b{b}.f32")
    if os.path.exists(ref_path):
        ref = np.fromfile(ref_path, dtype=np.float32).reshape(H, W, 3)[H - 772:H - 764, 160:172]
        same = (blk.view(np.uint32) == ref.view(np.uint32)).all(axis=2)
        assert same.sum() == same.size - 1 and not same[772 - 1 - 768, 165 - 160], same
        # one of 1000 samples took another direction after its third hit: bounded by that sample's own radiance / spp
        assert np.abs(blk[772 - 1 - 768, 5].astype(np.float64) - ref[772 - 1 - 768, 5]).max() <= (np.abs(sample).max() + 64.0) / spp
    sc.close()


@pytest.mark.parametrize("name", GOLDEN_FLAT)
def test_closest_hit_records_match_reference_hits(name):
    """cro_closest_hit on the camera rays of the reference's own known-answer records: semantics 0 (the reference's traversal)
    reproduces instIndex, polyIndex and distance bit for bit, and semantics 1 (the device traversal's slab test) gives the same
    records on those rays."""
    sc = O.OracleScene(os.path.join(GOLDEN, name + ".crscene"))
    h = np.fromfile(os.path.join(GOLDEN, name + ".hits.bin"), dtype=O.HIT_KAT_DTYPE)
    rays = np.concatenate([h["o"], h["d"]], axis=1)
    ref, c0 = sc.closest_hit(rays, O.SEM_REFERENCE)
    assert np.array_equal(ref["inst"], h["instIndex"])
    assert np.array_equal(ref["poly"], h["polyIndex"])
    hit = h["instIndex"] >= 0
    assert hit.any()
    assert np.array_equal(ref["t"][hit].view(np.uint32), h["distance"][hit].view(np.uint32))
    assert (ref["t"][~hit] == np.float32(np.finfo(np.float32).max)).all()
    dev, c1 = sc.closest_hit(rays, O.SEM_DEVICE)
    assert dev.tobytes() == ref.tobytes()
    assert c0["rays"] == c1["rays"] == len(rays) and c0["tri_tests"] + c0["sphere_tests"] > 0
    # the batch is split over threads: the records and the totals do not depend on how
    one, c1b = sc.closest_hit(rays, O.SEM_DEVICE, threads=1)
    assert one.tobytes() == dev.tobytes() and c1b == c1
    sc.close()


def test_device_semantics_cull_zero_direction_components_exactly():
    """A horizon ray (d.y == +0) through the middle of the scene: the reference's slab test turns the y axis into NaNs and drops it,
    entering every box the ray's x/z projection crosses; semantics 1 culls that axis exactly and visits fewer node pairs, with
    the same hit.  Also -0 and a denormal direction component, which overflow 1/d to +-inf the same way."""
    sc = O.OracleScene(os.path.join(GOLDEN, "g_legacy.crscene"))
    o = np.fromfile(os.path.join(GOLDEN, "g_legacy.hits.bin"), dtype=O.HIT_KAT_DTYPE)["o"][0]     # the camera position
    for dy in (0.0, -0.0, 1e-45):
        rays = np.array([[o[0], o[1], o[2], 0.3, dy, 1.0]], np.float32)
        r0, c0 = sc.closest_hit(rays, O.SEM_REFERENCE, threads=1)
        r1, c1 = sc.closest_hit(rays, O.SEM_DEVICE, threads=1)
        assert c1["node_pairs"] < c0["node_pairs"], (dy, c0, c1)
        assert r0.tobytes() == r1.tobytes(), (dy, r0, r1)
    sc.close()


def test_path_rays_start_with_the_camera_ray():
    """cro_trace_region lists every ray of every bounce of a region's paths; the first ray of a path is its camera ray."""
    sc = O.OracleScene(os.path.join(GOLDEN, "g_single.crscene"))
    rays = sc.path_rays(3, 2, 4, 3, passes=(1, 1))
    k = sc.trace_kat(3, 2, 1)
    assert 1 <= len(rays) <= sc.s.prefs.bounces
    assert np.array_equal(rays[0].view(np.uint32), np.concatenate([k["o"], k["d"]]).view(np.uint32))
    rec, _ = sc.closest_hit(rays[:1], O.SEM_REFERENCE)
    assert rec["inst"][0] == k["instIndex"] and rec["poly"][0] == k["polyIndex"]
    sc.close()


def test_zero_bounces_is_black():
    """prefs.bounces == 0: pathTrace's loop never runs (pathtrace.c:36-59) — the reference renders an all-zero frame
    (checked against cray_ref_strict with "bounces": 0 in the JSON)."""
    sc = O.OracleScene(os.path.join(GOLDEN, "g_single.crscene"))
    sc.s.prefs.bounces = 0
    img = sc.render(threads=2)
    assert not img.any()
    sc.close()


# ------------------------------------------------------------------------------------------------ path steps and libm semantics
def chain_frame(o, semantics):
    """The frame of cro_render, rebuilt from cro_path_step one bounce at a time from the camera states, and the running average
    of renderer.c:288-291 in numpy fp32.  Returns (frame, per-pixel count of flagged samples)."""
    W, H, spp, B = o.W, o.H, o.s.prefs.sample_count, o.s.prefs.bounces
    cur = o.camera_states(0, 0, W, H, semantics=semantics)
    n = len(cur)
    L = np.zeros((n, 3), np.float32)
    flag = cur["pad"] != 0
    idx = np.arange(n)
    for depth in range(B):
        if len(cur) == 0:
            break
        r = o.path_step(cur, depth, semantics=semantics)
        flag[idx] |= r["flag"] != 0
        dead = r["alive"] == 0
        L[idx[dead]] = r["next"]["L"][dead]
        idx, cur = idx[~dead], r["next"][~dead]
    assert len(cur) == 0 or B == 0
    Ls = L.reshape(H, W, spp, 3)
    out = np.zeros((H, W, 3), np.float32)
    for p in range(spp):
        out = (out * np.float32(p)) + Ls[:, :, p]
        out = out * (np.float32(1) / np.float32(p + 1))
    return out[::-1], flag.reshape(H, W, spp).sum(axis=2)[::-1]


def _synthetic_flat(tmp_path):
    from test_gpu_trace import _write_synthetic, _flatten
    d = str(tmp_path)
    return {n: _flatten(p, os.path.join(d, n + ".crscene")) for n, p in _write_synthetic(os.path.join(d, "syn")).items()}


def test_path_step_chain_is_the_render(tmp_path):
    """cro_path_step is pathTrace's loop body: chained one bounce at a time from the camera states, it reproduces cro_render's
    framebuffer bit for bit (semantics 0) on every golden and synthetic scene, and cro_render_sem's (semantics 1)."""
    scenes = {n: os.path.join(GOLDEN, n + ".crscene") for n in GOLDEN_FLAT}
    scenes.update(_synthetic_flat(tmp_path))
    for name, path in scenes.items():
        o = O.OracleScene(path)
        ref = o.render(threads=os.cpu_count())
        img, _ = chain_frame(o, O.SEM_REFERENCE)
        assert np.array_equal(img.view(np.uint32), ref.view(np.uint32)), name
        ref1, fl1 = o.render_sem(O.SEM_DEVICE)
        img1, fl = chain_frame(o, O.SEM_DEVICE)
        assert np.array_equal(img1.view(np.uint32), ref1.view(np.uint32)), name
        assert np.array_equal(fl, fl1), name
        r0, f0 = o.render_sem(O.SEM_REFERENCE)
        assert np.array_equal(r0.view(np.uint32), ref.view(np.uint32)) and not f0.any(), name
        o.close()


def test_non_finite_weight_reaches_radiance():
    """A weight that is not finite makes the reference's finalColor NaN at every hit, emissive or not (pathtrace.c:44): both
    semantics must say so, with the radiance flag set, although semantics 1 skips the add of zero emission for finite weights."""
    o = O.OracleScene(os.path.join(GOLDEN, "g_single.crscene"))
    st = o.camera_states(0, 0, o.W, o.H, passes=(0, 1))
    r = o.path_step(st, 0, semantics=O.SEM_REFERENCE)
    hit = r["rec"]["inst"] >= 0
    assert hit.any()
    st = st[hit]
    for w in (np.inf, -np.inf, np.nan):
        st["weight"] = w
        for sem in (O.SEM_REFERENCE, O.SEM_DEVICE):
            r = o.path_step(st, 1, semantics=sem)
            assert (r["next"]["has_l"] == 1).all() and np.isnan(r["next"]["L"]).any(axis=1).all(), (w, sem)
    o.close()


_F32 = np.finfo(np.float32)


def _sweeps():
    """(function, x, y) sweeps over the inputs where fp32 libm results go wrong"""
    rng = np.random.default_rng(5)
    f = np.float32
    specials = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, -1e-45, _F32.tiny, -_F32.tiny, _F32.max, -_F32.max, 1.0, -1.0], f)

    def around(c, k=64):                      # floats within k ulps of c
        c = f(c)
        up, dn = [c], [c]
        for _ in range(k):
            up.append(np.nextafter(up[-1], f(np.inf)))
            dn.append(np.nextafter(dn[-1], f(-np.inf)))
        return np.array(up + dn, f)

    out = []
    trig = [specials, rng.uniform(-10, 10, 20000).astype(f), (rng.uniform(-1, 1, 5000) * f(1e30)).astype(f),
            (10.0 ** rng.uniform(3, 38, 5000)).astype(f) * np.where(rng.integers(0, 2, 5000) == 1, f(1), f(-1))]
    trig += [around(k * np.pi / 2) for k in range(-8, 9)]
    trig = np.concatenate(trig)
    out += [("sin", trig, None), ("cos", trig, None)]
    out.append(("tan", np.concatenate([specials, rng.uniform(-10, 10, 20000).astype(f)] + [around(k * np.pi / 2, 256) for k in (-3, -1, 1, 3)]), None))
    vals = np.concatenate([specials, (np.array([0, 1, 2, 4, 8, -0.5], f)[:, None] * np.ones(1, f)).ravel(), rng.normal(size=4000).astype(f),
                           (10.0 ** rng.uniform(-40, 38, 4000)).astype(f) * np.where(rng.integers(0, 2, 4000) == 1, f(1), f(-1))])
    X, Y = np.meshgrid(vals[:60], vals[:60])
    out.append(("atan2", np.concatenate([X.ravel(), vals]), np.concatenate([Y.ravel(), vals[::-1]])))
    unit = np.concatenate([specials, around(1.0, 256), around(-1.0, 256), around(0.0, 64), rng.uniform(-1, 1, 20000).astype(f),
                           np.array([1.0000001, -1.0000001, 2.0, -2.0], f)])
    out += [("acos", unit, None), ("asin", unit, None)]
    logs = np.concatenate([specials, np.array([2 ** -149, 2 ** -140, 2 ** -127, 2 ** -126, 1e-40], f), around(1.0, 256),
                           (10.0 ** rng.uniform(-45, 38.5, 20000)).astype(f), -np.abs(rng.normal(size=100)).astype(f)])
    out += [("log", logs, None), ("log10", logs, None)]
    px = np.concatenate([specials, around(1.0, 32), np.array([-2.0, -0.5, -1.0, -3.0, 0.5, 2.0, 10.0], f),
                         (10.0 ** rng.uniform(-45, 38, 3000)).astype(f), rng.uniform(0, 1, 3000).astype(f)])
    py = np.concatenate([specials, np.array([2.0, 3.0, -2.0, 0.5, 2.4, 0.4166666667, -0.1332047592, -0.0755148492, 5.0, 1e6, -1e6,
                                             999999.94, -999999.94, 1000000.06, 3e7, -3e7], f), around(1e6, 8), rng.normal(size=200).astype(f) * 40])
    X, Y = np.meshgrid(px, py)
    out.append(("pow", X.ravel(), Y.ravel()))
    near1 = around(1.0, 2048)
    big = np.concatenate([rng.uniform(-1e6, 1e6, 2048), np.array([1e5, -1e5, 4e5, -7e5])]).astype(f)
    out.append(("pow", np.resize(near1, len(near1) * 8), np.resize(big, len(near1) * 8)))
    return out


def _exact(fn, x, y):
    """the correctly rounded fp32 result, from numpy.longdouble (x87 80-bit) evaluation"""
    X = x.astype(np.longdouble)
    with np.errstate(all="ignore"):
        if fn == "atan2":
            r = np.arctan2(X, y.astype(np.longdouble))
        elif fn == "pow":
            r = np.power(X, y.astype(np.longdouble))
        else:
            r = {"sin": np.sin, "cos": np.cos, "tan": np.tan, "log": np.log, "log10": np.log10, "acos": np.arccos, "asin": np.arcsin}[fn](X)
        return r.astype(np.float32)


def same_bits(a, b):
    """bit-identical fp32, except that any NaN equals any NaN"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def test_device_libm_semantics_are_correctly_rounded_unless_flagged():
    """Semantics 1's stand-ins (the device's fp64-then-round evaluation) give the correctly rounded fp32 result of the same
    function, from an 80-bit evaluation, everywhere they do not raise the near-tie flag; and they raise it rarely."""
    assert np.finfo(np.longdouble).nmant >= 63, "needs x87 long double"
    total = flagged = 0
    for fn, x, y in _sweeps():
        got, flag = O.libm(fn, O.SEM_DEVICE, x, y)
        ok = same_bits(got, _exact(fn, x, y))
        bad = np.nonzero(~ok & ~flag)[0]
        assert len(bad) == 0, (fn, x[bad[:5]], None if y is None else y[bad[:5]], got[bad[:5]], _exact(fn, x, y)[bad[:5]])
        total += len(x)
        flagged += int(flag.sum())
    print(f"libm sweeps: {flagged} of {total} evaluations flagged")
    assert flagged <= total * 1e-3
    # exact results far from any boundary are not flagged
    v, fl = O.libm("pow", O.SEM_DEVICE, np.array([1.5, 4.0], np.float32), np.array([1.0, 0.5], np.float32))
    assert not fl.any() and v[0] == 1.5 and v[1] == 2.0
