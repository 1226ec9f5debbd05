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
