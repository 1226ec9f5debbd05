"""Cost of deforming meshes of a resident scene against reloading it (crgpu_scene_set_meshes, include/crgpu.h).

Cases (tests/test_gpu_mesh_edit.py builds the same deformations):
  hdr       Venus (274,243 triangles, one instance) in hdr.json, at bench.py's frame size
  statues   Venus under 55 instances in statues.json
  teapot    one teapot mesh (3 instances) in scene.json
  grid      a generated 1,002,528-triangle grid mesh
  reload    crloader_load_json_buf of the deformed scene + crgpu_prepare + crgpu_scene_create_prepared (what the edit costs without
            set_meshes)
  first     the first set_meshes of the mesh (it also creates the scene's pairs and instance blocks and the mesh's region)
  later     later set_meshes calls (alternating the deformed and the original geometry)
Each edit is also checked against a fresh upload of the deformed scene at a small size (frame and traced records, bit for bit).
Then bench.py runs once on the unedited default workload and its frame CRC is printed.  Times are host wall clock around calls that
end in a device synchronise; medians of --reps.  The bytes are the pairs block (uploaded pairs, top region, mesh regions) plus the
instance block (last-instance table, item records), and the call's scratch without the builder's own, from crgpu_api.cu's layout.

    python tools/mesh_edit_probe.py [--reps 10] [--out results.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "c-ray_b200"), os.path.join(ROOT, "tests")]

import crgpu  # noqa: E402
import crscene  # noqa: E402
import test_gpu_mesh_edit as M  # noqa: E402
import test_gpu_scene_edit as T  # noqa: E402

CASES = {"hdr": ("hdr", ["venusscaled.obj"], (1920, 1080, 1000, 32)), "statues": ("statues", ["venusscaled.obj"], (1920, 1080, 64, 30)),
         "teapot": ("scene", ["teapot.obj"], (1920, 1080, 64, 50)), "grid": (None, ["grid.obj"], (1920, 1080, 64, 8))}


def a256(b):
    return (b + 255) // 256 * 256


def layout_bytes(flat, meshes):
    """(pairs block + instance block, scratch without the builder's own) bytes of a first set_meshes of `meshes` on a scene uploaded
    from `flat`."""
    A = crscene.arrays(flat)
    internal = sum((int(b["node_count"]) - 1) // 2 for i, b in enumerate(A["bvhs"]) if b["node_count"] > 1)
    n_inst = len(A["instances"])
    regions = sum(max(1, int(A["meshes"][m]["poly_count"]) - 1) for m in meshes)
    blocks = (internal + max(1, n_inst - 1) + regions) * 64 + (a256(n_inst * 4) + n_inst * 64 if n_inst else 0)
    scratch = 0
    for m in meshes:
        mesh = A["meshes"][m]
        n = int(mesh["poly_count"])
        polys = A["polys"][int(mesh["poly_offset"]):int(mesh["poly_offset"]) + n]
        v = polys["v"].ravel()
        nn = polys["n"][polys["has_normals"] != 0].ravel()
        t = polys["t"][(polys["t"][:, 0] != -1)].ravel() if mesh["texcoord_count"] else np.zeros(0, np.int32)
        rng = lambda x, w: a256((int(x.max()) - int(x.min()) + 1) * w if len(x) else 0)
        scratch += (a256(n * 44) + rng(v, 12) + rng(nn, 12) + rng(t, 8) + a256(n * 24) + a256(n * 12) + a256(max(1, n - 1) * 64)
                    + a256(n * 4) + a256(n * 48) + a256(n * 4) + a256(n) + a256(n * 80))
    scratch += (a256(len(A["bvhs"]) * 24) + a256(n_inst * 24) + a256(n_inst * 12) + a256(n_inst * 4) + a256(n_inst * 128)
                + a256(max(1, n_inst - 1) * 64) + a256(n_inst * 4))
    return blocks, scratch


def docs(case):
    name, files, cfg = CASES[case]
    sa, sb = M.Assets(), M.Assets()
    if case == "grid":
        k = 708
        xs = np.arange(k + 1) / k
        X, Y = np.meshgrid(xs, xs, indexing="ij")
        sa.write("grid.obj", M.grid_obj(k, np.zeros_like(X)))
        sb.write("grid.obj", M.grid_obj(k, 3.0 * np.sin(6.0 * X) * np.cos(5.0 * Y)))
        doc = M.gen_scene(["grid.obj"])
    else:
        doc = T.scene_json(name)
        for i, f in enumerate(files):
            sb.write(f, M.deform_obj(sb.original(f), seed=1 + i))
    return doc, sa, sb, cfg


def wall(fn):
    t = time.perf_counter()
    fn()
    return (time.perf_counter() - t) * 1e3


def reload_ms(doc, asset_dir, cfg):
    L = crgpu.lib()
    L.crgpu_prepare.argtypes = [C.POINTER(crgpu.FlatScene), C.POINTER(C.c_void_p)]
    L.crgpu_prepared_free.argtypes = [C.c_void_p]
    t = time.perf_counter()
    b = M.LoadedFrom(doc, asset_dir, *cfg)
    p, h = C.c_void_p(), C.c_void_p()
    crgpu._check(L.crgpu_prepare(C.byref(b.flat), C.byref(p)), "crgpu_prepare")
    crgpu._check(L.crgpu_scene_create_prepared(p, 0, C.byref(h)), "crgpu_scene_create_prepared")
    ms = (time.perf_counter() - t) * 1e3
    L.crgpu_scene_destroy(h)
    L.crgpu_prepared_free(p)
    b.free()
    return ms


def probe(case, reps):
    doc, sa, sb, cfg = docs(case)
    a, b = M.LoadedFrom(doc, sa.dir, *cfg), M.LoadedFrom(doc, sb.dir, *cfg)
    ch = M.changed_meshes(a, b)
    n_inst = len(a.instances)
    polys = int(sum(crscene.arrays(a.flat)["meshes"]["poly_count"][ch]))
    block_bytes, scratch_bytes = layout_bytes(a.flat, ch)
    g = a.upload()
    first = wall(lambda: g.set_meshes(b.flat, ch))
    later = [wall(lambda k=k: g.set_meshes((a if k % 2 == 0 else b).flat, ch)) for k in range(reps)]
    g.close()
    reload = [reload_ms(doc, sb.dir, cfg) for _ in range(max(3, reps // 3))]
    a.free()
    b.free()
    small = (160, 90, 2, 8)                       # the same edit at a small size, against a fresh upload
    a, b = M.LoadedFrom(doc, sa.dir, *small), M.LoadedFrom(doc, sb.dir, *small)
    g = a.upload()
    g.set_meshes(b.flat, ch)
    T.assert_same_as_fresh(g, b, T.ray_set(b.camera, n=4096))
    g.close()
    a.free()
    b.free()
    sa.close()
    sb.close()
    return dict(case=case, meshes=ch, triangles=polys, instances=n_inst, size=cfg[:2],
                set_meshes_first_ms=first, set_meshes_ms=float(np.median(later)), reload_prepare_create_ms=float(np.median(reload)),
                pairs_instance_blocks_bytes=block_bytes, scratch_bytes=scratch_bytes, checked=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--no-bench", action="store_true")
    ap.add_argument("--out", default=None, help="also write the results to this JSON file")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True).stdout.strip()
    print("gpu:", gpu)
    out = dict(gpu=gpu, cases=[])
    for case in CASES:
        r = probe(case, args.reps)
        out["cases"].append(r)
        print(json.dumps(r))
    if not args.no_bench:
        r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", "1", "--warmup", "1"],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, cwd=ROOT)
        line = [x for x in r.stdout.splitlines() if x.startswith("{")][-1]
        out["bench_frame_crc32"] = json.loads(line).get("frame_crc32")
        print("bench frame_crc32 (unedited hdr):", out["bench_frame_crc32"])
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
