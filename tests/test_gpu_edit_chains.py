"""Seeded random chains of edits on one resident GPU scene, next to a host-side model of what that scene should be.

Every edit entry point (include/crgpu.h) is tested alone and in short fixed orders elsewhere; here a chain of 20 steps mixes them, so
that the bookkeeping they share (the pairs block with its top region and mesh regions, the instance, geometry, materials, shading and
views blocks, view 0's framebuffer and the host mirrors later calls trust) is reached in orders no fixed test takes.

The model is a JSON document with its asset directory (OBJ / MTL / texture files, rewritten by mesh deformations), the render
settings, the view cameras, whether the scene is armed and its path budget.  Each step changes the model and makes the matching call
on the device scene.  After every step the device scene must render its frame, trace a ray set (records and P/T/S/I counts) and
render its views bit for bit as a fresh upload of the model; every edit must leave the framebuffer's bytes as they were.  Every
CHECKPOINT steps and at the end the model is saved as a flat scene and the edited device scene is compared with the CPU oracle in
device semantics: K2 records and instrumented counts on path rays and test_gpu_trace.adversarial_rays, and the frame outside
flagged pixels.  A failure names the seed, the step and the operations up to it; replay(seed, steps) runs one chain to a step.

Added meshes without polys stay without instances: the scene loader refuses a scene that instances one, so no model holds it.

CPU: the generator's determinism, its coverage of every operation and composition, and crgpu_prepare on every model state.  GPU:
the chains.  CRGPU_CHAIN_STEPS lengthens the chains for soak runs (default 20).
"""
import copy
import ctypes as C
import os
import random
import shutil
import tempfile
import time

import numpy as np
import pytest

import crgpu
import crscene
import oracle_lib as O
from conftest import GOLDEN, SUMMARY_LINES
from test_gpu_add_objects import with_mesh, with_sphere
from test_gpu_instance_list import duplicated, removed
from test_gpu_mesh_edit import Assets, LoadedFrom, changed_meshes, deform_obj
from test_gpu_render_settings import Src, _At
from test_gpu_scene_edit import Loaded, assert_same_as_fresh, full, ray_set, scene_json
from test_gpu_shade import FLAG_SHARE, Tally
from test_gpu_shading_edit import prepared_shading, recolour_doc, set_shading_rc, shading_variant
from test_gpu_trace import adversarial_rays, check_counters, check_records
from test_gpu_views import cameras, grid, single
from test_gpu_worlds import World, _instance_transforms, prepare_error
from test_oracle import same_bits

SEEDS = range(12)
STEPS = int(os.environ.get("CRGPU_CHAIN_STEPS", "20"))
CHECKPOINT = 6
BAD_ARGUMENT, UNSUPPORTED = -3, -4
# the start scene of each chain: a random world of test_gpu_worlds (its seed), or a bundled scene
START = {0: 0, 1: 1, 2: 2, 3: "hdr", 4: 4, 5: 5, 6: 6, 7: "refraction", 8: 8, 9: 9, 10: 10, 11: 12}
BUNDLED_CFG = {"hdr": (64, 36, 2, 32), "refraction": (64, 36, 2, 16)}
SCALE = {"hdr": 0.05, "refraction": 40.0}             # the size of an added object and of a move, by start scene (worlds: 1)
OPS = ["set_camera", "set_instances", "set_instance_list", "set_meshes", "set_shading", "add_objects", "set_views", "set_render",
       "refused", "interrupted"]
WEIGHTS = [2, 2, 2.5, 3, 1.5, 2, 1, 1.5, 1.5, 1]
EDITS = OPS[:7]                                        # what an interrupted render is followed by
RECORD = ("poly_offset", "poly_count", "material_offset", "material_count", "texcoord_count", "bvh")   # what set_meshes keeps
# the orders of edits the chains must reach (checked on the operation logs)
COMPOSITIONS = ["add as the first geometry edit", "add after a deformed uploaded mesh and an earlier add",
                "set_meshes on an added mesh after a later add", "list outgrowing every earlier list after a geometry edit",
                "set_meshes on an empty list, then instances back", "empty mesh added, then more edits",
                "set_shading after an add", "resize with several views after an add, then the cached tile set",
                "edit after a refused edit", "interrupted armed render", "render in flight drained by an edit"]


# ---- the model -------------------------------------------------------------------------------------------------------------------

class Model:
    """What the device scene should be: JSON document, asset directory, render settings, view cameras (bytes, view 0 is the scene
    camera), armed, path budget."""

    def __init__(self, seed, root):
        self.seed = seed
        self.rng = random.Random(31000 + seed)
        self.start = START[seed]
        self.dir = os.path.join(root, "chain%d" % seed)
        if isinstance(self.start, str):
            self.assets = Assets()
            self.dir = self.assets.dir
            self.doc = copy.deepcopy(scene_json(self.start))
            self.cfg = BUNDLED_CFG[self.start]
            self.scale = SCALE[self.start]
        else:
            w = World(os.path.join(root, "worlds"), self.start)
            assert w.refusal is None, (self.start, w.refusal)
            self.assets = None
            shutil.copytree(w.dir, self.dir)
            self.doc = copy.deepcopy(w.doc)
            W, H, spp, b = w.cfg
            self.cfg = (W, H, min(spp, 4), b)
            self.scale = 1.0
        for name in ("ico.obj", "ico.mtl", "rgba.png", "gray.png", "rgb.png"):
            self.write(name, open(os.path.join(GOLDEN, "assets", name), "rb").read().decode("latin-1"))
        self.write("empty.obj", "o empty\nv 0 0 0\n")
        self.armed = seed % 3 == 1
        self.max_paths = [None, 1024, 4096][seed % 3 if seed % 2 else 0]
        self.views = None                                  # None: one view, the scene camera
        self.cams = None
        self.rects = None                                  # the tile set of the views checks, kept while it fits
        self.added = 0                                     # files written for added meshes

    def write(self, name, text):
        if self.assets and os.path.dirname(name):
            self.assets.write(name, text)                  # a file in a linked subdirectory: the directory is copied first
            return
        path = os.path.join(self.dir, name)
        if os.path.lexists(path):
            os.unlink(path)                                # a link into the bundled input/ is replaced, never written through
        with open(path, "w", encoding="latin-1") as f:
            f.write(text)

    def read(self, name):
        return open(os.path.join(self.dir, name), encoding="latin-1").read()

    def load(self):
        """the model as a flat scene at its settings (test_gpu_scene_edit.Loaded), the bounce limit 0 included"""
        W, H, spp, b = self.cfg
        if self.assets:
            x = LoadedFrom(self.doc, self.dir, W, H, spp, b)
        else:
            x = Loaded(self.doc, W, H, spp, b, cwd=self.dir, asset_path=self.dir)
        Src(x.flat, None).camera(self.cfg)
        x.cfg = self.cfg
        return x

    def objects(self):
        s = self.doc["scene"]
        return [("sphere", k, p) for k, p in enumerate(s.get("primitives", []))] + \
               [("mesh", k, m) for k, m in enumerate(s.get("meshes", []))]

    def mesh_files(self):
        """the OBJ files of the document's meshes that load and have faces"""
        out = []
        for m in self.doc["scene"].get("meshes", []):
            f = m["fileName"]
            p = os.path.join(self.dir, f)
            if f not in out and os.path.exists(p) and any(ln.startswith("f ") for ln in self.read(f).split("\n")):
                out.append(f)
        return out

    def move(self, r):
        return {"type": "translate", "x": round(r.uniform(-1, 1) * self.scale, 4), "y": round(r.uniform(-0.5, 0.5) * self.scale, 4),
                "z": round(r.uniform(-1, 1) * self.scale, 4)}

    def close(self):
        if self.assets:
            self.assets.close()


# ---- the operations: each changes the model and returns (what the log says, the device call) --------------------------------------
# A device call is act(g, cur, new) -> return code, where cur / new are the model loaded before / after the step.

def op_camera(m, r):
    m.doc["camera"].setdefault("transforms", []).extend([{"type": "rotateY", "degrees": round(r.uniform(-3, 3), 2)}, m.move(r)])
    return "set_camera", lambda g, cur, new: g.set_camera(new.camera)


def op_instances(m, r):
    for _, _, ob in m.objects():
        for inst in ob.get("instances", []):
            if m.assets:                                   # a bundled scene: its placement, re-placed about the object's origin
                kind = r.choice(["plain", "mirror1", "mirror2", "aniso", "quarter", "odd", "half_exact"])
                tf = [t for t in _instance_transforms(r, kind)[1] if t["type"] != "translate"]
                inst["transforms"] = [t for t in inst.get("transforms", []) if t["type"] == "translate"] + tf + [m.move(r)]
            else:
                inst["transforms"] = _instance_transforms(r)[1]
    return "set_instances", lambda g, cur, new: g.set_instances(new.instances)


def op_list(m, r):
    objs = m.objects()
    on = [o for o in objs if o[2].get("instances")]
    off = [o for o in objs if not o[2].get("instances") and not (o[0] == "mesh" and o[2]["fileName"] == "empty.obj")]
    choices = ["dup", "many", "remove", "retarget", "revive", "empty"] if on else ["revive"]
    what = r.choice(choices if off or not on else [c for c in choices if c != "revive"])
    if what in ("dup", "many"):
        kind, k, ob = r.choice(on)
        for _ in range(1 if what == "dup" else r.randrange(20, 60)):
            if kind == "mesh" and r.random() < 0.5:
                m.doc = duplicated(m.doc, None, ob["fileName"], round(r.uniform(-1, 1) * m.scale, 4))
                ob = next(x for x in m.doc["scene"]["meshes"] if x["fileName"] == ob["fileName"] and x.get("instances"))
            else:
                extra = copy.deepcopy(r.choice(ob["instances"]))
                extra["transforms"] = extra.get("transforms", []) + [m.move(r)]
                ob["instances"].append(extra)
    elif what == "remove":
        kind, k, ob = r.choice(on)
        if kind == "sphere" and r.random() < 0.5:
            m.doc = removed(m.doc, k)
        else:
            ob["instances"] = ob["instances"][:r.randrange(len(ob["instances"]))]
    elif what == "retarget":                               # one instance moves to another object of its kind
        kind, k, ob = r.choice(on)
        others = [o for o in objs if o[0] == kind and o[2] is not ob and not (kind == "mesh" and o[2]["fileName"] == "empty.obj")]
        if others:
            inst = ob["instances"].pop(r.randrange(len(ob["instances"])))
            r.choice(others)[2].setdefault("instances", []).append(inst)
    elif what == "revive":                                 # an object without an instance gets one
        kind, k, ob = r.choice(off)
        src = [i for o in on if o[0] == kind for i in o[2]["instances"]]
        ob["instances"] = [copy.deepcopy(r.choice(src)) if src else {"transforms": [m.move(r)]}]
    else:
        for _, _, ob in objs:
            ob["instances"] = []
    return "set_instance_list(%s)" % what, lambda g, cur, new: g.set_instance_list(new.instances)


def _material_names(m, obj_text):
    for ln in obj_text.split("\n"):
        if ln.startswith("mtllib "):
            p = os.path.join(m.dir, ln.split(None, 1)[1].strip())
            if os.path.exists(p):
                return [x.split(None, 1)[1].strip() for x in open(p, encoding="latin-1") if x.startswith("newmtl ")]
    return []


def op_meshes(m, r, files=None):
    files = files or m.mesh_files()
    picked = r.sample(files, min(len(files), r.choice([1, 1, 2])))
    kinds = []
    for f in picked:
        text = m.read(f)
        have = {k for k in ("vn", "vt") if any(ln.startswith(k + " ") for ln in text.split("\n"))}
        names = _material_names(m, text)
        used = [ln for ln in text.split("\n") if ln.startswith("usemtl ")]
        kind = r.choice(["v", "v", "mat"] + sorted(have))
        if kind == "mat" and (len(names) < 2 or not used):
            kind = "v"
        if kind == "mat":                                  # poly materials within the mesh's range: usemtl names rotated
            rot = {a: names[(i + 1) % len(names)] for i, a in enumerate(names)}
            text = "\n".join("usemtl " + rot.get(ln[7:].strip(), ln[7:].strip()) if ln.startswith("usemtl ") else ln for ln in text.split("\n"))
        else:
            text = deform_obj(text, kind, r.randrange(1 << 30), amp=r.choice([0.002, 0.01, 0.05]))
        m.write(f, text)
        kinds.append("%s:%s" % (f, kind))

    def act(g, cur, new):
        return g.set_meshes(new.flat, changed_meshes(cur, new))
    return "set_meshes(%s)" % ",".join(kinds), act


def op_shading(m, r):
    if m.assets and r.random() < 0.5:
        m.doc = recolour_doc(m.start, m.doc)
        what = "recolour"
    else:
        m.doc = shading_variant(m.doc, m.dir, r.randrange(1 << 20))
        what = "redrawn"
    return "set_shading(%s)" % what, lambda g, cur, new: g.set_shading(new.flat)


def op_add(m, r):
    parts = []
    for _ in range(r.choice([1, 1, 2])):
        what = r.choice(["mesh", "mesh", "empty", "sphere"])
        if what == "sphere" and m.doc["scene"].get("primitives"):
            k = r.randrange(len(m.doc["scene"]["primitives"]))
            rad = r.choice([None, round(r.uniform(0.2, 1.0) * m.scale, 4)])
            m.doc = with_sphere(m.doc, k, tuple(m.move(r)[a] for a in "xyz"), rad, instanced=r.random() < 0.8)
            parts.append("sphere")
        elif what == "empty":
            m.doc = with_mesh(m.doc, {"fileName": "empty.obj", "bsdf": "lambertian", "instances": []}, instanced=False)
            parts.append("empty mesh")
        else:                                              # a mesh of its own file, so that later deformations reach it alone
            src = r.choice(m.mesh_files() + ["ico.obj"])
            m.added += 1
            name = "add%d.obj" % m.added
            m.write(name, m.read(src))
            entry = {"fileName": name, "bsdf": r.choice(["lambertian", "metal", "plastic", "glass"]),
                     "instances": [{"transforms": [{"type": "scaleUniform", "scale": m.scale * r.choice([0.3, 1.0])}]}]}
            m.doc = with_mesh(m.doc, entry, tuple(m.move(r)[a] for a in "xyz"), instanced=r.random() < 0.85)
            parts.append("mesh")
    return "add_objects(%s)" % "+".join(parts), lambda g, cur, new: g.add_objects(new.flat)


def op_views(m, r):
    n = r.choice([k for k in (1, 2, 3, 4) if k != (m.views or 1)])
    m.views = n                                            # the cameras are made from the loaded model (finish)
    return "set_views(%d)" % n, None


def op_render(m, r):
    W, H, spp, b = m.cfg
    if r.random() < 0.6:
        W, H = r.randrange(16, 97), r.randrange(16, 97)
    if (m.views or 1) > 1 and r.random() < 0.5:           # larger: the views' cached tile set still fits
        W, H = r.randrange(W, 97), r.randrange(H, 97)
    spp = r.randrange(1, 5)
    b = r.choice([0, 1, 2, 5, 8, b])
    resize = (W, H) != m.cfg[:2]
    m.cfg = (W, H, spp, b)
    return "set_render(%dx%dx%d b%d%s)" % (W, H, spp, b, "" if resize else ", same size"), None


REFUSALS = ["instance count", "camera size", "mesh record", "material count", "list kind", "list count", "add fewer",
            "render zero", "views size"]


def refusal(g, cur, what):
    """one refused call on the scene (the model does not change): its return code"""
    L = crgpu.lib()
    A = crscene.arrays(cur.flat)
    inst = np.ascontiguousarray(A["instances"])
    if what == "instance count":
        return L.crgpu_scene_set_instances(g.handle, inst.ctypes.data, len(inst) + 1)
    if what == "camera size":
        cam = crgpu.Camera.from_buffer_copy(cur.camera)
        cam.width += 1
        return L.crgpu_scene_set_camera(g.handle, C.byref(cam))
    if what == "mesh record":
        meshes = A["meshes"].copy()
        keep = A["meshes"].copy()
        meshes["material_count"][0] += 1
        C.memmove(cur.flat.meshes, meshes.ctypes.data, meshes.nbytes)
        try:
            idx = np.zeros(1, np.uint32)
            return L.crgpu_scene_set_meshes(g.handle, C.byref(cur.flat), idx.ctypes.data, 1)
        finally:
            C.memmove(cur.flat.meshes, keep.ctypes.data, keep.nbytes)
    if what == "material count":
        f = crgpu.FlatScene.from_buffer_copy(cur.flat)
        f.material_count -= 1
        return L.crgpu_scene_set_shading(g.handle, C.byref(f))
    if what == "list kind":
        bad = inst.copy()
        bad["kind"][0] = 2
        return L.crgpu_scene_set_instance_list(g.handle, bad.ctypes.data, len(bad))
    if what == "list count":                              # refused before any instance is read
        one = np.zeros(1, dtype=crscene.INSTANCE)
        return L.crgpu_scene_set_instance_list(g.handle, (inst if len(inst) else one).ctypes.data, 4194305)
    if what == "add fewer":
        f = crgpu.FlatScene.from_buffer_copy(cur.flat)
        if f.mesh_count:
            f.mesh_count -= 1
        else:
            f.sphere_count -= 1
        return L.crgpu_scene_add_objects(g.handle, C.byref(f))
    if what == "render zero":
        return L.crgpu_scene_set_render(g.handle, 0, g.H, g.samples, g.bounces, None, g.view_count())
    cam = crgpu.Camera.from_buffer_copy(cur.camera)
    cam.height += 1
    return L.crgpu_scene_set_views(g.handle, C.byref(cam), 1)


def raw_set_meshes(g, flat, meshes):
    idx = np.asarray(meshes, np.uint32)
    return crgpu.lib().crgpu_scene_set_meshes(g.handle, C.byref(flat), idx.ctypes.data, len(idx))


def refusals_for(cur):
    f = cur.flat
    out = ["camera size", "material count", "list count", "render zero", "views size"]
    if f.instance_count:
        out += ["instance count", "list kind"]
    if f.mesh_count:
        out.append("mesh record")
    if f.mesh_count or f.sphere_count:
        out.append("add fewer")
    return out


# ---- a chain ---------------------------------------------------------------------------------------------------------------------

class ChainFailure(AssertionError):
    pass


def _draw(m, r, step, steps, geom_done, instances, last):
    """the operation of a step: weighted, with a geometry edit forced into the last step of a chain without one, and an empty list
    followed by a mesh edit (the ninst == 0 branch), then by a list edit, more often than the weights alone would give"""
    if step == steps - 1 and not geom_done:
        return r.choice(["set_meshes", "add_objects"])
    if instances == 0 and last != "set_meshes" and m.mesh_files() and r.random() < 0.7:
        return "set_meshes"
    if instances == 0 and last == "set_meshes" and r.random() < 0.6:
        return "set_instance_list"
    op = r.choices(OPS, WEIGHTS)[0]
    if op == "set_meshes" and not m.mesh_files():
        op = "add_objects"
    return op


MAKE = {"set_camera": op_camera, "set_instances": op_instances, "set_instance_list": op_list, "set_meshes": op_meshes,
        "set_shading": op_shading, "add_objects": op_add, "set_views": op_views, "set_render": op_render}


def run_chain(seed, steps=STEPS, root=None, device=False, stats=None):
    """Run chain `seed` for `steps` steps: on the model alone (device=False: the operation log and crgpu_prepare of every state), or
    on the model and a device scene, checking after every step.  Returns the operation log [(op, label)] and the compositions it reached."""
    own = root is None
    root = root or tempfile.mkdtemp(prefix="crgpu_chain_")
    m = Model(seed, root)
    r = m.rng
    log, facts = [], set()
    cur = m.load()
    g = None
    upload_meshes = cur.flat.mesh_count
    # the history the compositions are read from
    h = dict(geom=0, adds=0, deformed_uploaded=False, added_mesh_at={}, max_list=len(cur.instances), regions=False,
             empty_then_meshes=False, refused=False)
    try:
        if device:
            g = cur.upload(max_paths=m.max_paths)
            if m.armed:
                g.enable_stop()
        for step in range(steps):
            op = _draw(m, r, step, steps, h["geom"] > 0, cur.flat.instance_count, log[-1][0] if log else None)
            saved = (copy.deepcopy(m.doc), m.cfg, m.views, {f: m.read(f) for f in m.mesh_files()})
            inner, act, expect, label = None, None, 0, op
            if op == "refused":
                why = r.choice(refusals_for(cur))
                label = "refused(%s)" % why
                expect = UNSUPPORTED if why == "list count" else BAD_ARGUMENT
                act = lambda g, cur, new, why=why: refusal(g, cur, why)
            else:
                kind = op
                if op == "interrupted":
                    kind = r.choice([e for e in EDITS if e != "set_meshes" or m.mesh_files()])
                label, act = MAKE[kind](m, r)
                if op == "interrupted":
                    inner, label = kind, "interrupted %s %s" % ("armed" if m.armed else "in flight", label)
            new = cur if op == "refused" else m.load()
            kind = inner or op
            resize = kind == "set_render" and new.cfg[:2] != cur.cfg[:2]
            # cameras of the views: made from the loaded model at its size
            if kind == "set_views" or (kind == "set_render" and m.views and m.views > 1 and resize):
                n = m.views
                cams = cameras(m.doc, _At(Src(new.flat, None), new.cfg), n)
                m.views = n
                m.cams = [bytes(c) for c in cams]
                act = (lambda g, cur, new, cams=cams: g.set_views(cams)) if kind == "set_views" else \
                      (lambda g, cur, new, cams=cams: g.set_render(*new.cfg, cams))
            elif kind == "set_render":
                act = (lambda g, cur, new: g.set_render(*new.cfg, [new.camera])) if resize else (lambda g, cur, new: g.set_render(*new.cfg))
            if kind == "set_camera" and m.views and m.views > 1:
                m.cams[0] = bytes(new.camera)
            # a deformation whose tree the host builder cannot fit in 2n - 1 nodes: refused, and the model goes back
            ch = changed_meshes(cur, new) if kind == "set_meshes" else []
            if kind == "set_meshes":
                B = crscene.arrays(new.flat)
                A = crscene.arrays(cur.flat)
                for f in RECORD:
                    assert np.array_equal(A["meshes"][f], B["meshes"][f]), f"chain {seed} step {step}: {label} changed {f} of a mesh"
                big = [k for k in ch if B["bvhs"]["node_count"][B["meshes"]["bvh"][k]] > 2 * B["meshes"]["poly_count"][k] - 1]
                if big:
                    expect, label = UNSUPPORTED, label + " refused: a tree of more than 2n - 1 nodes"
            if kind == "set_shading" and prepared_shading(new.flat)[0]:
                expect = prepared_shading(new.flat)[0]
                label += " refused by crgpu_prepare (%d)" % expect
            refused_flat = None
            if expect and op != "refused":                 # the device is given the refused state; the model goes back
                refused_flat = new
                act = (lambda g, cur, new, x=refused_flat, ch=ch: raw_set_meshes(g, x.flat, ch)) if kind == "set_meshes" else \
                      (lambda g, cur, new, x=refused_flat: set_shading_rc(g, x.flat))
                m.doc, m.cfg, m.views = saved[0], saved[1], saved[2]
                for f, text in saved[3].items():
                    m.write(f, text)
                new = m.load()
            # the compositions this step reaches
            ok = expect == 0
            if kind in ("set_meshes", "add_objects") and ok:
                if kind == "add_objects":
                    if h["geom"] == 0:
                        facts.add(COMPOSITIONS[0])
                    if h["deformed_uploaded"] and h["adds"]:
                        facts.add(COMPOSITIONS[1])
                    for k in range(cur.flat.mesh_count, new.flat.mesh_count):
                        h["added_mesh_at"][k] = h["adds"]
                    h["adds"] += 1
                    if "empty" in label:
                        facts.add(COMPOSITIONS[5])
                    if h["empty_then_meshes"] and new.flat.instance_count:
                        facts.add(COMPOSITIONS[4])
                    if new.flat.instance_count > h["max_list"] and h["regions"]:
                        facts.add(COMPOSITIONS[3])
                else:
                    if any(k < upload_meshes for k in ch):
                        h["deformed_uploaded"] = True
                    if any(k in h["added_mesh_at"] and h["added_mesh_at"][k] < h["adds"] - 1 for k in ch):
                        facts.add(COMPOSITIONS[2])
                    if new.flat.instance_count == 0:
                        h["empty_then_meshes"] = True
                h["geom"] += 1
                h["regions"] = True
            if kind == "set_instance_list" and ok:
                if new.flat.instance_count > h["max_list"] and h["regions"]:
                    facts.add(COMPOSITIONS[3])
                if h["empty_then_meshes"] and new.flat.instance_count:
                    facts.add(COMPOSITIONS[4])
            if kind == "set_shading" and ok and h["adds"]:
                facts.add(COMPOSITIONS[6])
            if (m.views or 1) > 1:                         # the views' tile set: the last one while it fits
                Wn, Hn = new.cfg[:2]
                fits = m.rects is not None and all(x1 <= Wn and y1 <= Hn for _, _, x1, y1 in m.rects)
                if fits and resize and h["adds"]:
                    facts.add(COMPOSITIONS[7])
                m.rects = m.rects if fits else grid(Wn, Hn)
            if op != "refused" and h["refused"]:
                facts.add(COMPOSITIONS[8])
            if op == "interrupted":
                facts.add(COMPOSITIONS[9] if m.armed else COMPOSITIONS[10])
            h["refused"] = op == "refused" or expect != 0
            h["max_list"] = max(h["max_list"], new.flat.instance_count)
            log.append((op, label))
            try:
                if not device:
                    err = _prepare_error(new)
                    assert err is None, f"chain {seed} step {step} ({label}): crgpu_prepare refuses the model: {err}"
                else:
                    try:
                        _device_step(m, g, cur, new, op, act, expect, resize, stats)
                        if step % CHECKPOINT == CHECKPOINT - 1 or step == steps - 1:
                            _checkpoint(g, new, root, seed, step, stats)
                    except AssertionError as e:
                        ops = "\n".join("  %2d %s" % (i, x[1]) for i, x in enumerate(log))
                        raise ChainFailure(f"chain {seed} (replay({seed}, {step + 1})), step {step}, {label}: {e}\n"
                                           f"operations:\n{ops}") from e
            finally:
                if refused_flat is not None:
                    refused_flat.free()
            if new is not cur:
                cur.free()
                cur = new
            if stats is not None:
                stats["steps"] += 1
    finally:
        if g is not None:
            g.close()
        cur.free()
        m.close()
        if own:
            shutil.rmtree(root, ignore_errors=True)
    return log, facts


def _prepare_error(x):
    fd, path = tempfile.mkstemp(suffix=".crscene")
    os.close(fd)
    try:
        L = crgpu.lib()
        L.crscene_save.argtypes = [C.POINTER(crgpu.FlatScene), C.c_char_p]
        assert L.crscene_save(C.byref(x.flat), path.encode()) == 0
        return prepare_error(path)
    finally:
        os.unlink(path)


def _device_step(m, g, cur, new, op, act, expect, resize, stats):
    """the step's device call and the checks against a fresh upload of the model"""
    W, H = g.W, g.H
    keep = op != "interrupted" and not resize
    if keep:                                               # passes on top of what the framebuffer holds: the edit keeps them
        g.render_tile(0, 0, W, H, 0, 1)
        before = g.read().copy()
    if op == "interrupted":
        g.render_tile(0, 0, W, H, flags=crgpu.FLAG_ASYNC)
        if m.armed:
            g.request_stop()
    rc = act(g, cur, new)
    if op == "interrupted" and m.armed:
        g.clear_stop()
    if expect:
        assert rc == expect, f"the call returned {rc}, expected {expect}"
    if keep:
        assert g.read().tobytes() == before.tobytes(), "the edit changed the framebuffer"
    if resize:
        img = g.read()
        assert img.shape == (new.cfg[1], new.cfg[0], 3) and not img.any(), "a new size must start from a zeroed framebuffer"
    rays = ray_set(new.camera, n=4096, seed=stats["steps"])
    assert_same_as_fresh(g, new, rays)
    stats["rays"] += len(rays)
    nv = g.view_count()
    assert nv == (m.views or 1), (nv, m.views)
    if nv > 1:
        for v in range(nv):
            g.view_clear(v)
        g.render_views(m.rects)
        fresh = new.upload()
        try:
            for v in range(nv):
                want = single(fresh, crgpu.Camera.from_buffer_copy(m.cams[v]), m.rects)[0]
                assert g.view_read(v).tobytes() == want.tobytes(), f"view {v} of {nv} differs from its single render"
        finally:
            fresh.close()


def _checkpoint(g, new, root, seed, step, stats):
    """the edited device scene against the oracle (device semantics) on the model's flat scene"""
    path = os.path.join(root, "chain%d_step%d.crscene" % (seed, step))
    L = crgpu.lib()
    L.crscene_save.argtypes = [C.POINTER(crgpu.FlatScene), C.c_char_p]
    assert L.crscene_save(C.byref(new.flat), path.encode()) == 0
    o = O.OracleScene(path)
    try:
        bw, bh = min(o.W, 32), min(o.H, 24)
        x0, y0 = (o.W - bw) // 2, (o.H - bh) // 2
        p = o.path_rays(x0, y0, x0 + bw, y0 + bh, passes=(0, min(2, o.s.prefs.sample_count)))
        a, _, _ = adversarial_rays(o, np.random.default_rng(seed * 1000 + step), n=256)
        rays = np.concatenate([p.reshape(-1, 6), a]).astype(np.float32)
        r1, c1 = o.closest_hit(rays, O.SEM_DEVICE)
        rec, perm, misses, st = g.trace_rays(rays, count=1)
        check_records(g, rec, perm, misses, r1, "oracle checkpoint")
        check_counters(st, c1, len(rays), "oracle checkpoint")
        img = full(g)
        ref, flagged = o.render_sem(O.SEM_DEVICE)
    finally:
        o.close()
        os.unlink(path)
    spp = new.cfg[2]
    tally = Tally(f"chain {seed}, frame samples")
    tally.add(img.shape[0] * img.shape[1] * spp, flagged.sum())
    assert tally.flagged <= max(1, tally.states * FLAG_SHARE), f"{tally.flagged} of {tally.states} samples flagged"
    bad = np.nonzero((~same_bits(img, ref)).any(axis=2) & (flagged == 0))
    assert len(bad[0]) == 0, f"oracle checkpoint: {len(bad[0])} unflagged pixels differ, first rows {bad[0][:5]} cols {bad[1][:5]}"
    if stats is not None:
        stats["checkpoints"] += 1
        stats["oracle rays"] += len(rays)
        stats["samples"] += tally.states
        stats["flagged"] += tally.flagged


def replay(seed, steps):
    """re-run chain `seed` on the device up to and including step `steps` - 1"""
    return run_chain(seed, steps, device=True, stats=_new_stats())


def _new_stats():
    return {"steps": 0, "rays": 0, "checkpoints": 0, "oracle rays": 0, "samples": 0, "flagged": 0}


def _needs(seed):
    if isinstance(START[seed], str):
        scene_json(START[seed])                            # skips where the bundled scenes are not available


# ---- CPU -------------------------------------------------------------------------------------------------------------------------

_LOGS = {}


def chain_log(seed):
    """the operation log of a chain on the model alone, run once per session"""
    _needs(seed)
    if seed not in _LOGS:
        _LOGS[seed] = run_chain(seed)
    return _LOGS[seed]


def test_generator_is_deterministic():
    for seed in (0, 7):
        _needs(seed)
        a = run_chain(seed, 8)
        b = run_chain(seed, 8)
        assert a[0] == b[0] and a[1] == b[1]
        assert chain_log(seed)[0][:7] == a[0][:7]                # the last step of a chain may be forced to a geometry edit


@pytest.mark.parametrize("seed", SEEDS)
def test_every_model_state_passes_prepare(seed):
    """run_chain on the model alone asserts crgpu_prepare on every state, so a device refusal can only be the edit's fault; it also
    asserts that a deformation keeps every mesh record"""
    log, _ = chain_log(seed)
    assert len(log) == STEPS
    assert any(op in ("set_meshes", "add_objects") for op, _ in log), "a chain without a geometry edit"


def test_every_operation_and_composition_occurs():
    ops, facts, refusals = set(), set(), set()
    for seed in SEEDS:
        log, f = chain_log(seed)
        ops |= {op for op, _ in log}
        facts |= f
        refusals |= {lab[len("refused("):-1] for op, lab in log if op == "refused"}
    assert ops == set(OPS), set(OPS) - ops
    assert facts == set(COMPOSITIONS), set(COMPOSITIONS) - facts
    assert len(refusals) >= 6, refusals


# ---- GPU -------------------------------------------------------------------------------------------------------------------------

TOTALS = _new_stats()
TOTALS["seconds"] = 0.0


@pytest.mark.gpu
@pytest.mark.parametrize("seed", SEEDS)
def test_edit_chain(seed):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    _needs(seed)
    t = time.time()
    stats = _new_stats()
    try:
        run_chain(seed, device=True, stats=stats)
    finally:
        TOTALS["seconds"] += time.time() - t
        for k in ("steps", "rays", "checkpoints", "oracle rays", "samples", "flagged"):
            TOTALS[k] += stats[k]


@pytest.mark.gpu
def test_edit_chain_totals():
    if not TOTALS["steps"]:
        pytest.skip("no chain ran")
    line = (f"edit chains: {TOTALS['steps']} steps in {TOTALS['seconds']:.0f} s, {TOTALS['rays']} rays against fresh uploads, "
            f"{TOTALS['checkpoints']} oracle checkpoints over {TOTALS['oracle rays']} rays and {TOTALS['samples']} frame samples "
            f"({TOTALS['flagged']} flagged)")
    print(line)
    SUMMARY_LINES.append(line)
