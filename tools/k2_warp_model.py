#!/usr/bin/env python3
"""Offline SIMT model of the traversal kernel's warp scheduling (K2, c-ray_b200/csrc/crgpu_trace.cu) — CPU only.

ncu says K2 is issue-bound with ~15 of 32 lanes active per warp instruction, so the next gains are in lane utilisation.
GPU time is scarce (180 min a round); this tool screens scheduling policies before any of them is written in CUDA:

  1. the oracle (bit-identical to the reference) records, for every ray of a region, the event sequence of the kernel's
     state machine: top-level child-pair step, instance step, bottom-level child-pair step with its triangle count
     (oracle/cray_oracle.c: cro_trace_region);
  2. rays are grouped per bounce in the order the wavefront presents them (pass-major, then pixel order; survivors keep
     their order), and a warp-level simulator replays a policy: every "round" costs an instruction weight and is executed
     by the lanes that take part in it; the figure of merit is ncu's `smsp__thread_inst_executed_per_inst_executed`,
     i.e. sum(active lanes x instructions) / sum(instructions), plus the total instruction count per ray (the time proxy
     for an issue-bound kernel);
  3. the instruction weights are rough SASS counts of the current kernel; they are checked against the three measured
     points of round 1 (flat loop 9.6, + persistent refill 11.6, + phase separation 15.0 active lanes on the bounce-1
     launch of hdr.json).

usage: tools/k2_warp_model.py [scene=hdr] [W H x0 y0 x1 y1 passes]     (defaults: hdr 1920x1080, a 512x64 strip, 2 passes)
       tools/k2_warp_model.py --orders [scene=hdr] [W H x0 y0 x1 y1 passes]
                                      the path orders of CRGPU_PATH_ORDER (crgpu_wave.cuh) over the region as ONE batch's pixel set
                                      (defaults: hdr 1920x1080, the 64x64 tile at (896, 512), 8 passes)
"""
import ctypes as C
import os
import sys
from collections import defaultdict

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "tests"), os.path.join(ROOT, "c-ray_b200")]
import oracle_lib as O                                                    # noqa: E402

# instruction weights (SASS instructions per round, rough counts from cuobjdump of k_trace<false,3>)
W_NODE, W_TRI, W_INST, W_REFILL, W_WRITEBACK, W_LOOP = 70, 48, 95, 45, 30, 14


def load_traces(scene, W, H, x0, y0, x1, y1, passes, with_keys=False):
    L = O.lib()
    L.cro_trace_region.restype = C.c_size_t
    L.cro_trace_region.argtypes = [C.POINTER(O.Scene)] + [C.c_int] * 6 + [C.c_void_p, C.c_size_t]
    sc = O.OracleScene(os.path.join(ROOT, "scenes", "_built", scene + ".crscene"), W, H, 1000, 32)
    cap = 1 << 30
    buf = np.empty(cap, dtype=np.uint8)
    n = L.cro_trace_region(C.byref(sc.s), x0, y0, x1, y1, 0, passes, buf.ctypes.data, cap)
    sc.close()
    raw = buf[:n]
    rays = defaultdict(list)          # depth -> [(order key, events, origin+direction)]
    pos = 0
    while pos + 36 <= n:
        x, y, p, d = np.frombuffer(raw[pos:pos + 8].tobytes(), dtype="<u2")
        cnt = int(np.frombuffer(raw[pos + 8:pos + 12].tobytes(), dtype="<u4")[0])
        od = np.frombuffer(raw[pos + 12:pos + 36].tobytes(), dtype="<f4")
        ev = raw[pos + 36:pos + 36 + cnt]
        rays[int(d)].append(((int(p), int(y), int(x)), ev, od))
        pos += 36 + cnt
    out, geo, keys = {}, {}, {}
    for d, lst in rays.items():
        lst.sort(key=lambda t: t[0])
        out[d] = [e for _, e, _ in lst]
        geo[d] = np.array([g for _, _, g in lst], dtype=np.float32).reshape(-1, 6)
        keys[d] = [k for k, _, _ in lst]                          # (pass, y, x) of each ray's path
    return (out, geo, keys) if with_keys else (out, geo)


class Ray:
    """Cursor over one ray's event list, exposing what the kernel's Traversal<> asks for next."""
    __slots__ = ("ev", "i", "n")

    def __init__(self, ev):
        self.ev, self.i, self.n = ev, 0, len(ev)

    def done(self):
        return self.i >= self.n

    def wants_inst(self):
        return self.i < self.n and self.ev[self.i] in (1, 2)

    def wants_node(self):
        return self.i < self.n and self.ev[self.i] not in (1, 2)

    def take(self):
        e = int(self.ev[self.i])
        self.i += 1
        return e


class Meter:
    def __init__(self):
        self.inst = 0.0
        self.lane_inst = 0.0

    def add(self, weight, active, rounds=1):
        self.inst += weight * rounds
        self.lane_inst += weight * active * rounds

    def active(self):
        return self.lane_inst / self.inst if self.inst else 0.0


def tri_rounds(meter, tris, cooperative=False):
    """Triangle loop of one node round: lane l tests tris[l] triangles.  Default: each lane loops over its own (the warp runs
    max(tris) iterations, iteration k executed by the lanes with more than k triangles).  cooperative: the (lane, triangle)
    pairs are dealt out over all 32 lanes with shuffles (+8 instructions per dealt round)."""
    if not tris:
        return
    if cooperative:
        total = sum(tris)
        full, rest = divmod(total, 32)
        meter.add(W_TRI + 8, 32, full)
        if rest:
            meter.add(W_TRI + 8, rest)
        return
    for k in range(max(tris)):
        meter.add(W_TRI, sum(1 for t in tris if t > k))


def simulate(rays, policy="phase", burst=3, refill=16, persistent=True, cooperative=False, tburst=2):
    """Replay one K2 launch over `rays` (list of event arrays in dispatch order).  Returns (active lanes per instruction,
    instructions per ray)."""
    m = Meter()
    queue = [Ray(e) for e in rays if len(e)]
    nrays = len(queue)
    qpos = 0
    # one persistent warp stands for all of them: the kernel's warps pull from ONE global counter in arrival order, and the
    # figure of merit is a ratio, so the interleaving of warps does not matter to first order.  (Non-persistent: a warp takes
    # 32 consecutive rays and retires when all are done.)
    pending = {}
    while qpos < nrays:
        lanes = [None] * 32
        while True:
            busy = sum(1 for r in lanes if r is not None)
            if (persistent or busy == 0) and busy < (refill if persistent else 1) and qpos < nrays:
                got = 0
                for i in range(32):
                    if lanes[i] is None and qpos < nrays:
                        lanes[i] = queue[qpos]
                        qpos += 1
                        got += 1
                m.add(W_REFILL, got)
            live = [r for r in lanes if r is not None]
            if not live:
                break
            m.add(W_LOOP, 32)
            if policy == "flat":
                # one step per lane per iteration: the node path and the instance path are two divergent branches
                nodes = [r for r in live if r.wants_node()]
                insts = [r for r in live if r.wants_inst()]
                if nodes:
                    codes = [r.take() for r in nodes]
                    m.add(W_NODE, len(nodes))
                    tri_rounds(m, [c - 64 for c in codes if c >= 64 and c > 64], cooperative)
                if insts:
                    for r in insts:
                        r.take()
                    m.add(W_INST, len(insts))
            elif policy == "trimode":
                # decoupled state machine: a lane that reaches a leaf switches to TRIANGLE mode and tests at most `tburst`
                # triangles per outer iteration (phase T, all triangle-mode lanes together) while the other lanes keep taking
                # node steps in phase N; it resumes traversal only when its leaf is finished (order and culling unchanged)
                for _ in range(burst):
                    nodes = [r for r in live if pending.get(id(r), 0) == 0 and r.wants_node()]
                    if not nodes:
                        break
                    m.add(W_NODE, len(nodes))
                    for r in nodes:
                        c = r.take()
                        if c > 64:
                            pending[id(r)] = c - 64
                for _ in range(tburst):
                    act = [k for k, v in pending.items() if v > 0]
                    if not act:
                        break
                    m.add(W_TRI + 6, len(act))
                    for k in act:
                        pending[k] -= 1
                insts = [r for r in live if pending.get(id(r), 0) == 0 and r.wants_inst()]
                if insts:
                    for r in insts:
                        r.take()
                    m.add(W_INST, len(insts))
            elif policy == "leafwait":
                # node rounds in which a lane that reaches a leaf WAITS (its triangles untested) until no lane can advance or
                # `burst` rounds passed; then ONE triangle phase for all waiting lanes; then the instance steps.  Visiting order
                # and the distance used for culling are unchanged for every ray: only the warp's interleaving differs.
                waiting = {}
                for _ in range(burst):
                    nodes = [r for r in live if id(r) not in waiting and r.wants_node()]
                    if not nodes:
                        break
                    m.add(W_NODE, len(nodes))
                    for r in nodes:
                        c = r.take()
                        if c > 64:
                            waiting[id(r)] = c - 64
                tri_rounds(m, list(waiting.values()), cooperative)
                insts = [r for r in live if r.wants_inst()]
                if insts:
                    for r in insts:
                        r.take()
                    m.add(W_INST, len(insts))
            else:
                # phase-separated: up to `burst` node rounds, then the pending instance steps together
                for _ in range(burst):
                    nodes = [r for r in live if r.wants_node()]
                    if not nodes:
                        break
                    codes = [r.take() for r in nodes]
                    m.add(W_NODE, len(nodes))
                    tri_rounds(m, [c - 64 for c in codes if c > 64], cooperative)
                insts = [r for r in live if r.wants_inst()]
                if insts:
                    for r in insts:
                        r.take()
                    m.add(W_INST, len(insts))
            fin = [i for i, r in enumerate(lanes) if r is not None and r.done() and pending.get(id(r), 0) == 0]
            if fin:
                m.add(W_WRITEBACK, len(fin))
                for i in fin:
                    lanes[i] = None
            if not persistent and all(r is None for r in lanes):
                break
    return m.active(), m.inst / max(1, nrays)


def first_cell_key(ev):
    """A cheap coherence key available before traversal would be octant + origin cell; offline we use what it approximates:
    the first instance the ray reaches and the length class of its walk (an upper bound on what sorting can achieve)."""
    first = next((i for i, e in enumerate(ev) if e in (1, 2)), 255)
    return (min(first, 255), int(np.log2(len(ev) + 1)))


ORDER_NAMES = {0: "pass-major, row strips (32x1 per warp)", 1: "pass-major, 8x4 Morton blocks", 2: "8 passes x 2x2 block",
               3: "4 passes x 4x2 block", 4: "2 passes x 4x4 block", 5: "8 passes x 4x1 strip"}


def path_ids(keys, x0, y0, w, h, passes, order):
    """path id of every (pass, y, x) of the region rendered as one batch (pixel set = the w x h rectangle) in path order `order`,
    from the library's own map (crgpu_path_order_map)"""
    import crgpu
    npix = w * h
    xy = np.zeros(npix, dtype=np.uint32)
    inv = np.zeros(npix * passes, dtype=np.uint32)
    assert crgpu.lib().crgpu_path_order_map(order, npix, passes, None, None, inv.ctypes.data, w, h, xy.ctypes.data) == 0
    local = np.empty(npix, dtype=np.int64)                        # (y - y0) * w + (x - x0) -> pixel index in the order
    local[(xy >> 16).astype(np.int64) * w + (xy & 0xffff).astype(np.int64)] = np.arange(npix)
    k = np.asarray(keys, dtype=np.int64).reshape(-1, 3)
    return inv[k[:, 0] * npix + local[(k[:, 1] - y0) * w + (k[:, 2] - x0)]]


def screen_orders(a):
    scene = a[0] if a else "hdr"
    W, H, x0, y0, x1, y1, passes = (int(v) for v in a[1:8]) if len(a) >= 8 else (1920, 1080, 896, 512, 960, 576, 8)
    traces, geo, keys = load_traces(scene, W, H, x0, y0, x1, y1, passes, with_keys=True)
    print(f"scene {scene} {W}x{H}, region x {x0}..{x1} y {y0}..{y1} as one batch of {passes} passes; rays per bounce:",
          {d: len(v) for d, v in sorted(traces.items()) if d < 4})
    print("K2 as built (phase-separated, burst 3, refill<16); bounce 1 keeps bounce 0's order for its survivors (K3's compaction),"
          " without K4's material buckets")
    for d in (0, 1):
        for o, name in ORDER_NAMES.items():
            ids = path_ids(keys[d], x0, y0, x1 - x0, y1 - y0, passes, o)
            rays = [traces[d][i] for i in np.argsort(ids, kind="stable")]
            act, ipr = simulate(rays, policy="phase", burst=3, refill=16)
            print(f"  bounce {d}  order {o}  {name:42s} active lanes {act:5.1f}   instructions/ray {ipr:7.0f}", flush=True)


def main():
    a = sys.argv[1:]
    if a and a[0] == "--orders":
        screen_orders(a[1:])
        return
    scene = a[0] if a else "hdr"
    W, H, x0, y0, x1, y1, passes = (int(v) for v in a[1:8]) if len(a) >= 8 else (1920, 1080, 704, 500, 1216, 564, 2)
    traces, geo = load_traces(scene, W, H, x0, y0, x1, y1, passes)
    print(f"scene {scene} {W}x{H}, region x {x0}..{x1} y {y0}..{y1}, {passes} passes; rays per bounce:",
          {d: len(v) for d, v in sorted(traces.items()) if d < 6})
    for d in (0, 1, 2):
        if d not in traces:
            continue
        rays = traces[d]
        ev = np.concatenate(rays) if rays else np.zeros(0, np.uint8)
        print(f"\nbounce {d}: {len(rays)} rays, per ray {np.mean([len(r) for r in rays]):.1f} steps "
              f"({(ev == 0).sum() / len(rays):.2f} top pairs, {(ev >= 64).sum() / len(rays):.2f} bottom pairs, "
              f"{np.maximum(ev[ev >= 64].astype(int) - 64, 0).sum() / len(rays):.2f} tris, {((ev == 1) | (ev == 2)).sum() / len(rays):.2f} instances)")
        rows = [
            ("flat loop, 32 rays per warp (r1: 9.6 measured)", dict(policy="flat", persistent=False)),
            ("flat + persistent refill<16 (r1: 11.6)", dict(policy="flat", persistent=True, refill=16)),
            ("phase-separated, burst 3, refill<16 (current; r1: 15.0)", dict(policy="phase", burst=3, refill=16)),
            ("  burst 1", dict(policy="phase", burst=1, refill=16)),
            ("  burst 6", dict(policy="phase", burst=6, refill=16)),
            ("  refill<24", dict(policy="phase", burst=3, refill=24)),
            ("  refill<31 (refill whenever a lane is free)", dict(policy="phase", burst=3, refill=31)),
            ("  + cooperative triangle tests", dict(policy="phase", burst=3, refill=16, cooperative=True)),
            ("leaves wait for a common triangle phase, burst 4", dict(policy="leafwait", burst=4, refill=16)),
            ("leaves wait, burst 8", dict(policy="leafwait", burst=8, refill=16)),
            ("leaves wait, burst 8, refill<24", dict(policy="leafwait", burst=8, refill=24)),
            ("leaves wait, burst 8 + cooperative triangles", dict(policy="leafwait", burst=8, refill=16, cooperative=True)),
            ("  refill<31 + cooperative triangles", dict(policy="phase", burst=3, refill=31, cooperative=True)),
            ("triangle MODE (decoupled), burst 3, 1 tri per iteration", dict(policy="trimode", burst=3, refill=16, tburst=1)),
            ("triangle MODE, burst 3, 2 tris per iteration", dict(policy="trimode", burst=3, refill=16, tburst=2)),
            ("triangle MODE, burst 3, 4 tris per iteration", dict(policy="trimode", burst=3, refill=16, tburst=4)),
            ("triangle MODE, burst 2, 2 tris, refill<24", dict(policy="trimode", burst=2, refill=24, tburst=2)),
        ]
        for name, kw in rows:
            act, ipr = simulate(rays, **kw)
            print(f"  {name:62s} active lanes {act:5.1f}   instructions/ray {ipr:7.0f}")
        srt = sorted(rays, key=first_cell_key)
        act, ipr = simulate(srt, policy="phase", burst=3, refill=16)
        print(f"  {'current policy, rays sorted by an oracle key (upper bound)':62s} active lanes {act:5.1f}   instructions/ray {ipr:7.0f}")
        # keys a kernel can compute before tracing: direction octant, then a Morton code of the origin in the batch's bounds
        g = geo[d]
        octant = (g[:, 3] < 0).astype(np.int64) | ((g[:, 4] < 0).astype(np.int64) << 1) | ((g[:, 5] < 0).astype(np.int64) << 2)
        lo, hi = g[:, :3].min(axis=0), g[:, :3].max(axis=0)
        order = np.argsort(octant, kind="stable")
        act, ipr = simulate([rays[i] for i in order], policy="phase", burst=3, refill=16)
        print(f"  {'current policy, rays binned by direction octant only (8 bins)':62s} active lanes {act:5.1f}   instructions/ray {ipr:7.0f}")
        dom = np.argmax(np.abs(g[:, 3:6]), axis=1).astype(np.int64)
        order = np.argsort(octant * 3 + dom, kind="stable")
        act, ipr = simulate([rays[i] for i in order], policy="phase", burst=3, refill=16)
        print(f"  {'current policy, rays binned by octant x dominant axis (24 bins)':62s} active lanes {act:5.1f}   instructions/ray {ipr:7.0f}")
        for bits in (2, 4):
            q = np.clip(((g[:, :3] - lo) / np.maximum(hi - lo, 1e-20) * (1 << bits)).astype(np.int64), 0, (1 << bits) - 1)
            morton = np.zeros(len(g), dtype=np.int64)
            for b in range(bits):
                for ax in range(3):
                    morton |= ((q[:, ax] >> b) & 1) << (3 * b + ax)
            for label, key in ((f"octant + {bits}-bit/axis origin cell", (octant << (3 * bits)) | morton), (f"{bits}-bit/axis origin cell only", morton)):
                order = np.argsort(key, kind="stable")
                act, ipr = simulate([rays[i] for i in order], policy="phase", burst=3, refill=16)
                print(f"  {'current policy, rays binned by ' + label:62s} active lanes {act:5.1f}   instructions/ray {ipr:7.0f}")
                act, ipr = simulate([rays[i] for i in order], policy="phase", burst=3, refill=16, cooperative=True)
                print(f"  {'   + cooperative triangle tests':62s} active lanes {act:5.1f}   instructions/ray {ipr:7.0f}")


if __name__ == "__main__":
    main()
