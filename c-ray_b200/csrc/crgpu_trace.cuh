/*
 * crgpu_trace.cuh — camera ray generation and two-level BVH closest-hit query (device functions).
 *
 * Restates, over the device layout of crgpu_scene.cuh:
 *   getCameraRay            reference src/datatypes/camera.c:50-87
 *   traverseBvhGeneric      reference src/accelerators/bvh.c:354-441 (+ intersectNode :326-352)
 *   intersectTopLevelLeaf   bvh.c:468-486      intersectBottomLevelLeaf  bvh.c:443-462
 *   intersectSphere/Mesh    src/datatypes/instance.c:45-60, 169-185 (closest-hit part)
 *   rayIntersectsWithPolygon src/datatypes/poly.c:17-53      intersect  src/datatypes/sphere.c:20-50
 *
 * The traversal visits nodes and primitives in EXACTLY the reference order (nearer child first,
 * farther pushed; both children tested with the maxDist valid before either leaf is processed), so
 * the closest hit — including exact-tie winners — is the reference's.
 */
#pragma once
#include "crgpu_math.cuh"
#include "crgpu_scene.cuh"

struct Hit {
	float t, u, v;
	int   inst;          /* -1 = miss */
	uint32_t prim;       /* global prim slot of the winning triangle */
};

struct TraceCounters { unsigned pairs, tris, spheres, insts; };

/* ---- camera.c:50-87 ---------------------------------------------------------------------------------------- */
CRD float cr_triangle_distribution(float v) {
	const float orig = v * 2.0f - 1.0f;
	v = cr_div(orig, cr_sqrtf(fabsf(orig)));
	v = cr_clamp(v, -1.0f, 1.0f);
	v = v - ((orig >= 0.0f) ? 1.0f : -1.0f);
	return v;
}

CRD void cr_camera_ray(const DevCamera &cam, int x, int y, uint64_t &rng, v3 &o, v3 &d) {
	const v3 right = v3make(cam.right[0], cam.right[1], cam.right[2]);
	const v3 up = v3make(cam.up[0], cam.up[1], cam.up[2]);
	const v3 forward = v3make(cam.forward[0], cam.forward[1], cam.forward[2]);
	const float jitterX = cr_triangle_distribution(cr_draw(rng));
	const float jitterY = cr_triangle_distribution(cr_draw(rng));
	const v3 pixX = v3scale(right, cr_div(cam.sensor_x, (float)cam.width));
	const v3 pixY = v3scale(up, cr_div(cam.sensor_y, (float)cam.height));
	const v3 pixV = v3add(forward, v3add(v3scale(pixX, (float)x - (float)cam.width * 0.5f + jitterX + 0.5f),
										 v3scale(pixY, (float)y - (float)cam.height * 0.5f + jitterY + 0.5f)));
	o = v3make(0.0f, 0.0f, 0.0f);
	d = v3norm(pixV);
	if (cam.aperture > 0.0f) {
		const float ft = cr_div(cam.focal_distance, v3dot(d, forward));
		const v3 focus = v3add(o, v3scale(d, ft));
		const float rr = cr_sqrtf(cr_draw(rng));                               /* vector.h:194-198 */
		const float theta = (cr_draw(rng) * (2.0f * CR_PI - 0.0f)) + 0.0f;
		float sn, cs;
		cr_sincosf(theta, &sn, &cs);
		const float lx = (rr * cs) * cam.aperture, ly = (rr * sn) * cam.aperture;
		o = v3add(o, v3add(v3scale(right, lx), v3scale(up, ly)));
		d = v3norm(v3sub(focus, o));
	}
	o = xf_point(cam.A, o);
	d = xf_vector(cam.A, d);
}

/* ---- bvh.c:326-352 -------------------------------------------------------------------------------------------- */
/* bits of RaySetup::bits (and of the low byte of Traversal::flags, which holds the current level's copy) */
#define CRG_RS_OX   1u      /* d.x has its sign bit set (bvh.c:369-371) */
#define CRG_RS_OY   2u
#define CRG_RS_OZ   4u
#define CRG_RS_DEG  3       /* bits 3..5: bit 3+a set when -o[a]/d[a] is not finite (1/d[a] is +-inf, or o[a]*(1/d[a]) overflows) — see cr_node_test */
#define CRG_RS_MASK 0x3fu

struct RaySetup {
	v3 invDir, scaledStart;
	unsigned bits;     /* CRG_RS_* */
};

CRD RaySetup cr_ray_setup(v3 o, v3 d) {                                                /* bvh.c:369-376 */
	RaySetup s;
	s.invDir = v3make(cr_div(1.0f, d.x), cr_div(1.0f, d.y), cr_div(1.0f, d.z));
	s.scaledStart = v3scale(v3mul(o, s.invDir), -1.0f);
	s.bits = (__float_as_uint(d.x) >> 31) | ((__float_as_uint(d.y) >> 31) << 1) | ((__float_as_uint(d.z) >> 31) << 2) |
			 ((isfinite(s.scaledStart.x) ? 0u : 1u) << CRG_RS_DEG) | ((isfinite(s.scaledStart.y) ? 0u : 2u) << CRG_RS_DEG) |
			 ((isfinite(s.scaledStart.z) ? 0u : 4u) << CRG_RS_DEG);
	return s;
}

/* bvh.c:318-324: `fastMultiplyAdd` is fmaf() when the compiler defines FP_FAST_FMAF (the reference's stock
 * -march=native build) and a*b+c otherwise (the strict oracle build).  The slab test only decides which nodes
 * are ENTERED, never a hit distance; the survey measured bit-identical framebuffers between them on hdr.json and
 * venus.json.  The two differ (a) by one rounding where a ray grazes a box face, which can decide whether a box of zero
 * thickness (a planar, axis-aligned leaf) is entered, and (b) where o*(1/d) overflows: the un-fused b*(1/d) + -inf is
 * NaN once b*(1/d) overflows too, and the reference's min/max chain drops that axis, while the fused result is -inf
 * and would reject every box.  Case (b) is culled exactly (below).  tests/test_gpu_trace.py holds K2 to the oracle in
 * these semantics.  Fused = 6 FFMA per child instead of 6 FMUL + 6 FADD.  Build with -DCRG_SLAB_UNFUSED to get the
 * two-rounding form. */
#ifdef CRG_SLAB_UNFUSED
#define CR_SLAB_MAD(a, b, c) ((a) * (b) + (c))
#else
#define CR_SLAB_MAD(a, b, c) __fmaf_rn((a), (b), (c))
#endif

/* Slab test of one child.  For ordinary rays this is intersectNode verbatim (bvh.c:326-352).
 *
 * Degenerate axes.  When a direction component is exactly 0 the reference computes b*inf + (-o*inf),
 * which is NaN for most bounds; its NaN-tolerant min/max chain then silently DROPS that axis (and, by
 * propagation, the x or y axis before it), so such a ray "enters" a large part of the BVH — up to
 * ~115,000 of Venus' 229,087 nodes per ray (measured with the oracle on hdr.json, horizon rays with
 * d.y == 0).  That is harmless on a CPU (~1 ms) but one GPU thread would need ~50-150 ms while the
 * whole wavefront waits.  The same happens on an axis whose 1/d is finite but so large that o*(1/d)
 * overflows (|d| below ~|o| / 3.4e38, e.g. d = FLT_MIN): there the fused form would even give -inf for
 * both planes and reject every box, missing hits the reference finds.  So every axis whose -o*(1/d) is
 * not finite is culled with the exact test (inside the slab iff lo <= o <= hi; along such an axis the
 * ray moves by less than |o| even at t = FLT_MAX).  The reference's degenerate test is
 * a superset of the exact one and the Möller–Trumbore test decides every hit on its own, so the closest
 * hit is the same; they could only differ for a ray that grazes a triangle within one ulp of its leaf's
 * bounding box.  All other rays take the verbatim path. */
CRD bool cr_node_test(const float *b, v3 invDir, v3 scaledStart, unsigned bits, v3 o, float maxDist, float &tEntry) {
	const bool ox = (bits & CRG_RS_OX) != 0u, oy = (bits & CRG_RS_OY) != 0u, oz = (bits & CRG_RS_OZ) != 0u;
	float tMinX = CR_SLAB_MAD((ox ? b[1] : b[0]), invDir.x, scaledStart.x);
	float tMaxX = CR_SLAB_MAD((ox ? b[0] : b[1]), invDir.x, scaledStart.x);
	float tMinY = CR_SLAB_MAD((oy ? b[3] : b[2]), invDir.y, scaledStart.y);
	float tMaxY = CR_SLAB_MAD((oy ? b[2] : b[3]), invDir.y, scaledStart.y);
	float tMinZ = CR_SLAB_MAD((oz ? b[5] : b[4]), invDir.z, scaledStart.z);
	float tMaxZ = CR_SLAB_MAD((oz ? b[4] : b[5]), invDir.z, scaledStart.z);
	const unsigned deg = (bits >> CRG_RS_DEG) & 7u;
	if (deg) {
		const float inf = __int_as_float(0x7f800000);
		if (deg & 1u) { const bool in = (b[0] <= o.x) && (o.x <= b[1]); tMinX = in ? -inf : inf; tMaxX = in ? inf : -inf; }
		if (deg & 2u) { const bool in = (b[2] <= o.y) && (o.y <= b[3]); tMinY = in ? -inf : inf; tMaxY = in ? inf : -inf; }
		if (deg & 4u) { const bool in = (b[4] <= o.z) && (o.z <= b[5]); tMinZ = in ? -inf : inf; tMaxZ = in ? inf : -inf; }
	}
	/* bvh.c:341-348 is a chain of `a > b ? a : b` (FSETP + FSEL each); fmaxf / fminf (one FMNMX) give the same value here.  No
	 * operand is NaN: an axis whose -o/d is not finite was replaced by +-inf above, and on every other axis 1/d and -o/d are
	 * finite, so b * (1/d) + (-o/d) is finite or +-inf for finite bounds.  The two forms can differ only in the sign of a zero
	 * (-0 against +0), and a zero's sign decides nothing below: tMin <= tMax and the caller's tL > tR compare -0 and +0 equal. */
	float tMin = fmaxf(tMinX, tMinY);
	float tMax = fminf(tMaxX, tMaxY);
	tMin = fmaxf(tMin, tMinZ);
	tMax = fminf(tMax, tMaxZ);
	tMin = fmaxf(tMin, 0.0f);
	tMax = fminf(tMax, maxDist);
	tEntry = tMin;
	return tMin <= tMax;
}

/* rayIntersectsWithPolygon over two leaves back to back (bvh.c:443-462 + poly.c:17-53): slots [firstA, firstA+nA) then
 * [firstB, firstB+nB), local to the BVH whose first slot is slot_base.  Only the distance of the closest hit is a register;
 * its u, v and slot are written to the caller's cold state (shared memory) when a triangle wins. */
template <bool COUNT>
CRD bool cr_leaf_tris(const DevScene &sc, uint32_t slot_base, uint32_t firstA, uint32_t nA, uint32_t firstB, uint32_t nB,
					  v3 o, v3 d, float &bestT, float &bestU, float &bestV, uint32_t &bestPrim, TraceCounters *ctr) {
	bool found = false;
	const PackedTri *__restrict__ tris = sc.tris + slot_base;
	const uint32_t total = nA + nB;
	for (uint32_t k = 0; k < total; ++k) {
		const uint32_t slot = k < nA ? firstA + k : firstB + (k - nA);
		const float4 *t4 = reinterpret_cast<const float4 *>(tris + slot);
		const float4 a = __ldg(t4 + 0), b = __ldg(t4 + 1), c4 = __ldg(t4 + 2);
		if (COUNT) ctr->tris++;
		const v3 v0 = v3make(a.x, a.y, a.z), e1 = v3make(a.w, b.x, b.y), e2 = v3make(b.z, b.w, c4.x);
		const v3 n = v3make(c4.y, c4.z, c4.w);
		const v3 c = v3sub(v0, o);
		const v3 r = v3cross(d, c);
		const float invDet = cr_div(1.0f, v3dot(n, d));
		const float u = v3dot(r, e2) * invDet;
		const float v = v3dot(r, e1) * invDet;
		if (u >= 0.0f && v >= 0.0f && u + v <= 1.0f) {
			const float t = v3dot(n, c) * invDet;
			if (t >= 0.0f && t < bestT) {
				bestT = t; bestU = u; bestV = v;
				bestPrim = slot_base + slot;
				found = true;
			}
		}
	}
	return found;
}

CRD bool cr_sphere_test(v3 o, v3 d, float radius, float &dist) {                   /* sphere.c:20-50 */
	const float A = v3dot(d, d);
	const float B = 2.0f * v3dot(d, o);
	const float C = v3dot(o, o) - (radius * radius);
	const float disc = B * B - 4.0f * A * C;
	if (disc < 0.0f) return false;
	const float sq = cr_sqrtf(disc);
	float t0 = cr_div(-B + sq, 2.0f);
	const float t1 = cr_div(-B - sq, 2.0f);
	if (t0 > t1 && t1 > 0.0f) t0 = t1;
	if (t0 < 0.00001f || t0 > dist) return false;
	dist = t0;
	return true;
}

/* object-space ray of an instance: transformRay(Ainv) + rayOffset advance (instance.c:47-50, 170-174) */
CRD void cr_object_ray(const float *Ainv, float ray_offset, v3 o, v3 d, v3 &oo, v3 &od) {
	oo = xf_point(Ainv, o);
	od = xf_vector(Ainv, d);
	oo = v3add(oo, v3scale(od, ray_offset));
}

#define CRG_END 0xffffffffu

/* getClosestIsect (pathtrace.c:26-30) = traverseTopLevelBvh → intersectTopLevelLeaf → intersectMesh →
 * traverseBottomLevelBvh, flattened into ONE loop so that the 32 lanes of a warp stay convergent:
 * every iteration a lane performs either one child-pair step (top OR bottom level — same code, only
 * the base pointer and the ray registers differ) or one instance step (transform the ray into the
 * next instance of a pending top-level leaf; spheres are tested on the spot, meshes switch the lane
 * to the bottom level).  The reference's recursion (a whole bottom-level traversal nested inside a
 * top-level leaf loop) serialised divergent lanes: ncu measured 3-6 active threads per warp.
 *
 * Order of evaluation is the reference's: both children are tested against the closest distance known
 * BEFORE either leaf is processed; left leaf, then right leaf; nearer internal child next, farther one
 * pushed; instances of a leaf in primIndices order; strict t < distance for triangles, t <= distance
 * for spheres.  The reference's `maxDist` copies always equal isect->distance at the time of a node
 * test (they are refreshed after every leaf that found something), so best.t is used directly. */
/* Where the traversal state lives.  K2 is bound by latency and pays for every resident warp (DESIGN §4), so a lane keeps only
 * what the hot loop touches in registers: best.t, the current level's ray and slab setup, node, sp/spBase, the pending-leaf cursors
 * and one flags word.  The rest is per-thread shared memory, laid out [field][thread] so that a warp's 32 accesses to one field
 * fall into 32 different banks:
 *   - the top CRG_SSTACK entries of the traversal stack (deeper entries spill to a thread-local array that is touched only
 *     when a lane's stack is that deep);
 *   - cold state: the world ray (read by an instance step and on the way back from a mesh), u, v, prim slot and instance of the
 *     closest hit (written on a hit, read at write-back), the top-level node to resume after a mesh and the mesh's instance;
 *   - the range of the current BVH's nodes that the block staged (CRGPU_TRACE_STAGE), read by a node step only when the block
 *     staged any: as two registers it cost the unstaged default 1.5% of the frame in spills (DESIGN §4).
 * Every kernel that runs a Traversal has at most CRG_TRAV_NT threads per block. */
#define CRG_SSTACK  8
#define CRG_OVF     (2 * CRG_MAX_STACK + 2)   /* capacity of the whole stack: CRG_MAX_STACK entries per level */
#define CRG_TRAV_NT 256

struct TravShared {
	uint32_t stack[CRG_SSTACK][CRG_TRAV_NT];
	float wo[3][CRG_TRAV_NT], wd[3][CRG_TRAV_NT];   /* world ray */
	float u[CRG_TRAV_NT], v[CRG_TRAV_NT];           /* closest hit so far */
	uint32_t prim[CRG_TRAV_NT];                     /* its global prim slot (a triangle) */
	int inst[CRG_TRAV_NT];                          /* its instance, -1 = miss */
	uint32_t topNext[CRG_TRAV_NT];                  /* top-level node to resume when the current mesh is exhausted */
	uint32_t stageBase[CRG_TRAV_NT], stageCount[CRG_TRAV_NT];   /* CRG_TF_STAGED: nodes [0, stageCount) of the current BVH are
	                                                   at crg_stage_smem[stageBase + node] */
	int curInst[CRG_TRAV_NT];                       /* the mesh instance being traversed */
};

/* the block's staged top-of-tree pair nodes (K2's dynamic shared memory, DevScene.stage_img); read only where Traversal::flags has CRG_TF_STAGED */
extern __shared__ __align__(128) unsigned char crg_stage_smem[];

/* bits of Traversal::flags above the current level's CRG_RS_* bits */
#define CRG_TF_BOTTOM  0x40u    /* in a mesh BVH */
#define CRG_TF_INSTHIT 0x80u    /* a triangle of the current mesh won */
#define CRG_TF_STAGED  0x100u   /* the block staged the top of every BVH in crg_stage_smem */
#define CRG_TF_SPHERE  0x200u   /* the closest hit's instance is a sphere (selects the shading-key table) */
#define CRG_TF_BUSY    0x400u   /* K2: the lane holds a ray */

template <bool COUNT>
struct Traversal {
	float bestT;
	v3 o, d;               /* ray of the current level */
	v3 invDir, scaledStart;/* its slab setup (RaySetup); the sign and degenerate-axis bits are in flags */
	uint32_t flags;        /* CRG_RS_* | CRG_TF_* */
	uint32_t pairOff;      /* first pair node of the current BVH in sc.pairs */
	uint32_t slotBase, node;
	uint32_t pendA, cntA, pendB, cntB;     /* pending top-level leaf items: A (left leaf) before B (right leaf) */
	uint32_t leafA, leafB, leafN;          /* DEFER: bottom-level leaf triangles not yet tested — slots [leafA, +nA) then [leafB, +nB), leafN = nA | nB << 16 */
	int sp, spBase;

	CRD static TravShared &sh() { __shared__ TravShared s; return s; }
	CRD static unsigned tid() { return threadIdx.x; }

	/* ovf: the caller's thread-local array of CRG_OVF entries, indexed by depth, for the entries at depth >= CRG_SSTACK.  It is
	 * a local of the calling kernel rather than a member: an array member with a runtime index would keep the whole struct
	 * in local memory. */
	CRD void push(uint32_t v, uint32_t *ovf) {
		if (sp < CRG_SSTACK) sh().stack[sp][tid()] = v;
		else ovf[sp] = v;
		++sp;
	}
	CRD uint32_t pop(const uint32_t *ovf) {
		--sp;
		return sp < CRG_SSTACK ? sh().stack[sp][tid()] : ovf[sp];
	}

	CRD bool bottom() const { return (flags & CRG_TF_BOTTOM) != 0u; }
	CRD bool done() const { return !bottom() && (cntA | cntB) == 0u && node == CRG_END && leafN == 0u; }

	CRD void set_ray(v3 ro, v3 rd) {
		o = ro; d = rd;
		const RaySetup rs = cr_ray_setup(o, d);
		invDir = rs.invDir; scaledStart = rs.scaledStart;
		flags = (flags & ~CRG_RS_MASK) | rs.bits;
	}
	CRD void set_stage(uint32_t base, uint32_t count) { sh().stageBase[tid()] = base; sh().stageCount[tid()] = count; }
	CRD void set_top(const DevScene &sc) {
		pairOff = sc.top.pair_offset;
		if (flags & CRG_TF_STAGED) set_stage(sc.top.stage_base, sc.top.stage_count);
	}

	/* staged: the block holds DevScene.stage_img in crg_stage_smem */
	CRD void begin(const DevScene &sc, v3 ro, v3 rd, bool staged) {
		TravShared &s = sh();
		const unsigned t = tid();
		bestT = CR_FLT_MAX; s.u[t] = 0.0f; s.v[t] = 0.0f; s.inst[t] = -1; s.prim[t] = 0u;
		s.wo[0][t] = ro.x; s.wo[1][t] = ro.y; s.wo[2][t] = ro.z;
		s.wd[0][t] = rd.x; s.wd[1][t] = rd.y; s.wd[2][t] = rd.z;
		flags = staged ? CRG_TF_STAGED : 0u;
		set_ray(ro, rd);
		set_top(sc);
		slotBase = 0u; node = 0u; s.topNext[t] = CRG_END;
		pendA = 0u; cntA = 0u; pendB = 0u; cntB = 0u;
		sp = 0; spBase = 0; s.curInst[t] = -1;
		leafA = 0u; leafB = 0u; leafN = 0u;
		if (sc.top.node_count < 1) {                                               /* bvh.c:362-365 */
			node = CRG_END;
		} else if (sc.top.node_count == 1) {                                       /* bvh.c:382-387 */
			float te;
			node = CRG_END;
			if (cr_node_test(sc.top.root_bounds, invDir, scaledStart, flags, o, bestT, te)) { pendA = sc.top.root_first; cntA = sc.top.root_count; }
		}
	}

	CRD bool wants_node() const { return leafN == 0u && (bottom() || ((cntA | cntB) == 0u && node != CRG_END)); }
	CRD bool wants_leaf() const { return leafN != 0u; }
	CRD bool wants_instance() const { return !bottom() && (cntA | cntB) != 0u; }

	/* the closest hit, once done() */
	CRD Hit result() const {
		const TravShared &s = sh();
		const unsigned t = tid();
		Hit h;
		h.t = bestT; h.u = s.u[t]; h.v = s.v[t]; h.inst = s.inst[t]; h.prim = s.prim[t];
		return h;
	}

	/* one iteration of the flat loop; precondition: !done() */
	CRD void step(const DevScene &sc, uint32_t *ovf, TraceCounters *ctr) {
		if (bottom() || (cntA | cntB) == 0u) node_step(sc, ovf, ctr);
		else instance_step(sc, ctr);
	}

	/* triangles of the current mesh: slots [firstA, +nA) then [firstB, +nB) */
	CRD void leaf_tris(const DevScene &sc, uint32_t firstA, uint32_t nA, uint32_t firstB, uint32_t nB, TraceCounters *ctr) {
		TravShared &s = sh();
		const unsigned t = tid();
		if (cr_leaf_tris<COUNT>(sc, slotBase, firstA, nA, firstB, nB, o, d, bestT, s.u[t], s.v[t], s.prim[t], ctr)) flags |= CRG_TF_INSTHIT;
	}

	/* the tail of a bottom-level step: once the mesh BVH is exhausted, back to the top level (instance.c:175-184) */
	CRD void finish_bottom(const DevScene &sc) {
		if (node == CRG_END) {
			TravShared &s = sh();
			const unsigned t = tid();
			if (flags & CRG_TF_INSTHIT) { s.inst[t] = s.curInst[t]; flags &= ~CRG_TF_SPHERE; }
			flags &= ~CRG_TF_BOTTOM;
			set_ray(v3make(s.wo[0][t], s.wo[1][t], s.wo[2][t]), v3make(s.wd[0][t], s.wd[1][t], s.wd[2][t]));
			set_top(sc);
			node = s.topNext[t];
			spBase = 0;
		}
	}

	/* DEFER: the triangles of the leaf/leaves the last node step reached (left leaf, then right leaf: bvh.c:402-418).  Until this has
	 * run the lane takes no further node step, so the visiting order and the distance every later box is culled with are exactly
	 * those of the in-line version; only the warp's interleaving differs: lanes that reached a leaf WAIT, and all waiting lanes of
	 * the warp test their triangles together after the node burst (K2 warp model, policy "leaves wait"). */
	CRD void leaf_step(const DevScene &sc, TraceCounters *ctr) {
		leaf_tris(sc, leafA, leafN & 0xffffu, leafB, leafN >> 16, ctr);
		leafN = 0u;
		finish_bottom(sc);
	}

	/* precondition: wants_node().  DEFER = true: leaf triangles are left pending for leaf_step() */
	template <bool DEFER = false>
	CRD void node_step(const DevScene &sc, uint32_t *ovf, TraceCounters *ctr) {
		{
			/* ---- one child-pair step (bvh.c:391-439) */
			float4 q0, q1, q2;
			uint4 q3;
			if ((flags & CRG_TF_STAGED) && node < sh().stageCount[tid()]) {      /* top of the tree: staged in shared memory by TMA */
				const float4 *p4 = reinterpret_cast<const float4 *>(reinterpret_cast<const PairNode *>(crg_stage_smem) + sh().stageBase[tid()] + node);
				q0 = p4[0]; q1 = p4[1]; q2 = p4[2];
				q3 = *reinterpret_cast<const uint4 *>(p4 + 3);
			} else {
				const float4 *p4 = reinterpret_cast<const float4 *>(sc.pairs + pairOff + node);
				q0 = __ldg(p4 + 0); q1 = __ldg(p4 + 1); q2 = __ldg(p4 + 2);
				q3 = __ldg(reinterpret_cast<const uint4 *>(p4 + 3));
			}
			const float lb[6] = { q0.x, q0.y, q0.z, q0.w, q1.x, q1.y };
			const float rb[6] = { q1.z, q1.w, q2.x, q2.y, q2.z, q2.w };
			if (COUNT) ctr->pairs++;
			float tL, tR;
			const bool hitL = cr_node_test(lb, invDir, scaledStart, flags, o, bestT, tL);
			const bool hitR = cr_node_test(rb, invDir, scaledStart, flags, o, bestT, tR);
			const bool leafL = (q3.z & CRG_LEAF_BIT) != 0u, leafR = (q3.w & CRG_LEAF_BIT) != 0u;
			const bool goL = hitL && !leafL, goR = hitR && !leafR;
			uint32_t next;
			if (goL & goR) {
				const bool swap = tL > tR;                                         /* bvh.c:424-431 */
				next = swap ? q3.y : q3.x;
				push(swap ? q3.x : q3.y, ovf);
			} else if (goL ^ goR) {
				next = goL ? q3.x : q3.y;
			} else {
				next = (sp == spBase) ? CRG_END : pop(ovf);
			}
			if (bottom()) {
				/* left leaf, then right leaf (bvh.c:402-418), as ONE loop so that lanes with a left leaf and lanes with a
				 * right leaf test their triangles together */
				const uint32_t nL = (hitL && leafL) ? (q3.z & ~CRG_LEAF_BIT) : 0u;
				const uint32_t nR = (hitR && leafR) ? (q3.w & ~CRG_LEAF_BIT) : 0u;
				node = next;
				if (DEFER && (nL + nR) != 0u && nL < 65536u && nR < 65536u) {
					leafA = q3.x; leafB = q3.y; leafN = nL | (nR << 16);               /* tested by leaf_step(), then finish_bottom() */
				} else {
					if (nL + nR) leaf_tris(sc, q3.x, nL, q3.y, nR, ctr);
					finish_bottom(sc);
				}
			} else {
				if (hitL && leafL) { pendA = q3.x; cntA = q3.z & ~CRG_LEAF_BIT; }
				if (hitR && leafR) { pendB = q3.y; cntB = q3.w & ~CRG_LEAF_BIT; }
				node = next;
			}
		}
	}

	/* into the BVH of mesh instance `inst` (pair_offset, slot_offset) with its object-space ray; nothing of it staged */
	CRD void enter_mesh(v3 oo, v3 od, uint32_t pair_offset, uint32_t slot_offset, int inst) {
		TravShared &s = sh();
		const unsigned t = tid();
		flags = (flags | CRG_TF_BOTTOM) & ~CRG_TF_INSTHIT;
		s.topNext[t] = node;
		set_ray(oo, od);
		pairOff = pair_offset;
		if (flags & CRG_TF_STAGED) set_stage(0u, 0u);
		slotBase = slot_offset;
		s.curInst[t] = inst;
		spBase = sp;
		node = 0u;
	}

	/* precondition: wants_instance() */
	CRD void instance_step(const DevScene &sc, TraceCounters *ctr) {
		{
			/* ---- one instance of a pending top-level leaf (bvh.c:468-486) */
			TravShared &s = sh();
			const unsigned t = tid();
			uint32_t idx;
			if (cntA) { idx = pendA++; --cntA; } else { idx = pendB++; --cntB; }
			const float4 *m4 = reinterpret_cast<const float4 *>(sc.top_items + sc.top.slot_offset + idx);    /* one DevTopItem */
			const float4 r0 = __ldg(m4 + 0), r1 = __ldg(m4 + 1), r2 = __ldg(m4 + 2);
			const float Ainv[12] = { r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w, r2.x, r2.y, r2.z, r2.w };
			const uint4 meta = __ldg(reinterpret_cast<const uint4 *>(m4 + 3));    /* inst | CRG_ITEM_*, ray_offset, shape, slot_offset */
			const int cur = (int)(meta.x & CRG_ITEM_INDEX);
			v3 oo, od;
			cr_object_ray(Ainv, __uint_as_float(meta.y), v3make(s.wo[0][t], s.wo[1][t], s.wo[2][t]), v3make(s.wd[0][t], s.wd[1][t], s.wd[2][t]), oo, od);
			if (meta.x & CRG_ITEM_MESH) {                                          /* instance.c:169-175 */
				if (COUNT) ctr->insts++;
				if (!(meta.x & CRG_ITEM_BVH)) {
					enter_mesh(oo, od, meta.z, meta.w, cur);                       /* the common mesh: nothing beyond the record */
				} else {
					const DevBvh *bvh = sc.bvhs + __ldg(&sc.instances[cur].bvh);
					const uint32_t nodeCount = __ldg(&bvh->node_count);
					if (nodeCount < 1u) {
						s.inst[t] = -1;                                            /* bvh.c:362-365 quirk */
					} else if (nodeCount == 1u) {                                  /* bvh.c:382-387 */
						const RaySetup ors = cr_ray_setup(oo, od);
						float rbnd[6], te;
						for (int k = 0; k < 6; ++k) rbnd[k] = __ldg(&bvh->root_bounds[k]);
						if (cr_node_test(rbnd, ors.invDir, ors.scaledStart, ors.bits, oo, bestT, te))
							if (cr_leaf_tris<COUNT>(sc, meta.w, __ldg(&bvh->root_first), __ldg(&bvh->root_count), 0u, 0u, oo, od, bestT, s.u[t], s.v[t], s.prim[t], ctr)) {
								s.inst[t] = cur;
								flags &= ~CRG_TF_SPHERE;
							}
					} else {                                                       /* a mesh with staged nodes */
						enter_mesh(oo, od, meta.z, meta.w, cur);
						if (flags & CRG_TF_STAGED) set_stage(__ldg(&bvh->stage_base), __ldg(&bvh->stage_count));
					}
				}
			} else {                                                               /* instance.c:45-51 */
				if (COUNT) ctr->spheres++;
				if (cr_sphere_test(oo, od, __uint_as_float(meta.z), bestT)) { s.inst[t] = cur; flags |= CRG_TF_SPHERE; }
			}
		}
	}
};

/* ---- cooperative leaf phase (K2, DEFER == 2) ------------------------------------------------------------------------------------
 * ncu: a quarter of K2's warp instructions are Möller–Trumbore tests executed with ~2 active lanes — at any step only
 * one or two lanes of a warp stand at a leaf, and the warp then runs the per-lane triangle loop max(leaf size) times for them.
 * Here the lanes that reached a leaf WAIT (Traversal::leafN, as in DEFER == 1) and, after the node burst, the warp deals all their
 * (ray, triangle) pairs out over its 32 lanes: one pass of the triangle code tests up to 32 pairs of up to 32 different rays.
 * The ray of a pair is read from its owner lane with shuffles; candidates go back through 3 x 32 floats of shared memory per warp and
 * every owner takes its winner IN LEAF ORDER with the reference's strict `t < distance` (poly.c:48, bvh.c:455-459: the first of equal
 * distances wins), so hit records stay bit-identical.  Must be called by all 32 lanes of the warp (convergent). */
struct CoopScratch { float t[32], u[32], v[32]; unsigned owner[32]; };

template <bool COUNT>
CRD void cr_coop_leaves(Traversal<COUNT> &tr, bool has, const DevScene &sc, CoopScratch &cs, unsigned lane, TraceCounters *ctr) {
	const unsigned FULL = 0xffffffffu;
	unsigned pending = __ballot_sync(FULL, has);
	while (pending) {
		const unsigned nA = tr.leafN & 0xffffu, nB = tr.leafN >> 16;
		unsigned cnt = has ? nA + nB : 0u;
		if (cnt > 32u) { tr.leaf_step(sc, ctr); has = false; cnt = 0u; }      /* an oversized leaf pair: the lane's own loop (rare) */
		unsigned incl = cnt;
#pragma unroll
		for (unsigned dlt = 1u; dlt < 32u; dlt <<= 1) { const unsigned x = __shfl_up_sync(FULL, incl, dlt); if (lane >= dlt) incl += x; }
		const bool fits = has && incl <= 32u;                 /* incl is non-decreasing over lanes: the lanes that fit form a prefix */
		const unsigned excl = incl - cnt;
		const unsigned startMask = __reduce_or_sync(FULL, fits ? (1u << (excl & 31u)) : 0u);
		const unsigned tot = __reduce_max_sync(FULL, fits ? incl : 0u);
		if (fits) cs.owner[excl & 31u] = lane;
		__syncwarp();
		/* pair `lane` of this round: owner = the lane whose segment [excl, incl) holds it */
		unsigned seg = 0u, ow = lane;
		if (lane < tot) { seg = 31u - (unsigned)__clz((int)(startMask & (0xffffffffu >> (31u - lane)))); ow = cs.owner[seg]; }
		const float ox = __shfl_sync(FULL, tr.o.x, ow), oy = __shfl_sync(FULL, tr.o.y, ow), oz = __shfl_sync(FULL, tr.o.z, ow);
		const float dx = __shfl_sync(FULL, tr.d.x, ow), dy = __shfl_sync(FULL, tr.d.y, ow), dz = __shfl_sync(FULL, tr.d.z, ow);
		const unsigned lA = __shfl_sync(FULL, tr.leafA, ow), lB = __shfl_sync(FULL, tr.leafB, ow), lN = __shfl_sync(FULL, tr.leafN, ow);
		const unsigned sb = __shfl_sync(FULL, tr.slotBase, ow);
		if (lane < tot) {
			const unsigned k = lane - seg, onA = lN & 0xffffu;
			const unsigned slot = k < onA ? lA + k : lB + (k - onA);
			const float4 *t4 = reinterpret_cast<const float4 *>(sc.tris + sb + slot);
			const float4 a = __ldg(t4 + 0), b = __ldg(t4 + 1), c4 = __ldg(t4 + 2);
			if (COUNT) ctr->tris++;
			const v3 o = v3make(ox, oy, oz), d = v3make(dx, dy, dz);
			const v3 v0 = v3make(a.x, a.y, a.z), e1 = v3make(a.w, b.x, b.y), e2 = v3make(b.z, b.w, c4.x);
			const v3 n = v3make(c4.y, c4.z, c4.w);
			const v3 c = v3sub(v0, o);
			const v3 r = v3cross(d, c);
			const float invDet = cr_div(1.0f, v3dot(n, d));
			const float u = v3dot(r, e2) * invDet;
			const float v = v3dot(r, e1) * invDet;
			float tt = __int_as_float(0x7f800000);              /* +inf: never `< distance` */
			if (u >= 0.0f && v >= 0.0f && u + v <= 1.0f) {
				const float t = v3dot(n, c) * invDet;
				if (t >= 0.0f) tt = t;
			}
			cs.t[lane] = tt; cs.u[lane] = u; cs.v[lane] = v;
		}
		__syncwarp();
		if (fits) {
			float bt = tr.bestT;
			int kb = -1;
			for (unsigned k = 0u; k < cnt; ++k) { const float x = cs.t[excl + k]; if (x < bt) { bt = x; kb = (int)k; } }
			if (kb >= 0) {
				const unsigned k = (unsigned)kb;
				TravShared &ts = tr.sh();
				const unsigned t = tr.tid();
				tr.bestT = bt; ts.u[t] = cs.u[excl + k]; ts.v[t] = cs.v[excl + k];
				ts.prim[t] = tr.slotBase + (k < nA ? tr.leafA + k : tr.leafB + (k - nA));
				tr.flags |= CRG_TF_INSTHIT;
			}
			tr.leafN = 0u;
			tr.finish_bottom(sc);
			has = false;
		}
		__syncwarp();
		pending = __ballot_sync(FULL, has);
	}
}

template <bool COUNT>
CRD Hit cr_closest_hit(const DevScene &sc, v3 wo, v3 wd, TraceCounters *ctr) {
	uint32_t ovf[CRG_OVF];
	Traversal<COUNT> tr;
	tr.begin(sc, wo, wd, false);
	while (!tr.done()) tr.step(sc, ovf, ctr);
	return tr.result();
}
