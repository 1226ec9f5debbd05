/*
 * crgpu_shade.cuh — hit reconstruction, node-graph evaluation and BSDF sampling (device functions).
 *
 * Restates:
 *   intersectSphere / intersectMesh (the post-hit half)   reference src/datatypes/instance.c:33-60,150-185
 *   poly.c:40-47 (barycentric normal), sphere.c:52-61
 *   textureGetPixel / Internal                             src/datatypes/image/texture.c:32-79
 *   color / value nodes                                    src/nodes/textures/{constant,image,checker,gradient,alpha}.c,
 *                                                          src/nodes/converter/{grayscale,blackbody}.c, src/nodes/valuenode.c
 *   bsdf nodes                                             src/nodes/shaders/{diffuse,metal,glass,plastic,mix,add,
 *                                                          transparent,emission,background,isotropic}.c
 *
 * The reference evaluates the graph through recursive function pointers.  Here the graph is a flat
 * table (crs_node) walked by a small interpreter: MIX and PLASTIC are tail calls (a loop), ADD uses an
 * explicit 4-entry operand stack, color<->value recursion is bounded at compile time (depth 3; deeper
 * graphs are rejected at upload with CRGPU_ERR_UNSUPPORTED).  Draw order is the reference's.
 */
#pragma once
#include "crgpu_math.cuh"
#include "crgpu_scene.cuh"
#include "crgpu_trace.cuh"


struct Rec {                  /* the fields of struct hitRecord (hitrecord.h:14-23) the nodes read */
	v3 inc_d;                 /* incident.direction */
	v3 p, n;                  /* hitPoint, surfaceNormal */
	v2 uv;
	float IOR;                /* material.IOR */
	float dist;               /* distance (input/raylength.c:39); FLT_MAX on a miss (pathtrace.c:27) */
};

struct BsdfSample { v3 out; col4 color; };

/* ---- texture.c:32-63 ------------------------------------------------------------------------------------------ */
/* x % extent for the size_t coordinates of textureGetPixelInternal (negative ints arrive sign-extended) */
CRD uint32_t cr_wrap(uint64_t x, uint32_t extent, uint32_t mask) {
	if (mask) return (uint32_t)x & mask;
	if ((x >> 32) == 0ull) return (uint32_t)x % extent;
	return (uint32_t)(x % extent);
}

CRD col4 cr_texel(const DevScene &sc, const DevTexture &t, uint64_t x64, uint64_t y64) {
	const uint32_t x = cr_wrap(x64, t.width, t.wmask);
	const uint32_t y = cr_wrap(y64, t.height, t.hmask);
	const size_t idx = ((size_t)x + (size_t)((t.height - 1u) - y) * t.width) * t.channels;
	const float *__restrict__ lut = sc.u8_to_unit;
	col4 o;
	if (t.channels == 1) {
		if (t.is_float) o.r = __ldg(reinterpret_cast<const float *>(t.data) + idx);
		else o.r = __ldg(lut + __ldg(t.data + idx));
		o.g = o.r; o.b = o.r; o.a = 1.0f;
	} else if (t.is_float) {
		const float *f = reinterpret_cast<const float *>(t.data);
		o.r = __ldg(f + idx); o.g = __ldg(f + idx + 1); o.b = __ldg(f + idx + 2);
		o.a = t.has_alpha ? __ldg(f + idx + 3) : 1.0f;
	} else if (t.channels == 4) {
		const uchar4 px = __ldg(reinterpret_cast<const uchar4 *>(t.data + idx));
		o.r = __ldg(lut + px.x); o.g = __ldg(lut + px.y); o.b = __ldg(lut + px.z);
		o.a = t.has_alpha ? __ldg(lut + px.w) : 1.0f;                 /* like every other branch: alpha only where the texture has one */
	} else {
		o.r = __ldg(lut + __ldg(t.data + idx));
		o.g = __ldg(lut + __ldg(t.data + idx + 1));
		o.b = __ldg(lut + __ldg(t.data + idx + 2));
		o.a = t.has_alpha ? __ldg(lut + __ldg(t.data + idx + 3)) : 1.0f;
	}
	return o;
}

/* alpha lane only (same arithmetic as cr_texel().a) */
CRD float cr_texel_alpha(const DevScene &sc, const DevTexture &t, uint64_t x64, uint64_t y64) {
	if (!t.has_alpha || t.channels != 4) return 1.0f;
	const uint32_t x = cr_wrap(x64, t.width, t.wmask);
	const uint32_t y = cr_wrap(y64, t.height, t.hmask);
	const size_t idx = ((size_t)x + (size_t)((t.height - 1u) - y) * t.width) * 4u;
	if (t.is_float) return __ldg(reinterpret_cast<const float *>(t.data) + idx + 3);
	return __ldg(sc.u8_to_unit + __ldg(t.data + idx + 3));
}

CRD col4 cr_texture_get(const DevScene &sc, const DevTexture &t, float x, float y, bool filtered) {             /* texture.c:66-79 */
	if (!filtered) return cr_texel(sc, t, cr_f2sz(x), cr_f2sz(y));
	x = x * (float)t.width;
	y = y * (float)t.height;
	const float xcopy = x - 0.5f;
	const float ycopy = y - 0.5f;
	const int xint = cr_f2i(xcopy);
	const int yint = cr_f2i(ycopy);
	const col4 tl = cr_texel(sc, t, (uint64_t)(int64_t)xint, (uint64_t)(int64_t)yint);
	const col4 tr = cr_texel(sc, t, (uint64_t)(int64_t)(xint + 1), (uint64_t)(int64_t)yint);
	const col4 bl = cr_texel(sc, t, (uint64_t)(int64_t)xint, (uint64_t)(int64_t)(yint + 1));
	const col4 br = cr_texel(sc, t, (uint64_t)(int64_t)(xint + 1), (uint64_t)(int64_t)(yint + 1));
	const float fx = xcopy - (float)xint, fy = ycopy - (float)yint;
	return c4mix(c4mix(tl, tr, fx), c4mix(bl, br, fx), fy);
}

CRD float cr_texture_get_alpha(const DevScene &sc, const DevTexture &t, float x, float y, bool filtered) {
	if (!filtered) return cr_texel_alpha(sc, t, cr_f2sz(x), cr_f2sz(y));
	x = x * (float)t.width;
	y = y * (float)t.height;
	const float xcopy = x - 0.5f;
	const float ycopy = y - 0.5f;
	const int xint = cr_f2i(xcopy);
	const int yint = cr_f2i(ycopy);
	const float tl = cr_texel_alpha(sc, t, (uint64_t)(int64_t)xint, (uint64_t)(int64_t)yint);
	const float tr = cr_texel_alpha(sc, t, (uint64_t)(int64_t)(xint + 1), (uint64_t)(int64_t)yint);
	const float bl = cr_texel_alpha(sc, t, (uint64_t)(int64_t)xint, (uint64_t)(int64_t)(yint + 1));
	const float br = cr_texel_alpha(sc, t, (uint64_t)(int64_t)(xint + 1), (uint64_t)(int64_t)(yint + 1));
	const float fx = xcopy - (float)xint, fy = ycopy - (float)yint;
	const float top = tl * (1.0f - fx) + tr * fx;
	const float bot = bl * (1.0f - fx) + br * fx;
	return top * (1.0f - fy) + bot * fy;
}

/* ---- color / value nodes ------------------------------------------------------------------------------------------
 * Two interpreters.  NodeEval<D> is the hot one: the node kinds a JSON scene can contain (every bundled scene), nesting budget
 * CRG_NODE_DEPTH.  A node kind it does not know falls through to NodeX<CRG_XNODE_DEPTH> (below): the complete interpreter — the
 * kinds only the reference's C constructors can build (SURVEY 8 f4: math, vecmath, fresnel, raylength, normal, vectocolor,
 * combine) plus the classic kinds again, because once inside a math chain every child may be of either sort — with its own
 * budget from the point where it takes over.  Keeping the two apart keeps the hot functions as small as they were (measured:
 * one merged interpreter with an 8-level budget made K3 slower on hdr.json). */
static __device__ __noinline__ col4 cr_xnode_color(const DevScene &sc, int node, const Rec &rec);
static __device__ __noinline__ float cr_xnode_value(const DevScene &sc, int node, const Rec &rec);
template <int D, bool X> struct NodeEval {
	static __device__ __noinline__ col4 color(const DevScene &sc, int node, const Rec &rec);
	static __device__ __noinline__ float value(const DevScene &sc, int node, const Rec &rec);
	static __device__ __noinline__ float alpha(const DevScene &sc, int node, const Rec &rec);
};

static __device__ __noinline__ col4 cr_image_color(const DevScene &sc, const crs_node &n, const Rec &rec) {            /* image.c:31-48 */
	if (n.tex < 0) return c4make(1.0f, 0.0f, 0.5f, 1.0f);
	const DevTexture t = sc.textures[n.tex];
	col4 out;
	if (n.options & CRS_IMG_NO_BILINEAR) {
		const float x = rec.uv.x * (float)t.width;
		const float y = rec.uv.y * (float)t.height;
		out = cr_texture_get(sc, t, x, y, false);
	} else {
		out = cr_texture_get(sc, t, rec.uv.x, rec.uv.y, true);
	}
	if (n.options & CRS_IMG_SRGB_TRANSFORM)
		out = c4make(cr_srgb_to_linear(out.r), cr_srgb_to_linear(out.g), cr_srgb_to_linear(out.b), out.a);
	return out;
}

static __device__ __noinline__ float cr_image_alpha(const DevScene &sc, const crs_node &n, const Rec &rec) {
	if (n.tex < 0) return 1.0f;
	const DevTexture t = sc.textures[n.tex];
	if (n.options & CRS_IMG_NO_BILINEAR)
		return cr_texture_get_alpha(sc, t, rec.uv.x * (float)t.width, rec.uv.y * (float)t.height, false);
	return cr_texture_get_alpha(sc, t, rec.uv.x, rec.uv.y, true);
}

CRD col4 cr_gradient(const crs_node &n, const Rec &rec) {                                   /* gradient.c:40-45 */
	const v3 unit = v3norm(rec.inc_d);
	const float t = 0.5f * (unit.y + 1.0f);
	return c4add(c4coef(1.0f - t, c4make(n.f[0], n.f[1], n.f[2], n.f[3])), c4coef(t, c4make(n.f[4], n.f[5], n.f[6], n.f[7])));
}

template <int D, bool X>
__device__ __noinline__ col4 NodeEval<D, X>::color(const DevScene &sc, int node, const Rec &rec) {
	while (true) {
		const crs_node &n = sc.nodes[node];
		switch (n.kind) {
		case CRS_COLOR_CONSTANT: return c4make(n.f[0], n.f[1], n.f[2], n.f[3]);             /* constant.c:39-42 */
		case CRS_COLOR_IMAGE: return cr_image_color(sc, n, rec);
		case CRS_COLOR_GRADIENT: return cr_gradient(n, rec);
		case CRS_COLOR_CHECKER: {                                                           /* checker.c:31-54 */
			const float coef = NodeEval<D - 1, X>::value(sc, n.in[2], rec);
			float sines;
			if (rec.uv.x >= 0) sines = cr_sinf(coef * rec.uv.x) * cr_sinf(coef * rec.uv.y);
			else sines = cr_sinf(coef * rec.p.x) * cr_sinf(coef * rec.p.y) * cr_sinf(coef * rec.p.z);
			node = sines < 0.0f ? n.in[0] : n.in[1];
			continue;                                                                       /* tail call */
		}
		case CRS_COLOR_BLACKBODY:                                                           /* blackbody.c:38-42 */
			return cr_color_for_kelvin(NodeEval<D - 1, X>::value(sc, n.in[0], rec));
		default: return X ? cr_xnode_color(sc, node, rec) : c4make(0.0f, 0.0f, 0.0f, 1.0f);
		}
	}
}
template <int D, bool X>
__device__ __noinline__ float NodeEval<D, X>::value(const DevScene &sc, int node, const Rec &rec) {
	const crs_node &n = sc.nodes[node];
	switch (n.kind) {
	case CRS_VALUE_CONSTANT: return n.f[0];
	case CRS_VALUE_GRAYSCALE: return cr_grayscale(NodeEval<D, X>::color(sc, n.in[0], rec));    /* grayscale.c:40-43 */
	case CRS_VALUE_ALPHA: return NodeEval<D, X>::alpha(sc, n.in[0], rec);                      /* alpha.c:38-41 */
	default: return X ? cr_xnode_value(sc, node, rec) : 0.0f;
	}
}
/* .alpha of a color node without evaluating the rgb lanes when the node kind allows it */
template <int D, bool X>
__device__ __noinline__ float NodeEval<D, X>::alpha(const DevScene &sc, int node, const Rec &rec) {
	const crs_node &n = sc.nodes[node];
	switch (n.kind) {
	case CRS_COLOR_CONSTANT: return n.f[3];
	case CRS_COLOR_IMAGE: return cr_image_alpha(sc, n, rec);
	case CRS_COLOR_BLACKBODY: return 0.0f;
	default: return NodeEval<D, X>::color(sc, node, rec).a;
	}
}
template <bool X> struct NodeEval<0, X> {   /* leaves only */
	static __device__ __noinline__ col4 color(const DevScene &sc, int node, const Rec &rec) {
		const crs_node &n = sc.nodes[node];
		switch (n.kind) {
		case CRS_COLOR_CONSTANT: return c4make(n.f[0], n.f[1], n.f[2], n.f[3]);
		case CRS_COLOR_IMAGE: return cr_image_color(sc, n, rec);
		case CRS_COLOR_GRADIENT: return cr_gradient(n, rec);
		default: return X ? cr_xnode_color(sc, node, rec) : c4make(0.0f, 0.0f, 0.0f, 1.0f);
		}
	}
	static __device__ __noinline__ float value(const DevScene &sc, int node, const Rec &rec) {
		const crs_node &n = sc.nodes[node];
		switch (n.kind) {
		case CRS_VALUE_CONSTANT: return n.f[0];
		case CRS_VALUE_GRAYSCALE: return cr_grayscale(color(sc, n.in[0], rec));
		case CRS_VALUE_ALPHA: return alpha(sc, n.in[0], rec);
		default: return X ? cr_xnode_value(sc, node, rec) : 0.0f;
		}
	}
	static __device__ __noinline__ float alpha(const DevScene &sc, int node, const Rec &rec) {
		const crs_node &n = sc.nodes[node];
		switch (n.kind) {
		case CRS_COLOR_CONSTANT: return n.f[3];
		case CRS_COLOR_IMAGE: return cr_image_alpha(sc, n, rec);
		default: return color(sc, node, rec).a;
		}
	}
};
template <bool X> using NodesT = NodeEval<CRG_NODE_DEPTH, X>;

/* ---- the complete interpreter (SURVEY 8 f4) ---------------------------------------------------------------------------------------
 * Every edge of the graph costs one level of the budget E (checked at upload: crgpu_api.cu xnode_depth). */
/* converter/math.c:44-97 (libm calls through the fp64 stand-ins of crgpu_math.cuh) */
static __device__ __noinline__ float cr_math_op(unsigned op, float a, float b) {
	switch (op) {
	case CRS_MATH_ADD: return a + b;
	case CRS_MATH_SUBTRACT: return a - b;
	case CRS_MATH_MULTIPLY: return a * b;
	case CRS_MATH_DIVIDE: return cr_div(a, b);
	case CRS_MATH_POWER: return cr_powf(a, b);
	case CRS_MATH_LOG: return cr_log10f(a);
	case CRS_MATH_SQRT: return cr_sqrtf(a);
	case CRS_MATH_ABS: return fabsf(a);
	case CRS_MATH_MIN: return CR_MIN(a, b);
	case CRS_MATH_MAX: return CR_MAX(a, b);
	case CRS_MATH_SINE: return cr_sinf(a);
	case CRS_MATH_COSINE: return cr_cosf(a);
	case CRS_MATH_TANGENT: return cr_tanf(a);
	case CRS_MATH_TO_RADIANS: return cr_div(a * CR_PI, 180.0f);                          /* transforms.c:18-20 */
	case CRS_MATH_TO_DEGREES: return a * cr_div(180.0f, CR_PI);                          /* transforms.c:22-24 */
	default: return 0.0f;
	}
}
/* converter/vecmath.c:43-83: the .v member of struct vectorValue; VecDot / VecLength fill .f only and leave .v zero */
static __device__ __noinline__ v3 cr_vec_op(unsigned op, v3 a, v3 b) {
	switch (op) {
	case CRS_VEC_ADD: return v3add(a, b);
	case CRS_VEC_SUBTRACT: return v3sub(a, b);
	case CRS_VEC_MULTIPLY: return v3mul(a, b);
	case CRS_VEC_AVERAGE: return v3scale(v3add(a, b), 0.5f);
	case CRS_VEC_CROSS: return v3cross(a, b);
	case CRS_VEC_NORMALIZE: return v3norm(a);
	case CRS_VEC_REFLECT: return v3reflect(a, b);
	case CRS_VEC_ABS: return v3make(fabsf(a.x), fabsf(a.y), fabsf(a.z));
	default: return v3make(0.0f, 0.0f, 0.0f);
	}
}
/* input/fresnel.c:43-55 (the reference evaluates IOR twice; the value is the same) */
static __device__ __noinline__ float cr_fresnel_value(const Rec &rec, float IOR) {
	float cosine;
	const float dn = v3dot(rec.inc_d, rec.n);
	if (dn > 0.0f) cosine = cr_div(IOR * v3dot(rec.inc_d, rec.n), v3len(rec.inc_d));
	else cosine = -cr_div(v3dot(rec.inc_d, rec.n), v3len(rec.inc_d));
	float r0 = cr_div(1.0f - IOR, 1.0f + IOR);                                           /* schlick, vector.h:268-272 */
	r0 = r0 * r0;
	return r0 + (1.0f - r0) * cr_pow5f(1.0f - cosine);
}

template <int E> struct NodeX {
	static __device__ __noinline__ col4 color(const DevScene &sc, int node, const Rec &rec) {
		const crs_node &n = sc.nodes[node];
		switch (n.kind) {
		case CRS_COLOR_CONSTANT: return c4make(n.f[0], n.f[1], n.f[2], n.f[3]);
		case CRS_COLOR_IMAGE: return cr_image_color(sc, n, rec);
		case CRS_COLOR_GRADIENT: return cr_gradient(n, rec);
		case CRS_COLOR_CHECKER: {                                                           /* checker.c:31-54 */
			const float coef = NodeX<E - 1>::value(sc, n.in[2], rec);
			float sines;
			if (rec.uv.x >= 0) sines = cr_sinf(coef * rec.uv.x) * cr_sinf(coef * rec.uv.y);
			else sines = cr_sinf(coef * rec.p.x) * cr_sinf(coef * rec.p.y) * cr_sinf(coef * rec.p.z);
			return NodeX<E - 1>::color(sc, sines < 0.0f ? n.in[0] : n.in[1], rec);
		}
		case CRS_COLOR_BLACKBODY: return cr_color_for_kelvin(NodeX<E - 1>::value(sc, n.in[0], rec));
		case CRS_COLOR_VECTOCOLOR: {                                                        /* vectocolor.c:38-43 */
			const v3 v = NodeX<E - 1>::vector(sc, n.in[0], rec);
			return c4make(v.x, v.y, v.z, 0.0f);
		}
		case CRS_COLOR_COMBINE_VALUE: {                                                     /* combine.c:38-43 */
			const float v = NodeX<E - 1>::value(sc, n.in[0], rec);
			return c4make(v, v, v, 1.0f);
		}
		case CRS_COLOR_COMBINE_RGB: {                                                       /* combinergb.c:44-53 */
			const float r = NodeX<E - 1>::value(sc, n.in[0], rec);
			const float g = NodeX<E - 1>::value(sc, n.in[1], rec);
			const float b = NodeX<E - 1>::value(sc, n.in[2], rec);
			return c4make(r, g, b, 1.0f);
		}
		default: return c4make(0.0f, 0.0f, 0.0f, 1.0f);
		}
	}
	static __device__ __noinline__ float value(const DevScene &sc, int node, const Rec &rec) {
		const crs_node &n = sc.nodes[node];
		switch (n.kind) {
		case CRS_VALUE_CONSTANT: return n.f[0];
		case CRS_VALUE_GRAYSCALE: return cr_grayscale(NodeX<E - 1>::color(sc, n.in[0], rec));
		case CRS_VALUE_ALPHA: return NodeX<E - 1>::color(sc, n.in[0], rec).a;
		case CRS_VALUE_MATH: {
			const float a = NodeX<E - 1>::value(sc, n.in[0], rec);
			const float b = NodeX<E - 1>::value(sc, n.in[1], rec);
			return cr_math_op(n.options, a, b);
		}
		case CRS_VALUE_FRESNEL: return cr_fresnel_value(rec, NodeX<E - 1>::value(sc, n.in[0], rec));
		case CRS_VALUE_RAYLENGTH: return rec.dist;                                          /* raylength.c:36-40 */
		default: return 0.0f;
		}
	}
	static __device__ __noinline__ v3 vector(const DevScene &sc, int node, const Rec &rec) {
		const crs_node &n = sc.nodes[node];
		switch (n.kind) {
		case CRS_VECTOR_CONSTANT: return v3make(n.f[0], n.f[1], n.f[2]);                    /* vectornode.c:38-42 */
		case CRS_VECTOR_NORMAL: return rec.n;                                               /* normal.c:36-40 */
		case CRS_VECTOR_VECMATH: {
			const v3 a = NodeX<E - 1>::vector(sc, n.in[0], rec);
			const v3 b = NodeX<E - 1>::vector(sc, n.in[1], rec);
			return cr_vec_op(n.options, a, b);
		}
		default: return v3make(0.0f, 0.0f, 0.0f);
		}
	}
};
template <> struct NodeX<0> {   /* leaves only */
	static __device__ __noinline__ col4 color(const DevScene &sc, int node, const Rec &rec) {
		const crs_node &n = sc.nodes[node];
		switch (n.kind) {
		case CRS_COLOR_CONSTANT: return c4make(n.f[0], n.f[1], n.f[2], n.f[3]);
		case CRS_COLOR_IMAGE: return cr_image_color(sc, n, rec);
		case CRS_COLOR_GRADIENT: return cr_gradient(n, rec);
		default: return c4make(0.0f, 0.0f, 0.0f, 1.0f);
		}
	}
	static __device__ __noinline__ float value(const DevScene &sc, int node, const Rec &rec) {
		const crs_node &n = sc.nodes[node];
		return n.kind == CRS_VALUE_CONSTANT ? n.f[0] : (n.kind == CRS_VALUE_RAYLENGTH ? rec.dist : 0.0f);
	}
	static __device__ __noinline__ v3 vector(const DevScene &sc, int node, const Rec &rec) {
		const crs_node &n = sc.nodes[node];
		return n.kind == CRS_VECTOR_CONSTANT ? v3make(n.f[0], n.f[1], n.f[2]) : (n.kind == CRS_VECTOR_NORMAL ? rec.n : v3make(0.0f, 0.0f, 0.0f));
	}
};
static __device__ __noinline__ col4 cr_xnode_color(const DevScene &sc, int node, const Rec &rec) { return NodeX<CRG_XNODE_DEPTH>::color(sc, node, rec); }
static __device__ __noinline__ float cr_xnode_value(const DevScene &sc, int node, const Rec &rec) { return NodeX<CRG_XNODE_DEPTH>::value(sc, node, rec); }

/* ---- vector.h:252-272 --------------------------------------------------------------------------------------------------- */
CRD bool cr_refract(v3 in, v3 normal, float niOverNt, v3 &refracted) {
	const v3 uv = v3norm(in);
	const float dt = v3dot(uv, normal);
	const float disc = 1.0f - niOverNt * niOverNt * (1.0f - dt * dt);
	if (disc > 0.0f) {
		const v3 A = v3scale(normal, dt);
		const v3 B = v3sub(uv, A);
		const v3 C = v3scale(B, niOverNt);
		const v3 D = v3scale(normal, cr_sqrtf(disc));
		refracted = v3sub(C, D);
		return true;
	}
	return false;
}
CRD float cr_schlick(float cosine, float IOR) {
	float r0 = cr_div(1.0f - IOR, 1.0f + IOR);
	r0 = r0 * r0;
	return r0 + (1.0f - r0) * cr_pow5f(1.0f - cosine);
}
/* shared by glass.c:53-67 and plastic.c:60-74 */
CRD float cr_fresnel_probability(const Rec &rec, float IOR, v3 &refracted) {
	v3 outward;
	float niOverNt, cosine;
	const float dn = v3dot(rec.inc_d, rec.n);
	if (dn > 0.0f) {
		outward = v3neg(rec.n);
		niOverNt = IOR;
		cosine = cr_div(IOR * dn, v3len(rec.inc_d));
	} else {
		outward = rec.n;
		niOverNt = cr_div(1.0f, IOR);
		cosine = -cr_div(dn, v3len(rec.inc_d));
	}
	if (cr_refract(rec.inc_d, outward, niOverNt, refracted)) return cr_schlick(cosine, IOR);
	return 1.0f;
}

/* one non-composite bsdf node; returns false when `node` is MIX/PLASTIC(diffuse branch)/ADD and sets next */
template <bool X>
CRD BsdfSample cr_sample_leaf(const DevScene &sc, const crs_node &n, uint64_t &rng, const Rec &rec) {
	BsdfSample s;
	switch (n.kind) {
	case CRS_BSDF_DIFFUSE:                                                                  /* diffuse.c:40-47 */
		s.out = v3norm(v3add(rec.n, cr_random_on_unit_sphere(rng)));
		s.color = NodesT<X>::color(sc, n.in[0], rec);
		return s;
	case CRS_BSDF_ISOTROPIC:                                                                /* isotropic.c:40-47 */
		s.out = v3norm(cr_random_on_unit_sphere(rng));
		s.color = NodesT<X>::color(sc, n.in[0], rec);
		return s;
	case CRS_BSDF_EMISSIVE: {                                                               /* emission.c:42-49 */
		s.out = v3norm(v3add(rec.n, cr_random_on_unit_sphere(rng)));
		const float strength = NodesT<X>::value(sc, n.in[1], rec);
		s.color = c4coef(strength, NodesT<X>::color(sc, n.in[0], rec));
		return s;
	}
	case CRS_BSDF_METAL: {                                                                  /* metal.c:40-55 */
		const v3 nd = v3norm(rec.inc_d);
		v3 reflected = v3reflect(nd, rec.n);
		const float rough = NodesT<X>::value(sc, n.in[1], rec);
		if (rough > 0.0f) reflected = v3add(reflected, v3scale(cr_random_on_unit_sphere(rng), rough));
		s.out = reflected;
		s.color = NodesT<X>::color(sc, n.in[0], rec);
		return s;
	}
	case CRS_BSDF_GLASS: {                                                                  /* glass.c:41-87 */
		/* glass.c:47 reads an uninitialised `refracted` when refract() failed and the draw is exactly 1.0f; defined as
		 * "total internal reflection always reflects" (DESIGN.md deviation #3, same as oracle/cray_oracle.c) */
		v3 reflected = v3reflect(rec.inc_d, rec.n);
		v3 refracted = reflected;
		const float IOR = NodesT<X>::value(sc, n.in[2], rec);
		const float prob = cr_fresnel_probability(rec, IOR, refracted);
		const float rough = NodesT<X>::value(sc, n.in[1], rec);
		if (rough > 0.0f) {
			const v3 fuzz = v3scale(cr_random_on_unit_sphere(rng), rough);
			reflected = v3add(reflected, fuzz);
			refracted = v3add(refracted, fuzz);
		}
		s.out = cr_draw(rng) < prob ? reflected : refracted;
		s.color = NodesT<X>::color(sc, n.in[0], rec);
		return s;
	}
	case CRS_BSDF_TRANSPARENT:                                                              /* transparent.c:40-44 */
		s.out = rec.inc_d;
		s.color = NodesT<X>::color(sc, n.in[0], rec);
		return s;
	default:
		s.out = v3make(0.0f, 0.0f, 0.0f);
		s.color = c4make(0.0f, 0.0f, 0.0f, 1.0f);
		return s;
	}
}

/* material.bsdf->sample(...) — pathtrace.c:46.  Explicit-stack evaluation of the bsdf tree: MIX and
 * PLASTIC→diffuse are tail calls; ADD pushes "combine" + B and continues with A, so A's draws come
 * before B's exactly as add.c:44-45. */
#define CRG_COMBINE (-2)
template <bool X>
CRD BsdfSample cr_sample_bsdf(const DevScene &sc, int root, uint64_t &rng, const Rec &rec) {
	int todo[CRG_ADD_STACK];
	BsdfSample vals[CRG_ADD_STACK / 2 + 1];
	int nt = 0, nv = 0;
	int node = root;
	while (true) {
		BsdfSample s;
		bool have = false;
		while (!have) {
			const crs_node &n = sc.nodes[node];
			if (n.kind == CRS_BSDF_MIX) {                                                   /* mix.c:42-50 */
				const float lerp = NodesT<X>::value(sc, n.in[2], rec);
				node = (cr_draw(rng) > lerp) ? n.in[0] : n.in[1];
			} else if (n.kind == CRS_BSDF_PLASTIC) {                                        /* plastic.c:42-87 */
				v3 refracted;
				const float prob = cr_fresnel_probability(rec, rec.IOR, refracted);
				if (cr_draw(rng) < prob) {                                                  /* sampleShiny :42-56 */
					v3 reflected = v3reflect(rec.inc_d, rec.n);
					const float rough = NodesT<X>::color(sc, n.in[1], rec).r;
					if (rough > 0.0f) reflected = v3add(reflected, v3scale(cr_random_on_unit_sphere(rng), rough));
					s.out = reflected;
					s.color = c4make(1.0f, 1.0f, 1.0f, 1.0f);
					have = true;
				} else {
					node = n.in[2];
				}
			} else if (n.kind == CRS_BSDF_ADD && nt + 2 <= CRG_ADD_STACK) {                 /* add.c:42-49 */
				todo[nt++] = CRG_COMBINE;
				todo[nt++] = n.in[1];
				node = n.in[0];
			} else {
				s = cr_sample_leaf<X>(sc, n, rng, rec);    /* (an over-deep ADD falls to the black default; rejected at upload) */
				have = true;
			}
		}
		if (nt == 0) return s;                          /* common case: no ADD in the graph */
		vals[nv++] = s;
		while (nt > 0 && todo[nt - 1] == CRG_COMBINE) {
			--nt;
			const BsdfSample b = vals[--nv];
			const BsdfSample a = vals[--nv];
			BsdfSample r;
			r.out = v3add(a.out, b.out);
			r.color = c4add(a.color, b.color);
			vals[nv++] = r;
		}
		if (nt == 0) return vals[0];
		node = todo[--nt];
	}
}

/* scene->background->sample(...) — background.c:39-66 (pathtrace.c:40) */
template <bool X>
static __device__ __noinline__ col4 cr_sample_background(const DevScene &sc, v3 dir) {
	const crs_node &n = sc.nodes[sc.background];
	Rec rec;
	rec.inc_d = dir;
	rec.p = v3make(0.0f, 0.0f, 0.0f);
	rec.n = v3make(0.0f, 0.0f, 0.0f);
	rec.uv.x = 0.0f; rec.uv.y = 0.0f;
	rec.IOR = 0.0f;
	rec.dist = CR_FLT_MAX;                                                                   /* pathtrace.c:27 */
	const v3 ud = v3norm(dir);
	const float phi = cr_div(cr_atan2f(ud.z, ud.x), 4.0f) + NodesT<X>::value(sc, n.in[2], rec);
	const float theta = cr_acosf(cr_div(-ud.y, 1.0f));
	float u = cr_div(theta, CR_PI);
	float v = cr_div(phi, CR_PI / 2.0f);
	u = cr_wrapMinMax(u, 0.0f, 1.0f);
	v = cr_wrapMinMax(v, 0.0f, 1.0f);
	rec.uv.x = v; rec.uv.y = u;
	const float strength = NodesT<X>::value(sc, n.in[1], rec);
	return c4coef(strength, NodesT<X>::color(sc, n.in[0], rec));
}

/* ---- hit reconstruction: everything intersectSphere/intersectMesh do after the closest primitive is known ------------------ */
CRD void cr_texmap_sphere(v3 ud, v2 &uv) {                                                  /* instance.c:33-43 */
	const float phi = cr_atan2f(ud.z, ud.x);
	const float theta = cr_asinf(ud.y);
	float v = cr_div(theta + CR_PI / 2.0f, CR_PI);
	float u = 1.0f - cr_div(phi + CR_PI, CR_PI * 2.0f);
	u = cr_wrapMinMax(u, 0.0f, 1.0f);
	v = cr_wrapMinMax(v, 0.0f, 1.0f);
	uv.x = u; uv.y = v;
}

/* fills rec (hitPoint, surfaceNormal, uv, IOR) and returns the global material index */
CRD int cr_reconstruct_hit(const DevScene &sc, v3 o, v3 d, const Hit &hit, Rec &rec, bool force_uv) {
	const DevInstance *inst = sc.instances + hit.inst;
	const float4 *m4 = reinterpret_cast<const float4 *>(inst->Ainv);
	float Ainv[12], A[12];
	{
		const float4 r0 = __ldg(m4 + 0), r1 = __ldg(m4 + 1), r2 = __ldg(m4 + 2);
		const float4 a0 = __ldg(m4 + 3), a1 = __ldg(m4 + 4), a2 = __ldg(m4 + 5);
		Ainv[0] = r0.x; Ainv[1] = r0.y; Ainv[2] = r0.z; Ainv[3] = r0.w; Ainv[4] = r1.x; Ainv[5] = r1.y; Ainv[6] = r1.z; Ainv[7] = r1.w;
		Ainv[8] = r2.x; Ainv[9] = r2.y; Ainv[10] = r2.z; Ainv[11] = r2.w;
		A[0] = a0.x; A[1] = a0.y; A[2] = a0.z; A[3] = a0.w; A[4] = a1.x; A[5] = a1.y; A[6] = a1.z; A[7] = a1.w;
		A[8] = a2.x; A[9] = a2.y; A[10] = a2.z; A[11] = a2.w;
	}
	const uint4 meta = __ldg(reinterpret_cast<const uint4 *>(&inst->kind));
	v3 oo, od;
	cr_object_ray(Ainv, __uint_as_float(meta.z), o, d, oo, od);
	const v3 p_obj = v3add(oo, v3scale(od, hit.t));                                         /* alongRay(copy, t) */
	rec.inc_d = d;
	rec.dist = hit.t;
	int material;
	if (meta.x == CRS_INST_MESH) {
		const uint32_t poly = __ldg(sc.slot_poly + hit.prim);
		const float4 *s4 = reinterpret_cast<const float4 *>(sc.spolys + poly);
		const float4 a = __ldg(s4 + 0), b = __ldg(s4 + 1), c = __ldg(s4 + 2), e = __ldg(s4 + 3);
		const uint4 f = __ldg(reinterpret_cast<const uint4 *>(s4 + 4));
		/* a=(n0.xyz,n1.x) b=(n1.yz,n2.xy) c=(n2.z,t0.xy,t1.x) e=(t1.y,t2.xy,material) f=(flags,...) */
		const float u = hit.u, v = hit.v;
		const float w = 1.0f - u - v;
		const uint32_t flags = f.x;
		v3 nrm;
		if (flags & 1u) {                                                                   /* poly.c:39-44 */
			const v3 up = v3scale(v3make(a.w, b.x, b.y), u);
			const v3 vp = v3scale(v3make(b.z, b.w, c.x), v);
			const v3 wp = v3scale(v3make(a.x, a.y, a.z), w);
			nrm = v3add(v3add(up, vp), wp);
		} else {
			nrm = v3make(a.x, a.y, a.z);                                                    /* n = e1 x e2 */
		}
		if (flags & 2u) {                                                                   /* instance.c:150-167 */
			const float ucx = c.w * u, ucy = e.x * u;        /* t1 * u */
			const float vcx = e.y * v, vcy = e.z * v;        /* t2 * v */
			const float wcx = c.y * w, wcy = c.z * w;        /* t0 * w */
			rec.uv.x = (ucx + vcx) + wcx;
			rec.uv.y = (ucy + vcy) + wcy;
		} else {
			rec.uv.x = -1.0f; rec.uv.y = -1.0f;
		}
		material = (int)__float_as_uint(e.w);
		rec.p = xf_point(A, p_obj);
		rec.n = v3norm(xf_vector_transpose(Ainv, nrm));                                     /* instance.c:179-181 */
	} else {
		const v3 nobj = v3norm(p_obj);                                                      /* sphere.c:56 */
		material = (int)__ldg(&inst->material);
		if (force_uv || (sc.materials[material].flags & 1u)) cr_texmap_sphere(nobj, rec.uv);
		else { rec.uv.x = 0.0f; rec.uv.y = 0.0f; }   /* uv is dead: no node of this material's graph reads it */
		rec.p = xf_point(A, p_obj);
		rec.n = xf_vector_transpose(Ainv, nobj);                                            /* not renormalised, instance.c:56 */
	}
	rec.IOR = sc.materials[material].IOR;
	return material;
}
